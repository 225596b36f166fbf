// A9-A11 semi-Lagrangian advection and N1 MacCormack.
//
// One thread per sample point of the advected field.  The velocity at the sample point comes from shift resampling
// (phi/field/_resample.py:341-364 -> PhiML/phiml/math/_nd.py:973-1003): identity for the component the face belongs
// to, 0.5/0.5 averages along every half-offset axis otherwise, ghost values from the velocity's boundary.
// The back-traced position is kept as (integer sample index, displacement in cells): the displacement
// -dt*v/dx is what the reference computes in world space (advect.py:20-24, _resample.py:257-258), and splitting it
// off keeps the interpolation weights accurate to fp32 epsilon instead of eps * resolution.
// Interpolation mirrors the NumPy-backend fallback (PhiML/phiml/math/_ops.py:1010-1014): weights are products
// over the axes of frac or (1 - frac), the result is the weighted sum over the 2^d neighbours, neighbours outside
// the array follow the field's boundary (periodic: wrap, zero-gradient: clamp, constant: the constant).
#include "phi_internal.cuh"
#include "launch.cuh"

template <int DIM, class T>
__device__ __forceinline__ T phi_velocity_at(const DGridT<T>& g, const DVecT<T>& vel, int a, int target, int b, int x, int y, int z)
{
    const T* va = vel.p[a];
    const DFieldT<T>& fa = vel.f[a];
    const T h = 0.5;
    if (target == a) return phi_fetch<DIM>(va, g, fa, b, x, y, z);
    const int ax = (a == 0), ay = (a == 1), az = (a == 2);
    {   // interior fast path: the bounding box of the 2 / 4 needed values lies inside the stored range
        const int t_ = target;
        const int x0 = x - (t_ == 0), y0 = y - (t_ == 1), z0 = z - (t_ == 2);
        bool inside = x0 >= fa.lo[0] && x + ax <= fa.hi[0] && y0 >= fa.lo[1] && y + ay <= fa.hi[1];
        if (DIM == 3) inside = inside && z0 >= fa.lo[2] && z + az <= fa.hi[2];
        if (inside) {
            const T* p = va + (long long)b * fa.sb + (DIM == 3 ? (long long)z * fa.sz : 0) + (long long)y * fa.sy + x;
            const long long sa = a == 0 ? 1 : (a == 1 ? fa.sy : fa.sz);
            if (t_ < 0) return __ldg(p + sa) * h + __ldg(p) * h;
            const long long st = t_ == 0 ? 1 : (t_ == 1 ? fa.sy : fa.sz);
            const T f00 = __ldg(p - st), f10 = __ldg(p - st + sa), f01 = __ldg(p), f11 = __ldg(p + sa);
            if (a < t_) { const T u0 = f10 * h + f00 * h, u1 = f11 * h + f01 * h; return u1 * h + u0 * h; }
            const T w0 = f01 * h + f00 * h, w1 = f11 * h + f10 * h;
            return w1 * h + w0 * h;
        }
    }
    if (target < 0) {                                       // cell centre: average the two faces of the cell along a
        const T lo = phi_fetch<DIM>(va, g, fa, b, x, y, z);
        const T hi = phi_fetch<DIM>(va, g, fa, b, x + ax, y + ay, z + az);
        return hi * h + lo * h;
    }
    const int t = target;
    const int tx = (t == 0), ty = (t == 1), tz = (t == 2);
    // four values: offsets da in {0,1} along a (faces of the cell), dt in {-1,0} along t (cells adjacent to the face)
    const T f00 = phi_fetch<DIM>(va, g, fa, b, x - tx, y - ty, z - tz);
    const T f10 = phi_fetch<DIM>(va, g, fa, b, x - tx + ax, y - ty + ay, z - tz + az);
    const T f01 = phi_fetch<DIM>(va, g, fa, b, x, y, z);
    const T f11 = phi_fetch<DIM>(va, g, fa, b, x + ax, y + ay, z + az);
    if (a < t) {       // sample_subgrid lerps the axes in spatial order: first a, then t
        const T u0 = f10 * h + f00 * h;
        const T u1 = f11 * h + f01 * h;
        return u1 * h + u0 * h;
    } else {           // first t, then a
        const T w0 = f01 * h + f00 * h;
        const T w1 = f11 * h + f10 * h;
        return w1 * h + w0 * h;
    }
}

template <class T>
struct Lookup { int i[3]; T t[3]; };    // base neighbour index and interpolation weight per axis

template <int DIM, class T>
__device__ __forceinline__ Lookup<T> phi_lookup(const DGridT<T>& g, const DVecT<T>& vel, int target, int b, int x, int y, int z, T dt)
{
    Lookup<T> L;
    const int idx[3] = {x, y, z};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (a >= DIM) { L.i[a] = 0; L.t[a] = 0; continue; }
        const T v = phi_velocity_at<DIM>(g, vel, a, target, b, x, y, z);
        const T delta = phi_div(-dt * v, g.dx[a], g.inv_dx[a]);
        const T fl = phi_floor(delta);
        L.i[a] = idx[a] + (int)fl;
        L.t[a] = delta - fl;
    }
    return L;
}

template <int DIM, bool LIMITS, class T>
__device__ __forceinline__ T phi_interp(const T* __restrict__ a, const DGridT<T>& g, const DFieldT<T>& f, int b, const Lookup<T>& L,
                                        T* vmin, T* vmax)
{
    const T one = 1;
    T acc = 0;
    T mn = 3.4e38f, mx = -3.4e38f;
    // interior fast path: all 2^d neighbours are stored values -> plain strided loads, same weights and summation order
    bool inside = L.i[0] >= f.lo[0] && L.i[0] + 1 <= f.hi[0] && L.i[1] >= f.lo[1] && L.i[1] + 1 <= f.hi[1];
    if (DIM == 3) inside = inside && L.i[2] >= f.lo[2] && L.i[2] + 1 <= f.hi[2];
    if (inside) {
        const T* p = a + (long long)b * f.sb + (DIM == 3 ? (long long)L.i[2] * f.sz : 0) + (long long)L.i[1] * f.sy + L.i[0];
        const T tx = L.t[0], ty = L.t[1], tz = L.t[2];
        const T n00 = __ldg(p), n10 = __ldg(p + 1), n01 = __ldg(p + f.sy), n11 = __ldg(p + f.sy + 1);
        if (DIM == 3) {
            const T m00 = __ldg(p + f.sz), m10 = __ldg(p + f.sz + 1), m01 = __ldg(p + f.sz + f.sy), m11 = __ldg(p + f.sz + f.sy + 1);
            const T w00 = (one - tx) * (one - ty), w01 = (one - tx) * ty, w10 = tx * (one - ty), w11 = tx * ty;
            acc += n00 * (w00 * (one - tz)); acc += m00 * (w00 * tz);
            acc += n01 * (w01 * (one - tz)); acc += m01 * (w01 * tz);
            acc += n10 * (w10 * (one - tz)); acc += m10 * (w10 * tz);
            acc += n11 * (w11 * (one - tz)); acc += m11 * (w11 * tz);
            if (LIMITS) { mn = phi_min(phi_min(phi_min(n00, n10), phi_min(n01, n11)), phi_min(phi_min(m00, m10), phi_min(m01, m11)));
                          mx = phi_max(phi_max(phi_max(n00, n10), phi_max(n01, n11)), phi_max(phi_max(m00, m10), phi_max(m01, m11))); }
        } else {
            acc += n00 * ((one - tx) * (one - ty)); acc += n01 * ((one - tx) * ty);
            acc += n10 * (tx * (one - ty)); acc += n11 * (tx * ty);
            if (LIMITS) { mn = phi_min(phi_min(n00, n10), phi_min(n01, n11)); mx = phi_max(phi_max(n00, n10), phi_max(n01, n11)); }
        }
        if (LIMITS) { *vmin = mn; *vmax = mx; }
        return acc;
    }
#pragma unroll
    for (int cx = 0; cx < 2; ++cx) {
        const T wx = cx ? L.t[0] : one - L.t[0];
#pragma unroll
        for (int cy = 0; cy < 2; ++cy) {
            const T wxy = wx * (cy ? L.t[1] : one - L.t[1]);
            if (DIM == 3) {
#pragma unroll
                for (int cz = 0; cz < 2; ++cz) {
                    const T w = wxy * (cz ? L.t[2] : one - L.t[2]);
                    const T n = phi_fetch<DIM>(a, g, f, b, L.i[0] + cx, L.i[1] + cy, L.i[2] + cz);
                    acc += n * w;
                    if (LIMITS) { mn = phi_min(mn, n); mx = phi_max(mx, n); }
                }
            } else {
                const T n = phi_fetch<DIM>(a, g, f, b, L.i[0] + cx, L.i[1] + cy, 0);
                acc += n * wxy;
                if (LIMITS) { mn = phi_min(mn, n); mx = phi_max(mx, n); }
            }
        }
    }
    if (LIMITS) { *vmin = mn; *vmax = mx; }
    return acc;
}

template <int DIM, class T>
__device__ __forceinline__ bool advect_index(const DGridT<T>& g, const DFieldT<T>& ff, int& b, int& x, int& y, int& z)
{
    x = blockIdx.x * blockDim.x + threadIdx.x;
    y = blockIdx.y;
    const int zb = blockIdx.z;
    if (DIM == 3) { z = zb % g.fext[2]; b = zb / g.fext[2]; } else { z = 0; b = zb; }
    if (x > ff.hi[0] || x < ff.lo[0] || y > ff.hi[1] || y < ff.lo[1]) return false;
    if (DIM == 3 && (z > ff.hi[2] || z < ff.lo[2])) return false;
    return true;
}

template <int DIM, class T>
__global__ void __launch_bounds__(128)
k_advect(DGridT<T> g, DVecT<T> vel, DFieldT<T> ff, int target, const T* __restrict__ src, T* __restrict__ dst, T dt)
{
    int b, x, y, z;
    if (!advect_index<DIM>(g, ff, b, x, y, z)) return;
    const Lookup<T> L = phi_lookup<DIM>(g, vel, target, b, x, y, z, dt);
    const T r = phi_interp<DIM, false, T>(src, g, ff, b, L, nullptr, nullptr);
    dst[(long long)b * ff.sb + (long long)z * ff.sz + (long long)y * ff.sy + x] = r;
}

// MacCormack (advect.py:182-215) = three passes over proven building blocks:
//   fwd = semi_lagrangian(field, dt)            (k_advect)
//   bwd = sample(fwd, x + dt v)                 (k_advect with -dt)
//   new = fwd + strength*0.5*(field - bwd), clamped to the min/max of the 2^d neighbours of the backward lookup
template <int DIM>
__global__ void __launch_bounds__(128)
k_mac_cormack_combine(DGrid g, DVec vel, DField ff, const float* __restrict__ src, const float* __restrict__ fwd,
                      float* bwd_dst, float dt, float half_strength)
{
    int b, x, y, z;
    if (!advect_index<DIM>(g, ff, b, x, y, z)) return;
    const long long off = (long long)b * ff.sb + (long long)z * ff.sz + (long long)y * ff.sy + x;
    const Lookup<float> Lb = phi_lookup<DIM>(g, vel, -1, b, x, y, z, dt);
    float mn, mx;
    (void)phi_interp<DIM, true>(src, g, ff, b, Lb, &mn, &mx);
    const float nv = fwd[off] + half_strength * (src[off] - bwd_dst[off]);
    bwd_dst[off] = fminf(fmaxf(nv, mn), mx);
}

template <class T>
static dim3 scalar_grid(const DGridT<T>& g)
{
    return dim3((g.fext[0] + 127) / 128, g.fext[1], g.fext[2] * g.batch);
}

template <class T>
static int launch_advect(const DGridT<T>& g, const DVecT<T>& vel, const DFieldT<T>& ff, int target_comp, const T* src, T* dst,
                         T dt, cudaStream_t s)
{
    if (g.dim == 3) k_advect<3, T><<<scalar_grid(g), 128, 0, s>>>(g, vel, ff, target_comp, src, dst, dt);
    else            k_advect<2, T><<<scalar_grid(g), 128, 0, s>>>(g, vel, ff, target_comp, src, dst, dt);
    return (int)cudaGetLastError();
}

int phi_launch_advect(const DGrid& g, const DVec& vel, const DField& ff, int target_comp, const float* src, float* dst,
                      float dt, cudaStream_t s)
{
    return launch_advect<float>(g, vel, ff, target_comp, src, dst, dt, s);
}

int phi_launch_advect(const DGridT<double>& g, const DVecT<double>& vel, const DFieldT<double>& ff, int target_comp, const double* src,
                      double* dst, double dt, cudaStream_t s)
{
    return launch_advect<double>(g, vel, ff, target_comp, src, dst, dt, s);
}

int phi_launch_mac_cormack(const DGrid& g, const DVec& vel, const DField& ff, const float* src, float* dst, float* tmp,
                           float dt, float strength, cudaStream_t s)
{
    const bool vec = !phi_scalar_kernels() && (long long)g.fext[0] * g.fext[1] * g.fext[2] * g.batch < (1ll << 31) - (1ll << 20);
    int err = vec ? phi_launch_advect_centered_vec(g, vel, ff, src, tmp, dt, nullptr, 0.f, s) : phi_launch_advect(g, vel, ff, -1, src, tmp, dt, s);
    if (err) return err;
    err = vec ? phi_launch_advect_centered_vec(g, vel, ff, tmp, dst, -dt, nullptr, 0.f, s) : phi_launch_advect(g, vel, ff, -1, tmp, dst, -dt, s);
    if (err) return err;
    const float hs = strength * 0.5f;
    if (g.dim == 3) k_mac_cormack_combine<3><<<scalar_grid(g), 128, 0, s>>>(g, vel, ff, src, tmp, dst, dt, hs);
    else            k_mac_cormack_combine<2><<<scalar_grid(g), 128, 0, s>>>(g, vel, ff, src, tmp, dst, dt, hs);
    return (int)cudaGetLastError();
}
