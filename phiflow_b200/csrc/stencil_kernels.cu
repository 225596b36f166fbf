// Finite-difference stencils of the projection step: laplace (A7), divergence (A5), gradient subtraction (A6),
// plus the two small per-step helpers of the notebook step (inflow axpy, buoyancy resampling, N2).
#include "phi_internal.cuh"
#include "launch.cuh"

// ---------------------------------------------------------------------------------------------------------
// A7  laplace  --  marching stencil, 8 B/cell (read x once, write y once)
// ---------------------------------------------------------------------------------------------------------
template <bool AXPY>
struct EpiLaplace {
    float* y; float coeff;
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid)
    {
        float4 o = q;
        if (AXPY) { o.x = c.x + coeff * q.x; o.y = c.y + coeff * q.y; o.z = c.z + coeff * q.z; o.w = c.w + coeff * q.w; }
        if (nvalid == 4) { *reinterpret_cast<float4*>(y + off) = o; }
        else { for (int j = 0; j < nvalid; ++j) y[off + j] = f4_get(o, j); }
    }
};

template <int DIM, bool AXPY>
__global__ void __launch_bounds__(PHI_WARPS_PER_CTA * 32)
k_laplace(DGrid g, DField f, UnitMap um, const float* __restrict__ x, float* __restrict__ y, float coeff)
{
    const int warp = threadIdx.x >> 5;
    for (int unit = blockIdx.x; unit < um.total_units; unit += gridDim.x) {
        const WarpUnit w = phi_warp_unit<DIM>(g, um, unit, warp);
        if (!w.valid) continue;
        SrcArray src{x};
        EpiLaplace<AXPY> epi{y, coeff};
        phi_march<DIM>(g, f, src, epi, w.b, w.xt0, w.t, w.m0, w.m1);
    }
}

int phi_launch_laplace(const DGrid& g, const DField& f, const float* x, float* y, float coeff, bool axpy, cudaStream_t s)
{
    if (phi_ring_enabled()) {
        const int e = phi_launch_laplace_ring(g, f, x, y, coeff, axpy, s);
        if (e != -100) return e;
    }
    UnitMap um = phi_make_unit_map(g, phi_sm_count() * 16);
    const int blocks = um.total_units;
    dim3 block(PHI_WARPS_PER_CTA * 32);
    if (g.dim == 3) {
        if (axpy) k_laplace<3, true><<<blocks, block, 0, s>>>(g, f, um, x, y, coeff);
        else      k_laplace<3, false><<<blocks, block, 0, s>>>(g, f, um, x, y, coeff);
    } else {
        if (axpy) k_laplace<2, true><<<blocks, block, 0, s>>>(g, f, um, x, y, coeff);
        else      k_laplace<2, false><<<blocks, block, 0, s>>>(g, f, um, x, y, coeff);
    }
    PhiLaunchInfo li = {}; li.kernel = PHI_KERNEL_LAPLACE_MARCH; li.generic = 1; li.total_units = um.total_units; li.grid_ctas = blocks;
    phi_note_launch(li);
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// Scalar (one thread per sample) kernels.  Index space = allocated extent so that upper boundary faces are covered.
// ---------------------------------------------------------------------------------------------------------
struct Idx { int b, x, y, z; };

template <int DIM>
__device__ __forceinline__ bool phi_thread_index(const DGrid& g, Idx& i)
{
    i.x = blockIdx.x * blockDim.x + threadIdx.x;
    i.y = blockIdx.y;
    const int zb = blockIdx.z;
    if (DIM == 3) { i.z = zb % g.fext[2]; i.b = zb / g.fext[2]; } else { i.z = 0; i.b = zb; }
    return i.x < g.fext[0];
}

__device__ __forceinline__ bool phi_in_range(const DField& f, int dim, int x, int y, int z)
{
    bool ok = x >= f.lo[0] && x <= f.hi[0] && y >= f.lo[1] && y <= f.hi[1];
    if (dim == 3) ok = ok && z >= f.lo[2] && z <= f.hi[2];
    return ok;
}

__device__ __forceinline__ long long phi_off(const DField& f, const Idx& i)
{
    return (long long)i.b * f.sb + (long long)i.z * f.sz + (long long)i.y * f.sy + i.x;
}

// A5: div = sum_d (v_d[i + e_d] - v_d[i]) / dx_d over the n_d + 1 faces of the baked field
template <int DIM>
__global__ void __launch_bounds__(128)
k_divergence(DGrid g, DVec v, DField cf, float* __restrict__ div, const float* __restrict__ accm)
{
    Idx i;
    if (!phi_thread_index<DIM>(g, i)) return;
    if (i.x >= g.n[0] || i.y >= g.n[1] || i.z >= g.n[2]) return;
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < DIM; ++c) {
        const float lo = phi_fetch<DIM>(v.p[c], g, v.f[c], i.b, i.x, i.y, i.z);
        const float hi = phi_fetch<DIM>(v.p[c], g, v.f[c], i.b, i.x + (c == 0), i.y + (c == 1), i.z + (c == 2));
        const float term = phi_div(hi - lo, g.dx[c], g.inv_dx[c]);
        acc = (c == 0) ? term : acc + term;
    }
    const long long o = phi_off(cf, i);
    div[o] = accm ? acc * accm[o] : acc;
}

// A6: v_d[face] -= (p[upper cell] - p[lower cell]) / dx_d on the stored faces
template <int DIM>
__global__ void __launch_bounds__(128)
k_grad_sub(DGrid g, DVec vin, DVecOut v, DField pf, const float* __restrict__ p, DField af, const float* __restrict__ accm)
{
    Idx i;
    if (!phi_thread_index<DIM>(g, i)) return;
    const long long off = phi_off(vin.f[0], i);
#pragma unroll
    for (int c = 0; c < DIM; ++c) {
        if (!phi_in_range(vin.f[c], DIM, i.x, i.y, i.z)) continue;
        const float up = phi_fetch<DIM>(p, g, pf, i.b, i.x, i.y, i.z);
        const float lw = phi_fetch<DIM>(p, g, pf, i.b, i.x - (c == 0), i.y - (c == 1), i.z - (c == 2));
        float grad = phi_div(up - lw, g.dx[c], g.inv_dx[c]);
        if (accm) {     // hard_bcs = min of the two adjacent cells' accessibility (fluid.py:134)
            const float au = phi_fetch<DIM>(accm, g, af, i.b, i.x, i.y, i.z);
            const float al = phi_fetch<DIM>(accm, g, af, i.b, i.x - (c == 0), i.y - (c == 1), i.z - (c == 2));
            grad *= fminf(au, al);
        }
        v.p[c][off] = vin.p[c][off] - grad;
    }
}

// N2: v_c[face] += ((s*b_c)[upper]*0.5 + (s*b_c)[lower]*0.5) * dt on the stored faces; a constant ghost of s stays c (not c * b_c,
// phi_fetch_scaled), so a face next to a constant side gets c/2 * dt even for b_c = 0
template <int DIM>
__global__ void __launch_bounds__(128)
k_buoyancy(DGrid g, DVec vin, DVecOut v, DField sf, const float* __restrict__ s, float b0, float b1, float b2, float dt)
{
    Idx i;
    if (!phi_thread_index<DIM>(g, i)) return;
    const long long off = phi_off(vin.f[0], i);
#pragma unroll
    for (int c = 0; c < DIM; ++c) {
        const float bc = c == 0 ? b0 : (c == 1 ? b1 : b2);
        if (!phi_in_range(vin.f[c], DIM, i.x, i.y, i.z)) continue;
        const float up = phi_fetch_scaled<DIM>(s, g, sf, i.b, i.x, i.y, i.z, bc);
        const float lw = phi_fetch_scaled<DIM>(s, g, sf, i.b, i.x - (c == 0), i.y - (c == 1), i.z - (c == 2), bc);
        v.p[c][off] = vin.p[c][off] + (up * 0.5f + lw * 0.5f) * dt;
    }
}

// N4: apply_boundary_conditions for stationary obstacles: v_c *= mask_c on the stored faces (fluid.py:212-240)
template <int DIM>
__global__ void __launch_bounds__(128)
k_mul_faces(DGrid g, DVec vin, DVecOut v, const float* m0, const float* m1, const float* m2)
{
    Idx i;
    if (!phi_thread_index<DIM>(g, i)) return;
    const long long off = phi_off(vin.f[0], i);
#pragma unroll
    for (int c = 0; c < DIM; ++c) {
        if (!phi_in_range(vin.f[c], DIM, i.x, i.y, i.z)) continue;
        const float* m = c == 0 ? m0 : (c == 1 ? m1 : m2);
        v.p[c][off] = vin.p[c][off] * m[off];
    }
}

template <int DIM>
__global__ void __launch_bounds__(128)
k_axpy(DGrid g, DField cf, float a, const float* __restrict__ x, float* __restrict__ y)
{
    Idx i;
    if (!phi_thread_index<DIM>(g, i)) return;
    if (i.x >= g.n[0] || i.y >= g.n[1] || i.z >= g.n[2]) return;
    const long long off = phi_off(cf, i);
    y[off] = y[off] + a * x[off];
}

static dim3 scalar_grid(const DGrid& g)
{
    return dim3((g.fext[0] + 127) / 128, g.fext[1], g.fext[2] * g.batch);
}

int phi_launch_divergence(const DGrid& g, const DVec& v, const DField& cf, float* div, const float* acc, cudaStream_t s)
{
    if (g.dim == 3) k_divergence<3><<<scalar_grid(g), 128, 0, s>>>(g, v, cf, div, acc);
    else            k_divergence<2><<<scalar_grid(g), 128, 0, s>>>(g, v, cf, div, acc);
    return (int)cudaGetLastError();
}

int phi_launch_grad_sub(const DGrid& g, const DVec& vin, const DVecOut& v, const DField& pf, const float* p,
                        const DField* af, const float* acc, cudaStream_t s)
{
    const DField a = af ? *af : pf;
    if (g.dim == 3) k_grad_sub<3><<<scalar_grid(g), 128, 0, s>>>(g, vin, v, pf, p, a, acc);
    else            k_grad_sub<2><<<scalar_grid(g), 128, 0, s>>>(g, vin, v, pf, p, a, acc);
    return (int)cudaGetLastError();
}

int phi_launch_buoyancy(const DGrid& g, const DVec& vin, const DVecOut& v, const DField& sf, const float* sarr,
                        const float b[3], float dt, cudaStream_t s)
{
    if (g.dim == 3) k_buoyancy<3><<<scalar_grid(g), 128, 0, s>>>(g, vin, v, sf, sarr, b[0], b[1], b[2], dt);
    else            k_buoyancy<2><<<scalar_grid(g), 128, 0, s>>>(g, vin, v, sf, sarr, b[0], b[1], 0.f, dt);
    return (int)cudaGetLastError();
}

int phi_launch_mul_faces(const DGrid& g, const DVec& vin, const DVecOut& v, const float* const mask[3], cudaStream_t s)
{
    if (g.dim == 3) k_mul_faces<3><<<scalar_grid(g), 128, 0, s>>>(g, vin, v, mask[0], mask[1], mask[2]);
    else            k_mul_faces<2><<<scalar_grid(g), 128, 0, s>>>(g, vin, v, mask[0], mask[1], nullptr);
    return (int)cudaGetLastError();
}

int phi_launch_axpy(const DGrid& g, const DField& cf, float a, const float* x, float* y, cudaStream_t s)
{
    if (g.dim == 3) k_axpy<3><<<scalar_grid(g), 128, 0, s>>>(g, cf, a, x, y);
    else            k_axpy<2><<<scalar_grid(g), 128, 0, s>>>(g, cf, a, x, y);
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// max |v_c| per component over the stored faces (owned planes only).  The semi-Lagrangian back-trace reaches
// ceil(max|v_z| dt / dz) + 1 planes into the neighbouring slab (phi/physics/advect.py:20-24, 156-179: the reference's
// lookup is unbounded), so the z-slab driver sizes its halo exchange from this number before every step (SURVEY.md 8e).
// Non-negative floats order like their bit patterns -> atomicMax on unsigned.
// ---------------------------------------------------------------------------------------------------------
template <int DIM>
__global__ void __launch_bounds__(256)
k_absmax(DGrid g, DVec v, unsigned* __restrict__ out)
{
    __shared__ float red[8];
    const int nx4 = g.fext[0] / 4;
#pragma unroll
    for (int c = 0; c < DIM; ++c) {
        const DField& f = v.f[c];
        const int ny = f.hi[1] - f.lo[1] + 1, nz = DIM == 3 ? f.hi[2] - f.lo[2] + 1 : 1;
        const long long total = (long long)g.batch * nz * ny * nx4;
        float m = 0.f;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
            const int x4 = (int)(i % nx4); long long r = i / nx4;
            const int y = (int)(r % ny) + f.lo[1]; r /= ny;
            const int z = DIM == 3 ? (int)(r % nz) + f.lo[2] : 0; const int b = (int)(r / nz);
            const float4 q = *reinterpret_cast<const float4*>(v.p[c] + (long long)b * f.sb + (long long)z * f.sz + (long long)y * f.sy + 4 * x4);
            const int x0 = 4 * x4;
            if (x0 + 0 >= f.lo[0] && x0 + 0 <= f.hi[0]) m = fmaxf(m, fabsf(q.x));
            if (x0 + 1 >= f.lo[0] && x0 + 1 <= f.hi[0]) m = fmaxf(m, fabsf(q.y));
            if (x0 + 2 >= f.lo[0] && x0 + 2 <= f.hi[0]) m = fmaxf(m, fabsf(q.z));
            if (x0 + 3 >= f.lo[0] && x0 + 3 <= f.hi[0]) m = fmaxf(m, fabsf(q.w));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, red[w]);
            if (!(m == m)) m = __int_as_float(0x7f800000);          // NaN -> +inf: "halo cannot be bounded"
            atomicMax(out + c, __float_as_uint(m));
        }
        __syncthreads();
    }
}

int phi_launch_absmax(const DGrid& g, const DVec& v, float* out, cudaStream_t s)
{
    cudaError_t e = cudaMemsetAsync(out, 0, 3 * sizeof(float), s);
    if (e != cudaSuccess) return (int)e;
    const int sms = phi_sm_count();
    if (g.dim == 3) k_absmax<3><<<sms * 8, 256, 0, s>>>(g, v, reinterpret_cast<unsigned*>(out));
    else            k_absmax<2><<<sms * 8, 256, 0, s>>>(g, v, reinterpret_cast<unsigned*>(out));
    return (int)cudaGetLastError();
}
