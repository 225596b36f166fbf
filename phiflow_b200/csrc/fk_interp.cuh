// Boundary-aware n-linear interpolation in three tiers (all neighbours stored / neighbours across periodic or zero-gradient sides /
// constant ghosts), shared by the semi-Lagrangian advection (fused_kernels.cu) and the point advection (points_kernels.cu).
//
// EXACT = false (advection): the weighted sum runs sequentially over the 2^d neighbours and nvcc may contract it into FMAs.
// EXACT = true (points): every operation is an explicitly rounded intrinsic, in the order of the NumPy fallback of math.grid_sample
// (PhiML/phiml/math/_ops.py:1010-1014): weight = prod over x, y, z of frac or fl(1 - frac), product = fl(value * weight), summed
// sequentially over the corners (0,0), (0,1), (1,0), (1,1) in 2-D and pairwise ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) in
// 3-D, which is how NumPy sums them (tests/golden/phiml_points.npz).
#pragma once
#include "phi_internal.cuh"

struct FkLookup { int i[3]; float t[3]; };

__device__ __forceinline__ void fk_lookup_axis(FkLookup& L, int a, int idx, float v, float dt, float dxa, float inv_dxa)
{
    const float delta = phi_div(-dt * v, dxa, inv_dxa);   // displacement in cells (advect.py:20-24, _resample.py:257-258)
    const float fl = floorf(delta);
    L.i[a] = idx + (int)fl;
    L.t[a] = delta - fl;
}

// the 2^d neighbours are all stored values (planes readable in the slab halo count as stored)
template <int DIM>
__device__ __forceinline__ bool fk_inside(const DField& f, const FkLookup& L)
{
    bool inside = L.i[0] >= f.lo[0] && L.i[0] + 1 <= f.hi[0] && L.i[1] >= f.lo[1] && L.i[1] + 1 <= f.hi[1];
    if (DIM == 3) {
        const int zlo = f.lo[2] - (f.klo[2] == PHI_BC_HALO ? f.halo : 0), zhi = f.hi[2] + (f.khi[2] == PHI_BC_HALO ? f.halo : 0);
        inside = inside && L.i[2] >= zlo && L.i[2] + 1 <= zhi;
    }
    return inside;
}

// EXACT weighted sum; n{x}{y} on the plane z0, m{x}{y} on z1
template <int DIM>
__device__ __forceinline__ float fk_sum_exact(float n00, float n01, float n10, float n11, float m00, float m01, float m10, float m11,
                                              float tx, float ty, float tz)
{
    const float ux = __fsub_rn(1.f, tx), uy = __fsub_rn(1.f, ty);
    const float w00 = __fmul_rn(ux, uy), w01 = __fmul_rn(ux, ty), w10 = __fmul_rn(tx, uy), w11 = __fmul_rn(tx, ty);
    if (DIM == 2)
        return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(n00, w00), __fmul_rn(n01, w01)), __fmul_rn(n10, w10)), __fmul_rn(n11, w11));
    const float uz = __fsub_rn(1.f, tz);
    const float r0 = __fmul_rn(n00, __fmul_rn(w00, uz)), r1 = __fmul_rn(m00, __fmul_rn(w00, tz));
    const float r2 = __fmul_rn(n01, __fmul_rn(w01, uz)), r3 = __fmul_rn(m01, __fmul_rn(w01, tz));
    const float r4 = __fmul_rn(n10, __fmul_rn(w10, uz)), r5 = __fmul_rn(m10, __fmul_rn(w10, tz));
    const float r6 = __fmul_rn(n11, __fmul_rn(w11, uz)), r7 = __fmul_rn(m11, __fmul_rn(w11, tz));
    return __fadd_rn(__fadd_rn(__fadd_rn(r0, r1), __fadd_rn(r2, r3)), __fadd_rn(__fadd_rn(r4, r5), __fadd_rn(r6, r7)));
}

// n-linear interpolation, all neighbours stored: weights = products of frac / (1 - frac), weighted sum over the 2^d
// neighbours in the order of the scalar kernel (PhiML/phiml/math/_ops.py:1010-1014).  32-bit element offsets.
template <int DIM, bool EXACT = false>
__device__ __forceinline__ float fk_interp_inside(const float* __restrict__ a, const DField& f, int b, const FkLookup& L)
{
    const int sy = (int)f.sy, sz = (int)f.sz;
    const float* p = a + (long long)b * f.sb + ((DIM == 3 ? L.i[2] * sz : 0) + L.i[1] * sy + L.i[0]);
    const float tx = L.t[0], ty = L.t[1], tz = L.t[2];
    const float n00 = __ldg(p), n10 = __ldg(p + 1), n01 = __ldg(p + sy), n11 = __ldg(p + sy + 1);
    float acc = 0.f;
    if (DIM == 3) {
        const float m00 = __ldg(p + sz), m10 = __ldg(p + sz + 1), m01 = __ldg(p + sz + sy), m11 = __ldg(p + sz + sy + 1);
        if (EXACT) return fk_sum_exact<DIM>(n00, n01, n10, n11, m00, m01, m10, m11, tx, ty, tz);
        const float w00 = (1.f - tx) * (1.f - ty), w01 = (1.f - tx) * ty, w10 = tx * (1.f - ty), w11 = tx * ty;
        acc += n00 * (w00 * (1.f - tz)); acc += m00 * (w00 * tz);
        acc += n01 * (w01 * (1.f - tz)); acc += m01 * (w01 * tz);
        acc += n10 * (w10 * (1.f - tz)); acc += m10 * (w10 * tz);
        acc += n11 * (w11 * (1.f - tz)); acc += m11 * (w11 * tz);
    } else {
        if (EXACT) return fk_sum_exact<DIM>(n00, n01, n10, n11, 0.f, 0.f, 0.f, 0.f, tx, ty, tz);
        acc += n00 * ((1.f - tx) * (1.f - ty)); acc += n01 * ((1.f - tx) * ty);
        acc += n10 * (tx * (1.f - ty)); acc += n11 * (tx * ty);
    }
    return acc;
}

// ONE out-of-line copy of the boundary-aware interpolation (neighbours outside the array follow the field's boundary)
template <int DIM, bool EXACT = false>
__device__ __noinline__ float fk_interp_slow(const float* __restrict__ a, const DGrid* gp, const DField* fp, int b,
                                             int i0, int i1, int i2, float tx, float ty, float tz)
{
    const DGrid& g = *gp; const DField& f = *fp;
    if (EXACT) {
        auto v = [&](int cx, int cy, int cz) { return phi_fetch<DIM>(a, g, f, b, i0 + cx, i1 + cy, i2 + cz); };
        if (DIM == 2) return fk_sum_exact<DIM>(v(0, 0, 0), v(0, 1, 0), v(1, 0, 0), v(1, 1, 0), 0.f, 0.f, 0.f, 0.f, tx, ty, tz);
        return fk_sum_exact<DIM>(v(0, 0, 0), v(0, 1, 0), v(1, 0, 0), v(1, 1, 0), v(0, 0, 1), v(0, 1, 1), v(1, 0, 1), v(1, 1, 1), tx, ty, tz);
    }
    float acc = 0.f;
#pragma unroll 1
    for (int c = 0; c < (DIM == 3 ? 8 : 4); ++c) {
        const int cx = DIM == 3 ? (c >> 2) : (c >> 1), cy = DIM == 3 ? ((c >> 1) & 1) : (c & 1), cz = DIM == 3 ? (c & 1) : 0;
        float w = (cx ? tx : 1.f - tx) * (cy ? ty : 1.f - ty);
        if (DIM == 3) w = w * (cz ? tz : 1.f - tz);
        acc += phi_fetch<DIM>(a, g, f, b, i0 + cx, i1 + cy, i2 + cz) * w;
    }
    return acc;
}

// neighbour pair (i, i + 1) of one axis mapped onto stored indices: PERIODIC wraps, ZERO_GRADIENT clamps, slab halo planes are
// stored values; false when a neighbour is a constant ghost (-> fk_interp_slow)
__device__ __forceinline__ bool fk_pair(const DField& f, int a, int i, int& i0, int& i1)
{
    float c;
    i0 = i; i1 = i + 1;
    return phi_resolve(i0, f, a, c) && phi_resolve(i1, f, a, c);
}

// middle tier: some neighbour lies across a periodic / zero-gradient / slab boundary - no constants involved.  Same weights
// and summation order as fk_interp_inside.
template <int DIM, bool EXACT = false>
__device__ __noinline__ float fk_interp_wrapped(const float* __restrict__ a, const DGrid* gp, const DField* fp, int b,
                                                int i0, int i1, int i2, float tx, float ty, float tz)
{
    const DField& f = *fp;
    int x0, x1, y0, y1, z0 = 0, z1 = 0;
    bool ok = fk_pair(f, 0, i0, x0, x1) && fk_pair(f, 1, i1, y0, y1);
    if (DIM == 3) ok = ok && fk_pair(f, 2, i2, z0, z1);
    if (!ok) return fk_interp_slow<DIM, EXACT>(a, gp, fp, b, i0, i1, i2, tx, ty, tz);
    const int sy = (int)f.sy, sz = (int)f.sz;
    const float* p = a + (long long)b * f.sb;
    const int r00 = z0 * sz + y0 * sy, r01 = z0 * sz + y1 * sy;
    const float n00 = __ldg(p + r00 + x0), n10 = __ldg(p + r00 + x1), n01 = __ldg(p + r01 + x0), n11 = __ldg(p + r01 + x1);
    float acc = 0.f;
    if (DIM == 3) {
        const int r10 = z1 * sz + y0 * sy, r11 = z1 * sz + y1 * sy;
        const float m00 = __ldg(p + r10 + x0), m10 = __ldg(p + r10 + x1), m01 = __ldg(p + r11 + x0), m11 = __ldg(p + r11 + x1);
        if (EXACT) return fk_sum_exact<DIM>(n00, n01, n10, n11, m00, m01, m10, m11, tx, ty, tz);
        const float w00 = (1.f - tx) * (1.f - ty), w01 = (1.f - tx) * ty, w10 = tx * (1.f - ty), w11 = tx * ty;
        acc += n00 * (w00 * (1.f - tz)); acc += m00 * (w00 * tz);
        acc += n01 * (w01 * (1.f - tz)); acc += m01 * (w01 * tz);
        acc += n10 * (w10 * (1.f - tz)); acc += m10 * (w10 * tz);
        acc += n11 * (w11 * (1.f - tz)); acc += m11 * (w11 * tz);
    } else {
        if (EXACT) return fk_sum_exact<DIM>(n00, n01, n10, n11, 0.f, 0.f, 0.f, 0.f, tx, ty, tz);
        acc += n00 * ((1.f - tx) * (1.f - ty)); acc += n01 * ((1.f - tx) * ty);
        acc += n10 * (tx * (1.f - ty)); acc += n11 * (tx * ty);
    }
    return acc;
}

template <int DIM, bool EXACT = false>
__device__ __forceinline__ float fk_interp(const float* __restrict__ a, const DGrid& g, const DField& f, int b, const FkLookup& L)
{
    if (fk_inside<DIM>(f, L)) return fk_interp_inside<DIM, EXACT>(a, f, b, L);
    return fk_interp_wrapped<DIM, EXACT>(a, &g, &f, b, L.i[0], L.i[1], L.i[2], L.t[0], L.t[1], L.t[2]);
}
