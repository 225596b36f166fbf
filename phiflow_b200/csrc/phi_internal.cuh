// Internal device-side definitions shared by all kernels of libphicuda.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/phicuda.h"

#define PHI_WARPS_PER_CTA 8
#define PHI_TILE_X 128           // cells per warp along x (32 lanes x float4)

// ---------------------------------------------------------------------------------------------------------
// Device views of the C-ABI structs
// ---------------------------------------------------------------------------------------------------------
struct DGrid {
    int dim, batch;
    int n[3];
    int cext[3], fext[3];          // allocated extents of centred arrays / staggered components
    int halo;                      // z-slab halo planes on each side of the owned range (0 on one GPU)
    float dx[3], inv_dx[3], inv_dx2[3];
};

// One scalar array: valid index range per axis + what lies outside it.
//   centred array:           [0, n-1] on every axis
//   staggered component c:   along c the stored faces [1-lo_stored, n-1+hi_stored]  (SURVEY.md Appendix A/B)
struct DField {
    int lo[3], hi[3];
    unsigned char klo[3], khi[3];
    float clo[3], chi[3];
    long long sy, sz, sb;          // strides (elements) of y, z, batch of this array
    int halo;                      // planes readable beyond [lo, hi] on the last axis (PHI_BC_HALO)
};

struct DVec {                      // a staggered vector field
    DField f[3];
    const float* p[3];
};
struct DVecOut {
    float* p[3];
};

// ---------------------------------------------------------------------------------------------------------
// Boundary resolution: maps an arbitrary index onto the stored range or yields the constant outside value.
// PERIODIC: index % n (extrapolation.py:668-669); ZERO_GRADIENT: clamp (:160-176); constant c: c (ring of c, _ops.py:912-918)
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool phi_resolve(int& i, const DField& f, int a, float& cval)
{
    const int lo = f.lo[a], hi = f.hi[a];
    if (i < lo) {
        const int k = f.klo[a];
        if (k == PHI_BC_HALO) { i = max(i, lo - f.halo); return true; }
        if (k == PHI_BC_PERIODIC) { const int per = hi - lo + 1; int r = (i - lo) % per; if (r < 0) r += per; i = lo + r; return true; }
        if (k == PHI_BC_ZERO_GRADIENT) { i = lo; return true; }
        cval = f.clo[a]; return false;
    }
    if (i > hi) {
        const int k = f.khi[a];
        if (k == PHI_BC_HALO) { i = min(i, hi + f.halo); return true; }
        if (k == PHI_BC_PERIODIC) { const int per = hi - lo + 1; i = lo + (i - lo) % per; return true; }
        if (k == PHI_BC_ZERO_GRADIENT) { i = hi; return true; }
        cval = f.chi[a]; return false;
    }
    return true;
}

template <int DIM>
__device__ __forceinline__ float phi_fetch(const float* __restrict__ a, const DGrid& g, const DField& f, int b, int x, int y, int z)
{
    // Outside in more than one axis: the reference pads axis by axis (math.pad, _ops.py:791-838), so a corner ghost cell holds what
    // the axis padded LAST put there - resolve the last axis first.  (Only visible when two axes carry different constants.)
    float c = 0.f;
    if (DIM == 3) { if (!phi_resolve(z, f, 2, c)) return c; } else z = 0;
    if (!phi_resolve(y, f, 1, c)) return c;
    if (!phi_resolve(x, f, 0, c)) return c;
    return __ldg(a + (long long)b * f.sb + (long long)z * f.sz + (long long)y * f.sy + x);
}

// value of the product s * k at (x, y, z): s * k on stored cells and across periodic / zero-gradient sides, but a constant side
// keeps its own value c, unscaled - multiplying a field by a constant leaves its boundary unchanged (phi/field/_field.py:809),
// so resample(s * (0, 0.1), to=v) averages c, not c * 0.1, into the faces next to a constant side of s
template <int DIM>
__device__ __forceinline__ float phi_fetch_scaled(const float* __restrict__ a, const DGrid& g, const DField& f, int b, int x, int y, int z, float k)
{
    float c = 0.f;
    if (DIM == 3) { if (!phi_resolve(z, f, 2, c)) return c; } else z = 0;
    if (!phi_resolve(y, f, 1, c)) return c;
    if (!phi_resolve(x, f, 0, c)) return c;
    return __ldg(a + (long long)b * f.sb + (long long)z * f.sz + (long long)y * f.sy + x) * k;
}

// a / b with a precomputed correctly rounded reciprocal inv_b = RN(1 / b) (DGrid.inv_dx, computed on the host): Markstein's
// correction q = RN(a * inv_b); r = a - q * b (exact in the FMA); q' = RN(q + r * inv_b) gives the correctly rounded quotient -
// the value the reference's `/ dx` produces (spatial_gradient, PhiML/phiml/math/_nd.py:813-815) - in 3 instructions instead of
// the ~35 of the IEEE division subroutine (ncu: the divisions were 75 % of the instructions of the stencil kernels).
// Exceptions (no overflow / denormal handling, significand of b all ones) do not occur for cell sizes.
__device__ __forceinline__ float phi_div(float a, float b, float inv_b)
{
    const float q = a * inv_b;
    const float r = fmaf(-q, b, a);
    return fmaf(r, inv_b, q);
}

__device__ __forceinline__ float4 f4_splat(float c) { return make_float4(c, c, c, c); }
__device__ __forceinline__ float f4_get(const float4& v, int j) { return j == 0 ? v.x : (j == 1 ? v.y : (j == 2 ? v.z : v.w)); }
__device__ __forceinline__ void f4_set(float4& v, int j, float s) { if (j == 0) v.x = s; else if (j == 1) v.y = s; else if (j == 2) v.z = s; else v.w = s; }

// ---------------------------------------------------------------------------------------------------------
// Reductions
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---------------------------------------------------------------------------------------------------------
// Marching 5/7-point stencil.
//
// A warp owns a 128-cell x-tile of one grid line and marches along the last spatial axis (z in 3-D, y in 2-D)
// keeping the three planes it needs in registers; in 3-D the eight warps of a CTA own eight consecutive y lines so
// that the y +/- 1 rows come out of L1.  x neighbours are exchanged with warp shuffles.  `Src` yields the value of
// the differenced array (a plain load for laplace / CG phase B, r + beta*d for CG phase A), `Epi` consumes
// (cell value, stencil value) for four cells at a time.
//
//   q = sum_axis (left + right - 2*centre) * inv_dx2[axis]          (PhiML/phiml/math/_nd.py:855-856)
// ---------------------------------------------------------------------------------------------------------
template <int DIM>
struct RowRef {            // a resolved grid line: either memory (off >= 0) or a constant
    long long off;         // element offset of x = 0 of the line, -1 if constant
    float cval;
};

template <int DIM>
__device__ __forceinline__ RowRef<DIM> phi_row(const DGrid& g, const DField& f, int b, int y, int z)
{
    RowRef<DIM> r; r.cval = 0.f; r.off = -1;
    if (DIM == 3) { if (!phi_resolve(z, f, 2, r.cval)) return r; } else z = 0;
    if (!phi_resolve(y, f, 1, r.cval)) return r;
    r.off = (long long)b * f.sb + (long long)z * f.sz + (long long)y * f.sy;
    return r;
}

// value of the ghost cells at x = -1 / x = n for a resolved line
template <int DIM, class Src>
__device__ __forceinline__ float phi_ghost_x(const Src& src, const DField& f, const RowRef<DIM>& row, bool upper)
{
    if (row.off < 0) return row.cval;
    const int k = upper ? f.khi[0] : f.klo[0];
    if (k == PHI_BC_PERIODIC) return src.load1(row.off + (upper ? f.lo[0] : f.hi[0]));
    if (k == PHI_BC_ZERO_GRADIENT) return src.load1(row.off + (upper ? f.hi[0] : f.lo[0]));
    return upper ? f.chi[0] : f.clo[0];
}

template <int DIM, class Src>
__device__ __forceinline__ float4 phi_load_row4(const Src& src, const RowRef<DIM>& row, int x0, bool active)
{
    if (!active) return f4_splat(0.f);
    if (row.off < 0) return f4_splat(row.cval);
    return src.load4(row.off + x0);
}

template <int DIM, class Src, class Epi>
__device__ __forceinline__ void phi_march(const DGrid& g, const DField& f, const Src& src, Epi& epi,
                                          int b, int xt0, int t, int m0, int m1)
{
    const int lane = threadIdx.x & 31;
    const int x0 = xt0 + lane * 4;
    const int nx = g.n[0];
    const bool active = x0 < nx;
    const int nvalid = active ? min(4, nx - x0) : 0;
    const float ix2 = g.inv_dx2[0], iy2 = g.inv_dx2[1], iz2 = g.inv_dx2[2];

    auto rowAt = [&](int tt, int mm) { return DIM == 3 ? phi_row<DIM>(g, f, b, tt, mm) : phi_row<DIM>(g, f, b, mm, 0); };

    float4 vm = phi_load_row4<DIM>(src, rowAt(t, m0 - 1), x0, active);
    RowRef<DIM> rc = rowAt(t, m0);
    float4 vc = phi_load_row4<DIM>(src, rc, x0, active);
    for (int m = m0; m < m1; ++m) {
        const float4 vp = phi_load_row4<DIM>(src, rowAt(t, m + 1), x0, active);
        float4 tl, th;
        if (DIM == 3) {
            tl = phi_load_row4<DIM>(src, rowAt(t - 1, m), x0, active);
            th = phi_load_row4<DIM>(src, rowAt(t + 1, m), x0, active);
        }
        // x neighbours
        float left = __shfl_up_sync(0xffffffffu, vc.w, 1);
        float right = __shfl_down_sync(0xffffffffu, vc.x, 1);
        if (active) {
            if (x0 == 0) left = phi_ghost_x<DIM>(src, f, rc, false);
            else if (lane == 0) left = src.load1(rc.off + x0 - 1);
            if (x0 + 4 >= nx) right = phi_ghost_x<DIM>(src, f, rc, true);
            else if (lane == 31) right = src.load1(rc.off + x0 + 4);
        }
        float4 xl = make_float4(left, vc.x, vc.y, vc.z);
        float4 xr = make_float4(vc.y, vc.z, vc.w, right);
        if (nvalid > 0 && nvalid < 4) f4_set(xr, nvalid - 1, right);      // row ends inside this float4
        float4 q;
        q.x = (xl.x + xr.x - 2.f * vc.x) * ix2;
        q.y = (xl.y + xr.y - 2.f * vc.y) * ix2;
        q.z = (xl.z + xr.z - 2.f * vc.z) * ix2;
        q.w = (xl.w + xr.w - 2.f * vc.w) * ix2;
        if (DIM == 3) {
            q.x += (tl.x + th.x - 2.f * vc.x) * iy2;
            q.y += (tl.y + th.y - 2.f * vc.y) * iy2;
            q.z += (tl.z + th.z - 2.f * vc.z) * iy2;
            q.w += (tl.w + th.w - 2.f * vc.w) * iy2;
        }
        const float im2 = (DIM == 3) ? iz2 : iy2;
        q.x += (vm.x + vp.x - 2.f * vc.x) * im2;
        q.y += (vm.y + vp.y - 2.f * vc.y) * im2;
        q.z += (vm.z + vp.z - 2.f * vc.z) * im2;
        q.w += (vm.w + vp.w - 2.f * vc.w) * im2;
        if (active) epi(rc.off + x0, vc, q, nvalid);
        vm = vc; vc = vp;
        rc = rowAt(t, m + 1);
    }
}

// N4: the same march with static obstacles (fluid.masked_laplace, phi/physics/fluid.py:197-202):
//   q_c = sum_faces min(acc_c, acc_nb) * (v_nb - v_c) / dx^2   for accessible cells (acc_c = 1),   q_c = v_c   inside obstacles.
// `acc` is the centred accessible mask; its ghost cells follow the value array's rows (periodic: wrapped, zero-gradient:
// clamped - the flux through such a face is zero anyway because the value ghost equals the centre), except that constant
// (Dirichlet) ghosts count as accessible (fluid._accessible_extrapolation: BOUNDARY -> ONE).
template <int DIM, class Src, class Epi>
__device__ __forceinline__ void phi_march_masked(const DGrid& g, const DField& f, const Src& src, const float* __restrict__ accp,
                                                 Epi& epi, int b, int xt0, int t, int m0, int m1)
{
    const int lane = threadIdx.x & 31;
    const int x0 = xt0 + lane * 4;
    const int nx = g.n[0];
    const bool active = x0 < nx;
    const int nvalid = active ? min(4, nx - x0) : 0;
    const float ix2 = g.inv_dx2[0], iy2 = g.inv_dx2[1], iz2 = g.inv_dx2[2];
    const float im2 = (DIM == 3) ? iz2 : iy2;
    struct SrcAcc {
        const float* a;
        __device__ __forceinline__ float4 load4(long long off) const { return *reinterpret_cast<const float4*>(a + off); }
        __device__ __forceinline__ float load1(long long off) const { return a[off]; }
    } sa{accp};
    DField fa = f;                                   // same rows, but constant ghosts are accessible (1)
    fa.clo[0] = fa.chi[0] = 1.f;
    auto rowAt = [&](int tt, int mm) { return DIM == 3 ? phi_row<DIM>(g, f, b, tt, mm) : phi_row<DIM>(g, f, b, mm, 0); };
    auto accRow = [&](RowRef<DIM> r) { r.cval = 1.f; return phi_load_row4<DIM>(sa, r, x0, active); };
    auto term = [](float vn, float vc, float an, float ac) { return fminf(an, ac) * (vn - vc); };

    RowRef<DIM> rm = rowAt(t, m0 - 1);
    float4 vm = phi_load_row4<DIM>(src, rm, x0, active), am = accRow(rm);
    RowRef<DIM> rc = rowAt(t, m0);
    float4 vc = phi_load_row4<DIM>(src, rc, x0, active), ac = accRow(rc);
    for (int m = m0; m < m1; ++m) {
        const RowRef<DIM> rp = rowAt(t, m + 1);
        const float4 vp = phi_load_row4<DIM>(src, rp, x0, active), ap = accRow(rp);
        float4 tl, th, al, ah;
        if (DIM == 3) {
            const RowRef<DIM> rl = rowAt(t - 1, m), rh = rowAt(t + 1, m);
            tl = phi_load_row4<DIM>(src, rl, x0, active); al = accRow(rl);
            th = phi_load_row4<DIM>(src, rh, x0, active); ah = accRow(rh);
        }
        float left = __shfl_up_sync(0xffffffffu, vc.w, 1), aleft = __shfl_up_sync(0xffffffffu, ac.w, 1);
        float right = __shfl_down_sync(0xffffffffu, vc.x, 1), aright = __shfl_down_sync(0xffffffffu, ac.x, 1);
        if (active) {
            if (x0 == 0) { left = phi_ghost_x<DIM>(src, f, rc, false); aleft = phi_ghost_x<DIM>(sa, fa, rc, false); }
            else if (lane == 0) { left = src.load1(rc.off + x0 - 1); aleft = sa.load1(rc.off + x0 - 1); }
            if (x0 + 4 >= nx) { right = phi_ghost_x<DIM>(src, f, rc, true); aright = phi_ghost_x<DIM>(sa, fa, rc, true); }
            else if (lane == 31) { right = src.load1(rc.off + x0 + 4); aright = sa.load1(rc.off + x0 + 4); }
        }
        float4 xl = make_float4(left, vc.x, vc.y, vc.z), axl = make_float4(aleft, ac.x, ac.y, ac.z);
        float4 xr = make_float4(vc.y, vc.z, vc.w, right), axr = make_float4(ac.y, ac.z, ac.w, aright);
        if (nvalid > 0 && nvalid < 4) { f4_set(xr, nvalid - 1, right); f4_set(axr, nvalid - 1, aright); }
        float4 q;
        q.x = (term(xl.x, vc.x, axl.x, ac.x) + term(xr.x, vc.x, axr.x, ac.x)) * ix2 + (term(vm.x, vc.x, am.x, ac.x) + term(vp.x, vc.x, ap.x, ac.x)) * im2;
        q.y = (term(xl.y, vc.y, axl.y, ac.y) + term(xr.y, vc.y, axr.y, ac.y)) * ix2 + (term(vm.y, vc.y, am.y, ac.y) + term(vp.y, vc.y, ap.y, ac.y)) * im2;
        q.z = (term(xl.z, vc.z, axl.z, ac.z) + term(xr.z, vc.z, axr.z, ac.z)) * ix2 + (term(vm.z, vc.z, am.z, ac.z) + term(vp.z, vc.z, ap.z, ac.z)) * im2;
        q.w = (term(xl.w, vc.w, axl.w, ac.w) + term(xr.w, vc.w, axr.w, ac.w)) * ix2 + (term(vm.w, vc.w, am.w, ac.w) + term(vp.w, vc.w, ap.w, ac.w)) * im2;
        if (DIM == 3) {
            q.x += (term(tl.x, vc.x, al.x, ac.x) + term(th.x, vc.x, ah.x, ac.x)) * iy2;
            q.y += (term(tl.y, vc.y, al.y, ac.y) + term(th.y, vc.y, ah.y, ac.y)) * iy2;
            q.z += (term(tl.z, vc.z, al.z, ac.z) + term(th.z, vc.z, ah.z, ac.z)) * iy2;
            q.w += (term(tl.w, vc.w, al.w, ac.w) + term(th.w, vc.w, ah.w, ac.w)) * iy2;
        }
        if (ac.x == 0.f) q.x = vc.x;
        if (ac.y == 0.f) q.y = vc.y;
        if (ac.z == 0.f) q.z = vc.z;
        if (ac.w == 0.f) q.w = vc.w;
        if (active) epi(rc.off + x0, vc, q, nvalid);
        vm = vc; vc = vp; am = ac; ac = ap;
        rc = rp;
    }
}

// Plain array source
struct SrcArray {
    const float* a;
    __device__ __forceinline__ float4 load4(long long off) const { return *reinterpret_cast<const float4*>(a + off); }
    __device__ __forceinline__ float load1(long long off) const { return a[off]; }
};

// ---------------------------------------------------------------------------------------------------------
// Decomposition of a grid into CTA units for the marching kernels
//   3-D: unit = (b, z-chunk, y-tile of 8 lines, x-tile);  warp w of the CTA takes line y = 8*ytile + w
//   2-D: unit = (b, group of 8 (y-chunk, x-tile) pairs);   warp w takes pair 8*group + w
// Units are numbered x-tile fastest so that CTAs running concurrently work on neighbouring data (L2 halo reuse).
// ---------------------------------------------------------------------------------------------------------
struct UnitMap {
    int nxt;          // x tiles
    int nyt;          // 3-D: y tiles (8 lines);  2-D: unused (1)
    int nmc;          // number of march chunks
    int mc;           // cells per march chunk
    int wu_per_batch; // 2-D: warp units per batch entry (nxt * nmc)
    int units_per_batch;
    int total_units;
};

struct WarpUnit {
    int b, xt0, t, m0, m1;
    bool valid;
};

template <int DIM>
__device__ __forceinline__ WarpUnit phi_warp_unit(const DGrid& g, const UnitMap& um, int unit, int warp)
{
    WarpUnit w;
    w.b = unit / um.units_per_batch;
    int u = unit - w.b * um.units_per_batch;
    const int nm = g.n[DIM - 1];
    if (DIM == 3) {
        const int xt = u % um.nxt; u /= um.nxt;
        const int yt = u % um.nyt; const int zc = u / um.nyt;
        w.xt0 = xt * PHI_TILE_X;
        w.t = yt * PHI_WARPS_PER_CTA + warp;
        w.m0 = zc * um.mc; w.m1 = min(nm, w.m0 + um.mc);
        w.valid = w.t < g.n[1];
    } else {
        const int wu = u * PHI_WARPS_PER_CTA + warp;
        w.valid = wu < um.wu_per_batch;
        const int xt = wu % um.nxt; const int yc = wu / um.nxt;
        w.xt0 = xt * PHI_TILE_X;
        w.t = 0;
        w.m0 = yc * um.mc; w.m1 = min(nm, w.m0 + um.mc);
    }
    return w;
}

// Host helpers (api.cu)
int phi_make_dgrid(const PhiGrid* g, DGrid* out);
int phi_make_centered(const PhiGrid* g, const PhiBC* bc, DField* out);
int phi_make_component(const PhiGrid* g, const PhiBC* bc, int c, DField* out);
int phi_pressure_bc(const PhiVBC* vbc, int dim, PhiBC* out);
UnitMap phi_make_unit_map(const DGrid& g, int target_units);
int phi_sm_count();                      // SMs of the current device
void phi_set_error(const char* fmt, ...);
void phi_note_launch(const PhiLaunchInfo& info);
void phi_note_cg_passes(int passes);       // sweeps per iteration of the last CG launch (phicuda_last_cg_passes)
void phi_note_cg_operator(int op);         // PHI_CG_OP_* of the last CG launch (phicuda_last_cg_operator)
