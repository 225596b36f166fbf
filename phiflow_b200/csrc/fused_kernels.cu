// Vectorised projection stencils (A5 divergence, A6 gradient subtraction, with or without static obstacle masks) and the
// one-launch semi-Lagrangian advection (A9-A11) of the incompressible step, replacing the one-thread-per-sample kernels of
// round 1 (stencil_kernels.cu / advect_kernels.cu keep those as the arithmetic these kernels must reproduce).
//
// Design (SURVEY.md section 8d byte table; profiles/r2_ncu_summary.md has the measurements behind each choice):
//   * a warp owns one grid line (y, z) and walks a 128-cell x segment; which neighbouring lines a stencil reads, and whether
//     the boundary turns them into wrapped lines, clamped lines or constants, is resolved ONCE per warp (warp-uniform), not
//     per access.  x neighbours come from warp shuffles, only the two edge lanes of a segment load them.
//   * divergence / grad_sub: one float4 (4 cells) per thread, every operand a 16-byte load; the y/z neighbour lines are L1/L2
//     hits, DRAM traffic is the compulsory 16 / 28 B per cell (ncu: 15.9 / 27.6).  `/ dx` is the 3-instruction exact quotient
//     phi_div: the first version spent 75 % of its instructions in the IEEE division subroutine and was issue-bound.
//   * advection: lanes own consecutive x (coalesced gathers for smooth displacement fields).  The three staggered components
//     are advected in ONE launch: the 11 velocity lines a cell's three faces need (shift resampling,
//     phi/field/_resample.py:341-364) are loaded once and shared, x-shifted values are shuffles; buoyancy
//     (resample(s * b, to=v), _resample.py:272-276) and the smoke inflow are epilogues of the same kernels.
//     The first version inlined the boundary resolution at every access: 24 000 SASS instructions, 39 % of the stall samples
//     "no instruction" (i-cache misses), 26 % of the executed instructions branch bookkeeping.  Now every 32-cell chunk is
//     classified once (warp-uniform): chunks whose lines are all stored lines and whose x range is periodic or interior run
//     straight-line code with 32-bit offsets; everything else goes through ONE out-of-line copy of the boundary-aware
//     per-sample code (the scalar kernel's arithmetic).
// Arithmetic (operation order, 0.5/0.5 lerp order of sample_subgrid, weighted 2^d sum of _ops.py:1010-1014) is identical to
// the scalar kernels, which are pinned against the oracle; tests/test_gpu_vectorised.py compares the two families bit by bit.
#include "phi_internal.cuh"
#include "launch.cuh"

#define FK_WARPS 8
#define FK_THREADS (FK_WARPS * 32)

// A resolved line is an element offset relative to the array pointer (which addresses the first OWNED plane: offsets of slab
// halo planes are negative) or a constant ghost line, marked by this sentinel.
#define FK_CONST_LINE (-(1ll << 62))

// value at index x of a resolved line; x outside the stored range follows the boundary (same resolution order as phi_fetch:
// z, then y, then x - a constant ghost LINE wins over a constant x ghost)
__device__ __forceinline__ float fk_ldx(const float* __restrict__ a, const RowRef<3>& r, const DField& f, int x)
{
    if (r.off == FK_CONST_LINE) return r.cval;
    if (x < f.lo[0] || x > f.hi[0]) { float c; if (!phi_resolve(x, f, 0, c)) return c; }
    return __ldg(a + r.off + x);
}

template <int DIM>
__device__ __forceinline__ RowRef<3> fk_row(const DGrid& g, const DField& f, int b, int y, int z)
{
    RowRef<3> r; r.cval = 0.f; r.off = FK_CONST_LINE;
    if (DIM == 3) { if (!phi_resolve(z, f, 2, r.cval)) return r; } else z = 0;
    if (!phi_resolve(y, f, 1, r.cval)) return r;
    r.off = (long long)b * f.sb + (long long)z * f.sz + (long long)y * f.sy;
    return r;
}

// four consecutive values x0 .. x0+3 of a resolved line (x0 % 4 == 0).  Fast when all four are stored values.
__device__ __forceinline__ float4 fk_ld4(const float* __restrict__ a, const RowRef<3>& r, const DField& f, int x0)
{
    if (x0 >= f.lo[0] && x0 + 3 <= f.hi[0] && r.off != FK_CONST_LINE) return __ldg(reinterpret_cast<const float4*>(a + r.off + x0));
    return make_float4(fk_ldx(a, r, f, x0), fk_ldx(a, r, f, x0 + 1), fk_ldx(a, r, f, x0 + 2), fk_ldx(a, r, f, x0 + 3));
}

struct FkLine { int b, y, z, x0; bool ok; };

// warp -> (line, 128-cell segment); lane -> float4 group.  Lines are numbered over the ALLOCATED extent so that upper
// boundary faces are covered.
template <int DIM>
__device__ __forceinline__ FkLine fk_line4(const DGrid& g)
{
    FkLine L;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    L.x0 = (blockIdx.x * 32 + lane) * 4;
    L.y = blockIdx.y * FK_WARPS + warp;
    const int zb = blockIdx.z;
    if (DIM == 3) { L.z = zb % g.fext[2] - g.halo; L.b = zb / g.fext[2]; } else { L.z = 0; L.b = zb; }
    L.ok = L.y < g.fext[1];
    return L;
}

// ---------------------------------------------------------------------------------------------------------
// A5  divergence:  div = sum_d (v_d[i + e_d] - v_d[i]) / dx_d      16 B/cell (3-D), 12 (2-D)
// MASK (N4): div *= accessible, one more float4 per group (20 / 16 B/cell); the product of k_divergence with a mask
// ---------------------------------------------------------------------------------------------------------
template <int DIM, bool MASK>
__global__ void __launch_bounds__(FK_THREADS)
k_div_vec(const __grid_constant__ DGrid g, const __grid_constant__ DVec v, const __grid_constant__ DField cf, float* __restrict__ div,
          const float* __restrict__ accm)
{
    const FkLine L = fk_line4<DIM>(g);
    if (!L.ok || L.y >= g.n[1] || L.z < 0 || L.z >= g.n[2]) return;          // whole warp leaves together
    const int lane = threadIdx.x & 31;
    const int x0 = L.x0;
    const bool in_line = x0 < g.n[0];
    // lines whose y / z neighbours are all stored lines of every component need no boundary resolution (warp-uniform)
    const bool interior = L.y >= max(v.f[0].lo[1], v.f[1].lo[1]) && L.y + 1 <= min(v.f[0].hi[1], v.f[1].hi[1])
                          && (DIM == 2 || (L.y >= v.f[2].lo[1] && L.y <= v.f[2].hi[1]
                                           && L.z >= max(max(v.f[0].lo[2], v.f[1].lo[2]), v.f[2].lo[2])
                                           && L.z + 1 <= min(min(v.f[0].hi[2], v.f[1].hi[2]), v.f[2].hi[2])));
    RowRef<3> rx, ry0, ry1, rz0, rz1;
    if (interior) {
        const long long base = (long long)L.b * v.f[0].sb + (long long)L.z * v.f[0].sz + (long long)L.y * v.f[0].sy;
        rx.off = base; ry0.off = base; ry1.off = base + v.f[0].sy; rz0.off = base; rz1.off = base + v.f[0].sz;
        rx.cval = ry0.cval = ry1.cval = rz0.cval = rz1.cval = 0.f;
    } else {
        rx = fk_row<DIM>(g, v.f[0], L.b, L.y, L.z);
        ry0 = fk_row<DIM>(g, v.f[1], L.b, L.y, L.z); ry1 = fk_row<DIM>(g, v.f[1], L.b, L.y + 1, L.z);
        rz0 = rx; rz1 = rx;
        if (DIM == 3) { rz0 = fk_row<DIM>(g, v.f[2], L.b, L.y, L.z); rz1 = fk_row<DIM>(g, v.f[2], L.b, L.y, L.z + 1); }
    }
    float4 ax = f4_splat(0.f), ay0 = ax, ay1 = ax, az0 = ax, az1 = ax;
    if (in_line) {
        ax = fk_ld4(v.p[0], rx, v.f[0], x0);
        ay0 = fk_ld4(v.p[1], ry0, v.f[1], x0); ay1 = fk_ld4(v.p[1], ry1, v.f[1], x0);
        if (DIM == 3) { az0 = fk_ld4(v.p[2], rz0, v.f[2], x0); az1 = fk_ld4(v.p[2], rz1, v.f[2], x0); }
    }
    float nx = __shfl_down_sync(0xffffffffu, ax.x, 1);                      // v_x[x0 + 4]
    if (in_line && (lane == 31 || x0 + 4 >= g.n[0])) nx = fk_ldx(v.p[0], rx, v.f[0], x0 + 4);
    if (!in_line) return;
    const float dx = g.dx[0], dy = g.dx[1], dz = g.dx[2], ix = g.inv_dx[0], iy = g.inv_dx[1], iz = g.inv_dx[2];
    float4 o;
    o.x = phi_div(ax.y - ax.x, dx, ix) + phi_div(ay1.x - ay0.x, dy, iy);
    o.y = phi_div(ax.z - ax.y, dx, ix) + phi_div(ay1.y - ay0.y, dy, iy);
    o.z = phi_div(ax.w - ax.z, dx, ix) + phi_div(ay1.z - ay0.z, dy, iy);
    o.w = phi_div(nx - ax.w, dx, ix) + phi_div(ay1.w - ay0.w, dy, iy);
    if (DIM == 3) {
        o.x += phi_div(az1.x - az0.x, dz, iz); o.y += phi_div(az1.y - az0.y, dz, iz);
        o.z += phi_div(az1.z - az0.z, dz, iz); o.w += phi_div(az1.w - az0.w, dz, iz);
    }
    const long long coff = (long long)L.b * cf.sb + (long long)L.z * cf.sz + (long long)L.y * cf.sy + x0;
    if (MASK) {                                                             // cext[0] % 4 == 0: the float4 stays in the row
        const float4 m = __ldg(reinterpret_cast<const float4*>(accm + coff));
        o.x = o.x * m.x; o.y = o.y * m.y; o.z = o.z * m.z; o.w = o.w * m.w;
    }
    float* dst = div + coff;
    const int nvalid = g.n[0] - x0;
    if (nvalid >= 4) *reinterpret_cast<float4*>(dst) = o;
    else for (int j = 0; j < nvalid; ++j) dst[j] = f4_get(o, j);
}

int phi_launch_divergence_vec(const DGrid& g, const DVec& v, const DField& cf, float* div, const float* acc, cudaStream_t s)
{
    dim3 grid((g.fext[0] / 4 + 31) / 32, (g.fext[1] + FK_WARPS - 1) / FK_WARPS, g.fext[2] * g.batch);
    if (g.dim == 3) {
        if (acc) k_div_vec<3, true><<<grid, FK_THREADS, 0, s>>>(g, v, cf, div, acc);
        else     k_div_vec<3, false><<<grid, FK_THREADS, 0, s>>>(g, v, cf, div, nullptr);
    } else {
        if (acc) k_div_vec<2, true><<<grid, FK_THREADS, 0, s>>>(g, v, cf, div, acc);
        else     k_div_vec<2, false><<<grid, FK_THREADS, 0, s>>>(g, v, cf, div, nullptr);
    }
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// A6  v_d[f] = vin_d[f] - (p[upper(f)] - p[lower(f)]) / dx_d on the stored faces       28 B/cell (3-D), 20 (2-D)
// Out of place (vout may equal vin): the fused step writes the projected velocity straight back into the caller's arrays.
// MASK (N4): the gradient is scaled by hard_bcs = min(acc[upper cell], acc[lower cell]) as k_grad_sub does with a mask, the
// accessibility ghosts from af (fluid._accessible_extrapolation); the acc lines are resolved and loaded like the p lines.
// ---------------------------------------------------------------------------------------------------------
template <int DIM, bool MASK>
__global__ void __launch_bounds__(FK_THREADS)
k_gradsub_vec(const __grid_constant__ DGrid g, const __grid_constant__ DVec vin, const __grid_constant__ DVecOut vout,
              const __grid_constant__ DField pf, const float* __restrict__ p, const __grid_constant__ DField af, const float* __restrict__ accm)
{
    const FkLine L = fk_line4<DIM>(g);
    if (!L.ok || (DIM == 3 && (L.z < 0 || L.z >= g.fext[2] - 2 * g.halo))) return;
    const int lane = threadIdx.x & 31;
    const int x0 = L.x0;
    const bool in_line = x0 < g.fext[0];
    // p lines (y, z), (y - 1, z), (y, z - 1) are all stored lines: no boundary resolution (warp-uniform)
    const bool interior = L.y >= 1 && L.y <= pf.hi[1] && (DIM == 2 || (L.z >= 1 && L.z <= pf.hi[2]));
    RowRef<3> r0;
    if (interior) { r0.off = (long long)L.b * pf.sb + (long long)L.z * pf.sz + (long long)L.y * pf.sy; r0.cval = 0.f; }
    else r0 = fk_row<DIM>(g, pf, L.b, L.y, L.z);
    float4 pc = f4_splat(0.f);
    if (in_line) pc = fk_ld4(p, r0, pf, x0);
    float pl = __shfl_up_sync(0xffffffffu, pc.w, 1);                         // p[x0 - 1]
    if (in_line && (lane == 0 || x0 == 0)) pl = fk_ldx(p, r0, pf, x0 - 1);
    // MASK: the same for the accessibility (centred like p: an interior line has p's offset)
    RowRef<3> ra0 = r0;
    float4 ac = f4_splat(1.f);
    float al = 1.f;
    if (MASK) {
        if (!interior) ra0 = fk_row<DIM>(g, af, L.b, L.y, L.z);
        if (in_line) ac = fk_ld4(accm, ra0, af, x0);
        al = __shfl_up_sync(0xffffffffu, ac.w, 1);
        if (in_line && (lane == 0 || x0 == 0)) al = fk_ldx(accm, ra0, af, x0 - 1);
    }
    if (!in_line) return;
    const long long off = (long long)L.b * vin.f[0].sb + (long long)L.z * vin.f[0].sz + (long long)L.y * vin.f[0].sy + x0;
    const float dx = g.dx[0], dy = g.dx[1], dz = g.dx[2], ix = g.inv_dx[0], iy = g.inv_dx[1], iz = g.inv_dx[2];
    const bool yz_c = L.y < g.n[1] && (DIM == 2 || L.z < g.n[2]);            // line inside the cell range in y and z
    {   // x component: faces lo..hi along x, cells along y, z
        const DField& f = vin.f[0];
        if (yz_c && x0 <= f.hi[0] && x0 + 3 >= f.lo[0]) {
            float4 a = *reinterpret_cast<const float4*>(vin.p[0] + off);
            if (MASK) {     // separate multiply and subtract, as k_grad_sub rounds them
                a.x -= __fmul_rn(phi_div(pc.x - pl, dx, ix), fminf(ac.x, al)); a.y -= __fmul_rn(phi_div(pc.y - pc.x, dx, ix), fminf(ac.y, ac.x));
                a.z -= __fmul_rn(phi_div(pc.z - pc.y, dx, ix), fminf(ac.z, ac.y)); a.w -= __fmul_rn(phi_div(pc.w - pc.z, dx, ix), fminf(ac.w, ac.z));
            } else {
                a.x -= phi_div(pc.x - pl, dx, ix); a.y -= phi_div(pc.y - pc.x, dx, ix);
                a.z -= phi_div(pc.z - pc.y, dx, ix); a.w -= phi_div(pc.w - pc.z, dx, ix);
            }
            if (x0 >= f.lo[0] && x0 + 3 <= f.hi[0]) *reinterpret_cast<float4*>(vout.p[0] + off) = a;
            else for (int j = 0; j < 4; ++j) if (x0 + j >= f.lo[0] && x0 + j <= f.hi[0]) vout.p[0][off + j] = f4_get(a, j);
        }
    }
    const int nvx = g.n[0] - x0;                                            // cells of this group inside the line
    if (nvx <= 0) return;
    {   // y component
        const DField& f = vin.f[1];
        if (L.y >= f.lo[1] && L.y <= f.hi[1] && (DIM == 2 || L.z < g.n[2])) {
            RowRef<3> rm = r0;
            if (interior) rm.off = r0.off - pf.sy; else rm = fk_row<DIM>(g, pf, L.b, L.y - 1, L.z);
            const float4 pm = fk_ld4(p, rm, pf, x0);
            float4 a = *reinterpret_cast<const float4*>(vin.p[1] + off);
            if (MASK) {
                RowRef<3> ram = ra0;
                if (interior) ram.off = ra0.off - af.sy; else ram = fk_row<DIM>(g, af, L.b, L.y - 1, L.z);
                const float4 am = fk_ld4(accm, ram, af, x0);
                a.x -= __fmul_rn(phi_div(pc.x - pm.x, dy, iy), fminf(ac.x, am.x)); a.y -= __fmul_rn(phi_div(pc.y - pm.y, dy, iy), fminf(ac.y, am.y));
                a.z -= __fmul_rn(phi_div(pc.z - pm.z, dy, iy), fminf(ac.z, am.z)); a.w -= __fmul_rn(phi_div(pc.w - pm.w, dy, iy), fminf(ac.w, am.w));
            } else {
                a.x -= phi_div(pc.x - pm.x, dy, iy); a.y -= phi_div(pc.y - pm.y, dy, iy);
                a.z -= phi_div(pc.z - pm.z, dy, iy); a.w -= phi_div(pc.w - pm.w, dy, iy);
            }
            if (nvx >= 4) *reinterpret_cast<float4*>(vout.p[1] + off) = a;
            else for (int j = 0; j < nvx; ++j) vout.p[1][off + j] = f4_get(a, j);
        }
    }
    if (DIM == 3) {   // z component
        const DField& f = vin.f[2];
        if (L.z >= f.lo[2] && L.z <= f.hi[2] && L.y < g.n[1]) {
            RowRef<3> rm = r0;
            if (interior) rm.off = r0.off - pf.sz; else rm = fk_row<DIM>(g, pf, L.b, L.y, L.z - 1);
            const float4 pm = fk_ld4(p, rm, pf, x0);
            float4 a = *reinterpret_cast<const float4*>(vin.p[2] + off);
            if (MASK) {
                RowRef<3> ram = ra0;
                if (interior) ram.off = ra0.off - af.sz; else ram = fk_row<DIM>(g, af, L.b, L.y, L.z - 1);
                const float4 am = fk_ld4(accm, ram, af, x0);
                a.x -= __fmul_rn(phi_div(pc.x - pm.x, dz, iz), fminf(ac.x, am.x)); a.y -= __fmul_rn(phi_div(pc.y - pm.y, dz, iz), fminf(ac.y, am.y));
                a.z -= __fmul_rn(phi_div(pc.z - pm.z, dz, iz), fminf(ac.z, am.z)); a.w -= __fmul_rn(phi_div(pc.w - pm.w, dz, iz), fminf(ac.w, am.w));
            } else {
                a.x -= phi_div(pc.x - pm.x, dz, iz); a.y -= phi_div(pc.y - pm.y, dz, iz);
                a.z -= phi_div(pc.z - pm.z, dz, iz); a.w -= phi_div(pc.w - pm.w, dz, iz);
            }
            if (nvx >= 4) *reinterpret_cast<float4*>(vout.p[2] + off) = a;
            else for (int j = 0; j < nvx; ++j) vout.p[2][off + j] = f4_get(a, j);
        }
    }
}

int phi_launch_grad_sub_vec(const DGrid& g, const DVec& vin, const DVecOut& vout, const DField& pf, const float* p,
                            const DField* af, const float* acc, cudaStream_t s)
{
    dim3 grid((g.fext[0] / 4 + 31) / 32, (g.fext[1] + FK_WARPS - 1) / FK_WARPS, g.fext[2] * g.batch);
    const DField a = af ? *af : pf;
    if (g.dim == 3) {
        if (acc) k_gradsub_vec<3, true><<<grid, FK_THREADS, 0, s>>>(g, vin, vout, pf, p, a, acc);
        else     k_gradsub_vec<3, false><<<grid, FK_THREADS, 0, s>>>(g, vin, vout, pf, p, a, nullptr);
    } else {
        if (acc) k_gradsub_vec<2, true><<<grid, FK_THREADS, 0, s>>>(g, vin, vout, pf, p, a, acc);
        else     k_gradsub_vec<2, false><<<grid, FK_THREADS, 0, s>>>(g, vin, vout, pf, p, a, nullptr);
    }
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// A9-A11  semi-Lagrangian advection, lanes = consecutive x
// ---------------------------------------------------------------------------------------------------------
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

// n-linear interpolation, all neighbours stored: weights = products of frac / (1 - frac), weighted sum over the 2^d
// neighbours in the order of the scalar kernel (PhiML/phiml/math/_ops.py:1010-1014).  32-bit element offsets.
template <int DIM>
__device__ __forceinline__ float fk_interp_inside(const float* __restrict__ a, const DField& f, int b, const FkLookup& L)
{
    const int sy = (int)f.sy, sz = (int)f.sz;
    const float* p = a + (long long)b * f.sb + ((DIM == 3 ? L.i[2] * sz : 0) + L.i[1] * sy + L.i[0]);
    const float tx = L.t[0], ty = L.t[1], tz = L.t[2];
    const float n00 = __ldg(p), n10 = __ldg(p + 1), n01 = __ldg(p + sy), n11 = __ldg(p + sy + 1);
    float acc = 0.f;
    if (DIM == 3) {
        const float m00 = __ldg(p + sz), m10 = __ldg(p + sz + 1), m01 = __ldg(p + sz + sy), m11 = __ldg(p + sz + sy + 1);
        const float w00 = (1.f - tx) * (1.f - ty), w01 = (1.f - tx) * ty, w10 = tx * (1.f - ty), w11 = tx * ty;
        acc += n00 * (w00 * (1.f - tz)); acc += m00 * (w00 * tz);
        acc += n01 * (w01 * (1.f - tz)); acc += m01 * (w01 * tz);
        acc += n10 * (w10 * (1.f - tz)); acc += m10 * (w10 * tz);
        acc += n11 * (w11 * (1.f - tz)); acc += m11 * (w11 * tz);
    } else {
        acc += n00 * ((1.f - tx) * (1.f - ty)); acc += n01 * ((1.f - tx) * ty);
        acc += n10 * (tx * (1.f - ty)); acc += n11 * (tx * ty);
    }
    return acc;
}

// ONE out-of-line copy of the boundary-aware interpolation (neighbours outside the array follow the field's boundary)
template <int DIM>
__device__ __noinline__ float fk_interp_slow(const float* __restrict__ a, const DGrid* gp, const DField* fp, int b,
                                             int i0, int i1, int i2, float tx, float ty, float tz)
{
    const DGrid& g = *gp; const DField& f = *fp;
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
template <int DIM>
__device__ __noinline__ float fk_interp_wrapped(const float* __restrict__ a, const DGrid* gp, const DField* fp, int b,
                                                int i0, int i1, int i2, float tx, float ty, float tz)
{
    const DField& f = *fp;
    int x0, x1, y0, y1, z0 = 0, z1 = 0;
    bool ok = fk_pair(f, 0, i0, x0, x1) && fk_pair(f, 1, i1, y0, y1);
    if (DIM == 3) ok = ok && fk_pair(f, 2, i2, z0, z1);
    if (!ok) return fk_interp_slow<DIM>(a, gp, fp, b, i0, i1, i2, tx, ty, tz);
    const int sy = (int)f.sy, sz = (int)f.sz;
    const float* p = a + (long long)b * f.sb;
    const int r00 = z0 * sz + y0 * sy, r01 = z0 * sz + y1 * sy;
    const float n00 = __ldg(p + r00 + x0), n10 = __ldg(p + r00 + x1), n01 = __ldg(p + r01 + x0), n11 = __ldg(p + r01 + x1);
    float acc = 0.f;
    if (DIM == 3) {
        const int r10 = z1 * sz + y0 * sy, r11 = z1 * sz + y1 * sy;
        const float m00 = __ldg(p + r10 + x0), m10 = __ldg(p + r10 + x1), m01 = __ldg(p + r11 + x0), m11 = __ldg(p + r11 + x1);
        const float w00 = (1.f - tx) * (1.f - ty), w01 = (1.f - tx) * ty, w10 = tx * (1.f - ty), w11 = tx * ty;
        acc += n00 * (w00 * (1.f - tz)); acc += m00 * (w00 * tz);
        acc += n01 * (w01 * (1.f - tz)); acc += m01 * (w01 * tz);
        acc += n10 * (w10 * (1.f - tz)); acc += m10 * (w10 * tz);
        acc += n11 * (w11 * (1.f - tz)); acc += m11 * (w11 * tz);
    } else {
        acc += n00 * ((1.f - tx) * (1.f - ty)); acc += n01 * ((1.f - tx) * ty);
        acc += n10 * (tx * (1.f - ty)); acc += n11 * (tx * ty);
    }
    return acc;
}

template <int DIM>
__device__ __forceinline__ float fk_interp(const float* __restrict__ a, const DGrid& g, const DField& f, int b, const FkLookup& L)
{
    if (fk_inside<DIM>(f, L)) return fk_interp_inside<DIM>(a, f, b, L);
    return fk_interp_wrapped<DIM>(a, &g, &f, b, L.i[0], L.i[1], L.i[2], L.t[0], L.t[1], L.t[2]);
}

#define FK_XCHUNKS 4        // a warp walks 4 chunks of 32 cells of its line

struct FkAdvLine { int b, y, z, xs; bool ok; };

template <int DIM>
__device__ __forceinline__ FkAdvLine fk_adv_line(const DGrid& g)
{
    FkAdvLine L;
    L.xs = blockIdx.x * 32 * FK_XCHUNKS;
    L.y = blockIdx.y * FK_WARPS + (threadIdx.x >> 5);
    const int zb = blockIdx.z;
    if (DIM == 3) { L.z = zb % g.fext[2] - g.halo; L.b = zb / g.fext[2]; } else { L.z = 0; L.b = zb; }
    L.ok = L.y < g.fext[1] && (DIM == 2 || (L.z >= 0 && L.z < g.fext[2] - 2 * g.halo));
    return L;
}

__device__ __forceinline__ float fk_avg4(float f00, float f10, float f01, float f11, bool a_first)
{
    // shift resampling = sample_subgrid lerps the axes in spatial order (PhiML/phiml/math/_nd.py:973-1003):
    // f{da}{dt}: da in {0,1} along the component's own axis a, dt in {-1 -> 0, 0 -> 1} along the target face axis t
    if (a_first) { const float u0 = f10 * 0.5f + f00 * 0.5f, u1 = f11 * 0.5f + f01 * 0.5f; return u1 * 0.5f + u0 * 0.5f; }
    const float w0 = f01 * 0.5f + f00 * 0.5f, w1 = f11 * 0.5f + f10 * 0.5f;
    return w1 * 0.5f + w0 * 0.5f;
}

// index of a neighbouring line (may be negative: slab halo planes); ok = false when the boundary makes it a constant ghost
// line (-> generic path)
__device__ __forceinline__ int fk_res(int i, const DField& f, int a, bool& ok)
{
    float c;
    if (!phi_resolve(i, f, a, c)) { ok = false; return 0; }
    return i;
}

// x indexing of a chunk on the fast path: own index (clamped into the line so that loads of inactive lanes stay in bounds),
// x - 1 and x + 1 (wrapped when x is periodic).  fast == false: the chunk touches a non-periodic x boundary.
struct FkX { int xo, xm, xp; bool fast; };

__device__ __forceinline__ FkX fk_x(const DField& fx, const DField& fc, int n0, int xb, int x)
{
    FkX X;
    const bool per = fx.klo[0] == PHI_BC_PERIODIC;                    // kinds agree between components
    const int lo = max(fx.lo[0], fc.lo[0]), hi = min(fx.hi[0], fc.hi[0]);
    X.fast = per || (xb - 1 >= lo && xb + 32 <= hi);
    X.xo = min(x, n0 - 1);
    X.xm = X.xo - 1; X.xp = X.xo + 1;
    if (per) { if (X.xm < 0) X.xm = n0 - 1; if (X.xp > n0 - 1) X.xp = 0; }
    return X;
}

// ---- generic (boundary-aware) per-sample code, one copy: the arithmetic of advect_kernels.cu -------------------------------
template <int DIM>
__device__ __forceinline__ float fk_velocity_at(const DGrid& g, const DVec& vel, int a, int target, int b, int x, int y, int z)
{
    const float* va = vel.p[a];
    const DField& fa = vel.f[a];
    if (target == a) return phi_fetch<DIM>(va, g, fa, b, x, y, z);
    const int ax = (a == 0), ay = (a == 1), az = (a == 2);
    if (target < 0) {
        const float lo = phi_fetch<DIM>(va, g, fa, b, x, y, z);
        const float hi = phi_fetch<DIM>(va, g, fa, b, x + ax, y + ay, z + az);
        return hi * 0.5f + lo * 0.5f;
    }
    const int tx = (target == 0), ty = (target == 1), tz = (target == 2);
    const float f00 = phi_fetch<DIM>(va, g, fa, b, x - tx, y - ty, z - tz);
    const float f10 = phi_fetch<DIM>(va, g, fa, b, x - tx + ax, y - ty + ay, z - tz + az);
    const float f01 = phi_fetch<DIM>(va, g, fa, b, x, y, z);
    const float f11 = phi_fetch<DIM>(va, g, fa, b, x + ax, y + ay, z + az);
    return fk_avg4(f00, f10, f01, f11, a < target);
}

// sample of field `f` (array src) back-traced from the sample point (x, y, z) of target component `target` (-1: cell centre)
template <int DIM>
__device__ __noinline__ float fk_generic_sample(const DGrid* gp, const DVec* velp, const DField* fp, const float* __restrict__ src,
                                                int target, int b, int x, int y, int z, float dt)
{
    const DGrid& g = *gp; const DVec& vel = *velp;
    FkLookup K; K.i[2] = 0; K.t[2] = 0.f;
    const int idx[3] = {x, y, z};
#pragma unroll
    for (int a = 0; a < DIM; ++a)
        fk_lookup_axis(K, a, idx[a], fk_velocity_at<DIM>(g, vel, a, target, b, x, y, z), dt, g.dx[a], g.inv_dx[a]);
    return fk_interp<DIM>(src, g, *fp, b, K);
}

// Centred field: dst = interp(src, x - dt v(x)) [+ add_scale * add]      (smoke advection + inflow of the notebook step)
template <int DIM>
__global__ void __launch_bounds__(FK_THREADS, 4)
k_advect_centered_vec(const __grid_constant__ DGrid g, const __grid_constant__ DVec vel, const __grid_constant__ DField ff,
                      const float* __restrict__ src, float* __restrict__ dst, float dt, const float* __restrict__ add, float add_scale)
{
    const FkAdvLine L = fk_adv_line<DIM>(g);
    if (!L.ok || L.y >= g.n[1] || (DIM == 3 && L.z >= g.n[2])) return;
    const int lane = threadIdx.x & 31;
    const int b = L.b, y = L.y, z = L.z, n0 = g.n[0];
    const float* vx = vel.p[0]; const float* vy = vel.p[1]; const float* vz = vel.p[2];
    // neighbouring lines: vx (y, z); vy (y, z), (y+1, z); vz (y, z), (y, z+1)
    bool rows_ok = true;
    const int yx = fk_res(y, vel.f[0], 1, rows_ok), zx = DIM == 3 ? fk_res(z, vel.f[0], 2, rows_ok) : 0;
    const int y0 = fk_res(y, vel.f[1], 1, rows_ok), y1 = fk_res(y + 1, vel.f[1], 1, rows_ok), zy = DIM == 3 ? fk_res(z, vel.f[1], 2, rows_ok) : 0;
    const int yz = DIM == 3 ? fk_res(y, vel.f[2], 1, rows_ok) : 0, z0 = DIM == 3 ? fk_res(z, vel.f[2], 2, rows_ok) : 0,
              z1 = DIM == 3 ? fk_res(z + 1, vel.f[2], 2, rows_ok) : 0;
    const int sy = (int)vel.f[0].sy, sz = (int)vel.f[0].sz;
    const int base = b * (int)vel.f[0].sb;
    const int rA = base + zx * sz + yx * sy, rB0 = base + zy * sz + y0 * sy, rB1 = base + zy * sz + y1 * sy;
    const int rC0 = base + z0 * sz + yz * sy, rC1 = base + z1 * sz + yz * sy;
    const long long line = (long long)b * ff.sb + (long long)z * ff.sz + (long long)y * ff.sy;
#pragma unroll 1
    for (int j = 0; j < FK_XCHUNKS; ++j) {
        const int xb = L.xs + 32 * j;
        if (xb >= n0) break;                                       // warp-uniform
        const int x = xb + lane;
        const FkX X = fk_x(vel.f[0], vel.f[1], n0, xb, x);
        float r;
        if (rows_ok && X.fast) {                                   // warp-uniform: straight-line code
            const float a0 = __ldg(vx + rA + X.xo);
            float a0p = __shfl_down_sync(0xffffffffu, a0, 1);
            if (lane == 31 || x == n0 - 1) a0p = __ldg(vx + rA + X.xp);
            const float b0 = __ldg(vy + rB0 + X.xo), b1 = __ldg(vy + rB1 + X.xo);
            FkLookup K; K.i[2] = 0; K.t[2] = 0.f;
            fk_lookup_axis(K, 0, x, a0p * 0.5f + a0 * 0.5f, dt, g.dx[0], g.inv_dx[0]);
            fk_lookup_axis(K, 1, y, b1 * 0.5f + b0 * 0.5f, dt, g.dx[1], g.inv_dx[1]);
            if (DIM == 3) {
                const float c0 = __ldg(vz + rC0 + X.xo), c1 = __ldg(vz + rC1 + X.xo);
                fk_lookup_axis(K, 2, z, c1 * 0.5f + c0 * 0.5f, dt, g.dx[2], g.inv_dx[2]);
            }
            if (x >= n0) continue;
            r = fk_interp<DIM>(src, g, ff, b, K);
        } else {
            if (x >= n0) continue;
            r = fk_generic_sample<DIM>(&g, &vel, &ff, src, -1, b, x, y, z, dt);
        }
        if (add) r = r + add_scale * __ldg(add + line + x);
        dst[line + x] = r;
    }
}

// Staggered field, all components in one launch: dst_c = interp(src_c, face_c - dt v(face_c)) [+ dt * buoyancy_c] [* f_c]
//   buoyancy_c = (s * b_c)[upper cell] * 0.5 + (s * b_c)[lower cell] * 0.5      (sample_grid_at_faces; a constant ghost of s
//   stays c: the product keeps the boundary of s, phi/field/_field.py:809)
//   f_c (FACES, N4): face factors of stationary obstacles, 1 - resample(geometry, v, soft=True, balance=1) = apply_boundary_conditions
//   (phi/physics/fluid.py:212-240).  A separate rounded product after the stored-value arithmetic, as k_mul_faces forms it.
template <int DIM, bool BUOY, bool FACES>
__global__ void __launch_bounds__(FK_THREADS, 4)
k_advect_staggered_vec(const __grid_constant__ DGrid g, const __grid_constant__ DVec vel, const __grid_constant__ DVec fld,
                       const __grid_constant__ DVecOut dst, float dt, const __grid_constant__ DField sf, const float* __restrict__ s,
                       float b0, float b1, float b2, const float* __restrict__ f0, const float* __restrict__ f1, const float* __restrict__ f2)
{
    const FkAdvLine L = fk_adv_line<DIM>(g);
    if (!L.ok) return;
    const int lane = threadIdx.x & 31;
    const int y = L.y, z = L.z, b = L.b, n0 = g.n[0];
    const float* vx = vel.p[0]; const float* vy = vel.p[1]; const float* vz = vel.p[2];
    const DField& fx = vel.f[0]; const DField& fy = vel.f[1]; const DField& fz = vel.f[2];
    // which components store a face on this line (warp-uniform)
    const bool on0 = y >= fld.f[0].lo[1] && y <= fld.f[0].hi[1] && (DIM == 2 || (z >= fld.f[0].lo[2] && z <= fld.f[0].hi[2]));
    const bool on1 = y >= fld.f[1].lo[1] && y <= fld.f[1].hi[1] && (DIM == 2 || (z >= fld.f[1].lo[2] && z <= fld.f[1].hi[2]));
    const bool on2 = DIM == 3 && y >= fld.f[2].lo[1] && y <= fld.f[2].hi[1] && z >= fld.f[2].lo[2] && z <= fld.f[2].hi[2];
    if (!(on0 || on1 || on2)) return;
    // the 11 (3-D) / 4 (2-D) velocity lines the three faces of a cell read, as resolved (y, z) indices per component field
    bool rows_ok = true;
    const int xy0 = fk_res(y, fx, 1, rows_ok), xy1 = fk_res(y - 1, fx, 1, rows_ok);
    const int xz0 = DIM == 3 ? fk_res(z, fx, 2, rows_ok) : 0, xz1 = DIM == 3 ? fk_res(z - 1, fx, 2, rows_ok) : 0;
    const int yy0 = fk_res(y, fy, 1, rows_ok), yy1 = fk_res(y + 1, fy, 1, rows_ok);
    const int yz0 = DIM == 3 ? fk_res(z, fy, 2, rows_ok) : 0, yz1 = DIM == 3 ? fk_res(z - 1, fy, 2, rows_ok) : 0;
    const int zy0 = DIM == 3 ? fk_res(y, fz, 1, rows_ok) : 0, zy1 = DIM == 3 ? fk_res(y - 1, fz, 1, rows_ok) : 0;
    const int zz0 = DIM == 3 ? fk_res(z, fz, 2, rows_ok) : 0, zz1 = DIM == 3 ? fk_res(z + 1, fz, 2, rows_ok) : 0;
    const int sy = (int)fx.sy, sz = (int)fx.sz;
    const int base = b * (int)fx.sb;
    const int rA0 = base + xz0 * sz + xy0 * sy, rA1 = base + xz0 * sz + xy1 * sy, rA2 = base + xz1 * sz + xy0 * sy;
    const int rB0 = base + yz0 * sz + yy0 * sy, rB1 = base + yz0 * sz + yy1 * sy, rB2 = base + yz1 * sz + yy0 * sy, rB3 = base + yz1 * sz + yy1 * sy;
    const int rC0 = base + zz0 * sz + zy0 * sy, rC1 = base + zz1 * sz + zy0 * sy, rC2 = base + zz0 * sz + zy1 * sy, rC3 = base + zz1 * sz + zy1 * sy;
    // buoyancy lines of the centred field (upper cell = this index, lower cell = index - e_c)
    int rS = 0, rSy = 0, rSz = 0;
    bool s_fast = true;
    if (BUOY) {
        // every component's lower-cell line, also for b_c = 0: a constant ghost line adds c/2 * dt even then (-> generic code)
        const int s_y = fk_res(y, sf, 1, s_fast), s_ym = fk_res(y - 1, sf, 1, s_fast);
        const int s_z = DIM == 3 ? fk_res(z, sf, 2, s_fast) : 0, s_zm = DIM == 3 ? fk_res(z - 1, sf, 2, s_fast) : 0;
        const int ssy = (int)sf.sy, ssz = (int)sf.sz, sbase = b * (int)sf.sb;
        rS = sbase + s_z * ssz + s_y * ssy; rSy = sbase + s_z * ssz + s_ym * ssy; rSz = sbase + s_zm * ssz + s_y * ssy;
    }
    const int line = base + z * sz + y * sy;
    const int xend = g.fext[0];
#pragma unroll 1
    for (int j = 0; j < FK_XCHUNKS; ++j) {
        const int xb = L.xs + 32 * j;
        if (xb >= xend) break;                                     // warp-uniform
        const int x = xb + lane;
        const FkX X = fk_x(fx, fy, n0, xb, x);
        // a chunk that holds faces beyond the last cell (x = n0: stored upper boundary faces) is never "fast"
        // (the lower x neighbour of the buoyancy source is wrapped / clamped below; a constant x boundary of s needs xb >= 1 -
        // whatever b0 is, since the constant ghost enters unscaled)
        const bool fast = rows_ok && X.fast && xb + 32 <= n0 && (!BUOY || (s_fast && (sf.klo[0] != PHI_BC_CONST || xb >= 1)));
        float r0 = 0.f, r1 = 0.f, r2 = 0.f;
        // a fast chunk lies inside the stored x range of every component, so its store flags are warp-uniform
        const bool st0 = on0 && (fast || (x >= fld.f[0].lo[0] && x <= fld.f[0].hi[0]));
        const bool st1 = on1 && (fast || (x >= fld.f[1].lo[0] && x <= fld.f[1].hi[0]));
        const bool st2 = on2 && (fast || (x >= fld.f[2].lo[0] && x <= fld.f[2].hi[0]));
        if (fast) {                                                // warp-uniform: straight-line code, 32-bit offsets
            const float A0 = __ldg(vx + rA0 + X.xo), A1 = __ldg(vx + rA1 + X.xo);
            const float B0 = __ldg(vy + rB0 + X.xo), B1 = __ldg(vy + rB1 + X.xo);
            float A2 = 0.f, B2 = 0.f, B3 = 0.f, C0 = 0.f, C1 = 0.f, C2 = 0.f, C3 = 0.f;
            if (DIM == 3) {
                A2 = __ldg(vx + rA2 + X.xo); B2 = __ldg(vy + rB2 + X.xo); B3 = __ldg(vy + rB3 + X.xo);
                C0 = __ldg(vz + rC0 + X.xo); C1 = __ldg(vz + rC1 + X.xo); C2 = __ldg(vz + rC2 + X.xo); C3 = __ldg(vz + rC3 + X.xo);
            }
            float sc = 0.f, sy_ = 0.f, sz_ = 0.f;
            if (BUOY) {
                sc = __ldg(s + rS + X.xo);
                if (b1 != 0.f) sy_ = __ldg(s + rSy + X.xo);
                if (DIM == 3 && b2 != 0.f) sz_ = __ldg(s + rSz + X.xo);
            }
            float A0p = __shfl_down_sync(0xffffffffu, A0, 1), A1p = __shfl_down_sync(0xffffffffu, A1, 1), A2p = __shfl_down_sync(0xffffffffu, A2, 1);
            float B0m = __shfl_up_sync(0xffffffffu, B0, 1), B1m = __shfl_up_sync(0xffffffffu, B1, 1);
            float C0m = __shfl_up_sync(0xffffffffu, C0, 1), C1m = __shfl_up_sync(0xffffffffu, C1, 1);
            float scm = __shfl_up_sync(0xffffffffu, sc, 1);
            if (lane == 31) {
                A0p = __ldg(vx + rA0 + X.xp); A1p = __ldg(vx + rA1 + X.xp);
                if (DIM == 3) A2p = __ldg(vx + rA2 + X.xp);
            }
            if (lane == 0) {
                B0m = __ldg(vy + rB0 + X.xm); B1m = __ldg(vy + rB1 + X.xm);
                if (DIM == 3) { C0m = __ldg(vz + rC0 + X.xm); C1m = __ldg(vz + rC1 + X.xm); }
                if (BUOY && b0 != 0.f) {             // s(x - 1): wrapped (PERIODIC) or clamped (ZERO_GRADIENT) at x = 0
                    int sxm = x - 1;
                    if (sxm < 0) sxm = sf.klo[0] == PHI_BC_PERIODIC ? n0 - 1 : 0;
                    scm = __ldg(s + rS + sxm);
                }
            }
            FkLookup K0, K1, K2;
            K0.i[2] = K1.i[2] = K2.i[2] = 0; K0.t[2] = K1.t[2] = K2.t[2] = 0.f;
            const float dx = g.dx[0], dy = g.dx[1], dz = g.dx[2], ix = g.inv_dx[0], iy = g.inv_dx[1], iz = g.inv_dx[2];
            // x faces (target axis 0), y faces (1), z faces (2)
            fk_lookup_axis(K0, 0, x, A0, dt, dx, ix);
            fk_lookup_axis(K0, 1, y, fk_avg4(B0m, B1m, B0, B1, false), dt, dy, iy);
            fk_lookup_axis(K1, 0, x, fk_avg4(A1, A1p, A0, A0p, true), dt, dx, ix);
            fk_lookup_axis(K1, 1, y, B0, dt, dy, iy);
            if (DIM == 3) {
                fk_lookup_axis(K0, 2, z, fk_avg4(C0m, C1m, C0, C1, false), dt, dz, iz);
                fk_lookup_axis(K1, 2, z, fk_avg4(C2, C3, C0, C1, false), dt, dz, iz);
                fk_lookup_axis(K2, 0, x, fk_avg4(A2, A2p, A0, A0p, true), dt, dx, ix);
                fk_lookup_axis(K2, 1, y, fk_avg4(B2, B3, B0, B1, true), dt, dy, iy);
                fk_lookup_axis(K2, 2, z, C0, dt, dz, iz);
            }
            const bool all_in = fk_inside<DIM>(fld.f[0], K0) && fk_inside<DIM>(fld.f[1], K1) && (DIM == 2 || fk_inside<DIM>(fld.f[2], K2));
            if (all_in) {                                          // the common case: 24 independent gathers in flight
                r0 = fk_interp_inside<DIM>(fld.p[0], fld.f[0], b, K0);
                r1 = fk_interp_inside<DIM>(fld.p[1], fld.f[1], b, K1);
                if (DIM == 3) r2 = fk_interp_inside<DIM>(fld.p[2], fld.f[2], b, K2);
            } else {
                if (st0) r0 = fk_interp<DIM>(fld.p[0], g, fld.f[0], b, K0);
                if (st1) r1 = fk_interp<DIM>(fld.p[1], g, fld.f[1], b, K1);
                if (DIM == 3 && st2) r2 = fk_interp<DIM>(fld.p[2], g, fld.f[2], b, K2);
            }
            if (BUOY) {                                            // no constant ghost of s on a fast chunk: b_c = 0 adds 0
                if (b0 != 0.f) r0 = r0 + ((sc * b0) * 0.5f + (scm * b0) * 0.5f) * dt;
                if (b1 != 0.f) r1 = r1 + ((sc * b1) * 0.5f + (sy_ * b1) * 0.5f) * dt;
                if (DIM == 3 && b2 != 0.f) r2 = r2 + ((sc * b2) * 0.5f + (sz_ * b2) * 0.5f) * dt;
            }
        } else {                                                   // boundary chunks: per-sample generic code (one copy)
            if (x >= xend) continue;
#pragma unroll 1
            for (int c = 0; c < DIM; ++c) {
                const bool st = c == 0 ? st0 : (c == 1 ? st1 : st2);
                if (!st) continue;
                float r = fk_generic_sample<DIM>(&g, &vel, &fld.f[c], fld.p[c], c, b, x, y, z, dt);
                const float bc = c == 0 ? b0 : (c == 1 ? b1 : b2);
                if (BUOY) {                                        // a constant ghost of s enters unscaled (phi_fetch_scaled)
                    const float up = phi_fetch_scaled<DIM>(s, g, sf, b, x, y, z, bc);
                    const float lw = phi_fetch_scaled<DIM>(s, g, sf, b, x - (c == 0), y - (c == 1), z - (c == 2), bc);
                    r = r + (up * 0.5f + lw * 0.5f) * dt;
                }
                if (c == 0) r0 = r; else if (c == 1) r1 = r; else r2 = r;
            }
        }
        if (FACES) {
            if (st0) r0 = __fmul_rn(r0, __ldg(f0 + line + x));
            if (st1) r1 = __fmul_rn(r1, __ldg(f1 + line + x));
            if (DIM == 3 && st2) r2 = __fmul_rn(r2, __ldg(f2 + line + x));
        }
        if (st0) dst.p[0][line + x] = r0;
        if (st1) dst.p[1][line + x] = r1;
        if (DIM == 3 && st2) dst.p[2][line + x] = r2;
    }
}

static dim3 adv_grid(const DGrid& g)
{
    return dim3((g.fext[0] + 32 * FK_XCHUNKS - 1) / (32 * FK_XCHUNKS), (g.fext[1] + FK_WARPS - 1) / FK_WARPS, g.fext[2] * g.batch);
}

// the fast paths index with 32-bit element offsets
static bool fits_int32(const DGrid& g)
{
    return (long long)g.fext[0] * g.fext[1] * g.fext[2] * g.batch < (1ll << 31) - (1ll << 20);
}

int phi_launch_advect_centered_vec(const DGrid& g, const DVec& vel, const DField& ff, const float* src, float* dst, float dt,
                                   const float* add, float add_scale, cudaStream_t s)
{
    if (!fits_int32(g)) return -100;
    if (g.dim == 3) k_advect_centered_vec<3><<<adv_grid(g), FK_THREADS, 0, s>>>(g, vel, ff, src, dst, dt, add, add_scale);
    else            k_advect_centered_vec<2><<<adv_grid(g), FK_THREADS, 0, s>>>(g, vel, ff, src, dst, dt, add, add_scale);
    return (int)cudaGetLastError();
}

int phi_launch_advect_staggered_vec(const DGrid& g, const DVec& vel, const DVec& fld, const DVecOut& dst, float dt,
                                    const DField* sf, const float* sarr, const float bu[3], const float* const* faces, cudaStream_t s)
{
    if (!fits_int32(g)) return -100;
    const DField sfv = sf ? *sf : fld.f[0];
    bool const_side = false;                 // resample(s * b, to=v) is c/2 * dt next to a constant side c != 0 of s, even for b = 0
    for (int a = 0; a < g.dim; ++a)
        const_side = const_side || (sfv.klo[a] == PHI_BC_CONST && sfv.clo[a] != 0.f) || (sfv.khi[a] == PHI_BC_CONST && sfv.chi[a] != 0.f);
    const bool buoy = sarr != nullptr && bu && (bu[0] != 0.f || bu[1] != 0.f || (g.dim == 3 && bu[2] != 0.f) || const_side);
    const float b0 = buoy ? bu[0] : 0.f, b1 = buoy ? bu[1] : 0.f, b2 = (buoy && g.dim == 3) ? bu[2] : 0.f;
    const float* f0 = faces ? faces[0] : nullptr;
    const float* f1 = faces ? faces[1] : nullptr;
    const float* f2 = faces && g.dim == 3 ? faces[2] : nullptr;
#define FK_ADV_STAG(D, B, F) k_advect_staggered_vec<D, B, F><<<adv_grid(g), FK_THREADS, 0, s>>>(g, vel, fld, dst, dt, sfv, sarr, b0, b1, b2, f0, f1, f2)
    if (g.dim == 3) {
        if (faces) { if (buoy) FK_ADV_STAG(3, true, true); else FK_ADV_STAG(3, false, true); }
        else       { if (buoy) FK_ADV_STAG(3, true, false); else FK_ADV_STAG(3, false, false); }
    } else {
        if (faces) { if (buoy) FK_ADV_STAG(2, true, true); else FK_ADV_STAG(2, false, true); }
        else       { if (buoy) FK_ADV_STAG(2, true, false); else FK_ADV_STAG(2, false, false); }
    }
#undef FK_ADV_STAG
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// A11  math.grid_sample at caller-provided index-space coordinates (PhiML/phiml/math/_ops.py:936-1015): the Backend.grid_sample
// contract of the reference-side plugin (PhiML/phiml/backend/_backend.py:1578-1593).  frac = c % 1 = c - floor(c).
// ---------------------------------------------------------------------------------------------------------
template <int DIM>
__global__ void __launch_bounds__(256)
k_grid_sample(const __grid_constant__ DGrid g, const __grid_constant__ DField f, const float* __restrict__ grid,
              const float* __restrict__ coords, long long npoints, float* __restrict__ out)
{
    const long long total = npoints * g.batch;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / npoints);
        FkLookup K; K.i[2] = 0; K.t[2] = 0.f;
#pragma unroll
        for (int a = 0; a < DIM; ++a) {
            const float c = __ldg(coords + i * DIM + a);
            const float fl = floorf(c);
            K.i[a] = (int)fl; K.t[a] = c - fl;
        }
        out[i] = fk_interp<DIM>(grid, g, f, b, K);
    }
}

int phi_launch_grid_sample(const DGrid& g, const DField& f, const float* grid, const float* coords, long long npoints, float* out, cudaStream_t s)
{
    const long long total = npoints * g.batch;
    if (total <= 0) return 0;
    long long blocks = (total + 255) / 256;
    const long long max_blocks = (long long)phi_sm_count() * 32;
    if (blocks > max_blocks) blocks = max_blocks;
    if (g.dim == 3) k_grid_sample<3><<<(int)blocks, 256, 0, s>>>(g, f, grid, coords, npoints, out);
    else            k_grid_sample<2><<<(int)blocks, 256, 0, s>>>(g, f, grid, coords, npoints, out);
    return (int)cudaGetLastError();
}
