// TMA-staged shared-memory ring for the 5/7-point stencil: the H100 fast path of laplace (A7) and of the CG solve (A12).
//
// Why: the stencil kernels are pure HBM streams (8..20 B/cell).  Saturating 3.35 TB/s needs ~25 KB in flight per SM; with
// register-staged loads that costs occupancy the CG passes do not have.  Here ONE producer warp per CTA streams whole
// grid lines into a ring of shared-memory stages with cp.async.bulk (the TMA engine; SASS: UBLKCP) completing on
// mbarriers, and eight consumer warps compute out of shared memory.  Loads never occupy registers, the pipeline depth
// is a launch parameter, and every byte is fetched from L2/HBM exactly once per tile (+ halo lines).
//
// Tile = TY consecutive grid lines (full x extent) of one z plane (3-D) or of one image (2-D).  In 3-D a CTA marches a
// chunk of planes; plane z needs planes z-1, z, z+1, which sit in three consecutive ring slots.  Halo lines y0-1 / y0+TY
// and halo planes are fetched from wherever the boundary condition says the ghost values live:
//   PERIODIC -> the wrapped line, ZERO_GRADIENT -> the clamped line, constant -> not fetched (consumers substitute c).
// x ghosts are read from the staged line itself.  Outputs go straight from registers to global memory (STG.128).
//
// The consumer loop is issue-bound if written naively (first ncu capture: 200+ instructions per 4 cells), so every
// thread precomputes the geometry of the <= 4 float4 groups it owns once per kernel, boundary flags once per tile, and
// the common case runs a branch-free path: 5 LDS.128 + 2 SHFL + ~40 FP32 ops + 1 STG.128 per group.
#include <cooperative_groups.h>
#include <type_traits>
#include "cg_common.cuh"
#include <cstdlib>
#include <cstring>
#include "launch.cuh"

namespace cg = cooperative_groups;

#define RING_CONSUMERS 256
#define RING_THREADS (RING_CONSUMERS + 32)
#define RING_MAX_STAGES 8
#define RING_G 4                 // float4 groups per consumer thread and plane (TY * nx4 <= RING_G * 256)

struct RingCfg {
    int TY, R, pitch, nx4;
    int stage_floats;          // floats between consecutive stages
    int ZC, nyt, nzc;
    int units_per_batch, total_units;
    int consumers;             // consumer threads per CTA (256 or 512); the producer warp follows them
    int groups;                // ceil(TY * nx4 / consumers)
    int shfl_ok;               // lanes of a warp own consecutive groups of one line -> x neighbours via shuffles
    // "tail split" decomposition of the CG kernel (3-D, batch 1, fewer y tiles than persistent CTAs): CTA c < nyt marches tile c
    // over planes [0, Zm); the remaining CTAs share the tails [Zm, nz) of all tiles, split_t tiles each.  Keeps every SM busy
    // when the tile count does not divide the CTA count (128 tiles on 132 SMs for 512-wide slabs).
    int split, Zm, split_t;
};

// ---- PTX wrappers ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{ asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{ asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }

// ---- ring state (per thread, registers) ------------------------------------------------------------------------------
struct SlotIt {                 // a position in the ring: slot index + parity of its current use
    int slot; unsigned par;
    __device__ __forceinline__ void next(int R) { if (++slot == R) { slot = 0; par ^= 1u; } }
};

struct Ring {
    float* stage0;
    uint32_t stage0_s, full0, empty0;
    SlotIt pos;                // next plane to produce (producer) / first plane of the next unit (consumers)
};

__device__ __forceinline__ void ring_init(Ring& rg, unsigned char* smem, const RingCfg& cfg)
{
    // layout: [8 full barriers][8 empty barriers][stages]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
    rg.full0 = smem_u32(bars);
    rg.empty0 = smem_u32(bars + RING_MAX_STAGES);
    rg.stage0 = reinterpret_cast<float*>(smem + 128);
    rg.stage0_s = smem_u32(rg.stage0);
    rg.pos.slot = 0; rg.pos.par = 0;
    if (threadIdx.x == 0) {
        for (int s = 0; s < cfg.R; ++s) {
            mbar_init(rg.full0 + 8 * s, 1);
            mbar_init(rg.empty0 + 8 * s, cfg.consumers / 32);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
}

// Producer warp.  Lane l owns staged lines l, l+32, l+64, l+96 of a stage: first the NH haloed arrays (TY+2 lines
// each), then the NE element-wise arrays (TY lines each).  Everything that does not depend on the plane is resolved once
// per unit (ProdUnit); per plane the producer only resolves z, adds it to the line offsets and issues the bulk copies -
// the producer is a single warp, so its serial instruction count per plane bounds the whole pipeline.
struct ProdUnit {
    long long yoff[4];          // b*sb + y*sy of the source line (boundary already applied to y)
    const float* base[4];       // source array
    uint32_t dsto[4];           // byte offset of the destination line inside a stage
    uint32_t nbytes[4];         // bytes of the copy this lane issues: consecutive lines of one array are merged into one copy
    unsigned hmask, emask;      // which of the 4 lines are active haloed / element-wise lines
    int tot_h, tot_e;           // warp totals of active lines
};

// A line that continues the one held by the previous lane (same key = array, next source row yv) rides on that lane's copy.
// key < 0: the lane holds no line.  Returns whether this lane issues a copy; if so, nbytes covers its line and the ones that follow.
__device__ __forceinline__ bool prod_merge_lines(int key, int yv, bool mergeable, uint32_t row_bytes, uint32_t& nbytes)
{
    const int lane = threadIdx.x & 31;
    const int pkey = __shfl_up_sync(0xffffffffu, key, 1), pyv = __shfl_up_sync(0xffffffffu, yv, 1);
    const bool cont = mergeable && key >= 0 && lane > 0 && pkey == key && pyv + 1 == yv;
    const unsigned cm = __ballot_sync(0xffffffffu, cont);
    if (key < 0 || cont) return false;
    const unsigned follow = lane == 31 ? 0u : (cm >> (lane + 1));
    nbytes = (uint32_t)__ffs(~follow) * row_bytes;          // 1 + number of lines that continue this one
    return true;
}

// hactive: bit k set = haloed slot k is fetched (slot 1 idles in the first CG iteration; with obstacles the last slot is the mask)
// KSLOT (varying diffusivity): the last haloed slot is read from batch entry kb instead of b (kb = 0 broadcasts one k to all entries)
template <int DIM, bool KSLOT = false>
__device__ __forceinline__ void prod_unit_setup(ProdUnit& pu, const RingCfg& cfg, const DGrid& g, const DField& pf,
                                                unsigned hactive, int NHslots, int NE, const float* const* hsrc, const float* const* esrc,
                                                int b, int y0, int kb = 0)
{
    const int lane = threadIdx.x & 31, hrows = cfg.TY + 2;
    const uint32_t row_bytes = (uint32_t)cfg.pitch * 4u;
    const bool mergeable = pf.sy == cfg.pitch;      // neighbouring lines are contiguous in memory and in the stage
    pu.hmask = pu.emask = 0;
    int ch = 0, ce = 0;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int r = lane + 32 * it;
        pu.yoff[it] = 0; pu.base[it] = nullptr; pu.dsto[it] = 0; pu.nbytes[it] = row_bytes;
        int key = -1, yv = 0;                                    // array of an active line, its source row
        bool halo_line = false;
        if (r < NHslots * hrows) {
            const int arr = r / hrows, j = r - arr * hrows;
            int yy = y0 - 1 + j; float cv;
            if (((hactive >> arr) & 1u) && yy <= g.n[1] && phi_resolve(yy, pf, 1, cv)) {
                pu.yoff[it] = (long long)((KSLOT && arr == NHslots - 1) ? kb : b) * pf.sb + (long long)yy * pf.sy;
                pu.base[it] = hsrc[arr];
                pu.dsto[it] = 4u * (uint32_t)((arr * hrows + j) * cfg.pitch);
                key = arr; yv = yy; halo_line = true; ch++;
            }
        } else if (r < NHslots * hrows + NE * cfg.TY) {
            const int q = r - NHslots * hrows, arr = q / cfg.TY, j = q - arr * cfg.TY;
            const int yy = y0 + j;
            if (yy < g.n[1]) {
                pu.yoff[it] = (long long)b * pf.sb + (long long)yy * pf.sy;
                pu.base[it] = esrc[arr];
                pu.dsto[it] = 4u * (uint32_t)((NHslots * hrows + arr * cfg.TY + j) * cfg.pitch);
                key = 8 + arr; yv = yy; ce++;
            }
        }
        if (prod_merge_lines(key, yv, mergeable, row_bytes, pu.nbytes[it])) {
            if (halo_line) pu.hmask |= 1u << it; else pu.emask |= 1u << it;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { ch += __shfl_xor_sync(0xffffffffu, ch, o); ce += __shfl_xor_sync(0xffffffffu, ce, o); }
    pu.tot_h = ch; pu.tot_e = ce;
}

template <int DIM>
__device__ __forceinline__ void ring_produce(Ring& rg, const RingCfg& cfg, const DField& pf, const ProdUnit& pu, int z, bool interior)
{
    const int lane = threadIdx.x & 31;
    const int slot = rg.pos.slot;
    const uint32_t full = rg.full0 + 8 * slot;
    const uint32_t row_bytes = (uint32_t)cfg.pitch * 4u;
    const uint32_t sbase = rg.stage0_s + 4u * (uint32_t)(slot * cfg.stage_floats);
    float cv;
    bool zmem = true;
    if (DIM == 3) zmem = phi_resolve(z, pf, 2, cv); else z = 0;
    const long long zoff = (long long)z * pf.sz;
    unsigned mask = (zmem ? pu.hmask : 0u) | (interior ? pu.emask : 0u);
    const int cnt = (zmem ? pu.tot_h : 0) + (interior ? pu.tot_e : 0);
    if (lane == 0) {
        mbar_wait(rg.empty0 + 8 * slot, rg.pos.par ^ 1u);
        if (cnt > 0) mbar_expect_tx(full, (uint32_t)cnt * row_bytes); else mbar_arrive(full);
    }
    __syncwarp();
#pragma unroll
    for (int it = 0; it < 4; ++it)
        if (mask & (1u << it)) bulk_g2s(sbase + pu.dsto[it], pu.base[it] + pu.yoff[it] + zoff, pu.nbytes[it], full);
    rg.pos.next(cfg.R);
}

__device__ __forceinline__ void ring_wait_full(const Ring& rg, const SlotIt& s) { mbar_wait(rg.full0 + 8 * s.slot, s.par); }
__device__ __forceinline__ void ring_release(const Ring& rg, const SlotIt& s)
{
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(rg.empty0 + 8 * s.slot);
}
__device__ __forceinline__ const float* ring_ptr(const Ring& rg, const RingCfg& cfg, const SlotIt& s)
{ return rg.stage0 + (size_t)s.slot * cfg.stage_floats; }

// ---- consumer geometry --------------------------------------------------------------------------------------------------
#define GF_VALID 1u
#define GF_XLO   2u     // group holds x = 0
#define GF_XHI   4u     // group holds the last cell of the line
#define GF_YLOC  8u     // y-1 neighbour is a constant ghost
#define GF_YHIC  16u    // y+1 neighbour is a constant ghost

struct ThreadGroups {
    int soff[RING_G];       // float offset of the group inside a haloed array of a stage: (j+1)*pitch + x0
    int eoff[RING_G];       // float offset inside an element-wise array of a stage: j*pitch + x0
    int goff[RING_G];       // element offset relative to (y0, x=0) of the plane: j*sy + x0
    int j[RING_G];
    int xlo[RING_G], xro[RING_G];   // where the x-1 / x+4 neighbour lives in the staged line (ghosts resolved), fast path
    unsigned needl, needr;  // bit k: the neighbour of group k cannot come from a shuffle (warp edge or line end)
    unsigned flags[RING_G]; // per tile
    bool fast_ok;           // kernel-level eligibility of the branch-free path
};

__device__ __forceinline__ void groups_init(ThreadGroups& tg, const RingCfg& cfg, const DGrid& g, const DField& pf)
{
    const int lane = threadIdx.x & 31, nx = g.n[0];
    tg.needl = tg.needr = 0;
#pragma unroll
    for (int k = 0; k < RING_G; ++k) {
        const int gi = threadIdx.x + k * cfg.consumers;
        const int j = gi / cfg.nx4, x0 = (gi - j * cfg.nx4) * 4;
        tg.j[k] = (k < cfg.groups && j < cfg.TY && x0 < nx) ? j : -1;
        tg.soff[k] = (j + 1) * cfg.pitch + x0;
        tg.eoff[k] = j * cfg.pitch + x0;
        tg.goff[k] = j * (int)pf.sy + x0;
        tg.flags[k] = 0;
        const int row = (j + 1) * cfg.pitch;
        tg.xlo[k] = tg.soff[k] - 1; tg.xro[k] = tg.soff[k] + 4;
        if (lane == 0) tg.needl |= 1u << k;
        if (lane == 31) tg.needr |= 1u << k;
        if (x0 == 0) { tg.needl |= 1u << k; tg.xlo[k] = pf.klo[0] == PHI_BC_PERIODIC ? row + nx - 1 : row; }
        if (x0 + 4 >= nx) { tg.needr |= 1u << k; tg.xro[k] = pf.khi[0] == PHI_BC_PERIODIC ? row : row + nx - 1; }
        // lanes that take their neighbour from a shuffle still execute the (branch-free) edge load: one broadcast address
        if (!(tg.needl & (1u << k))) tg.xlo[k] = 0;
        if (!(tg.needr & (1u << k))) tg.xro[k] = 0;
    }
    tg.fast_ok = cfg.shfl_ok && (cfg.nx4 * 4 == nx) && (cfg.TY * cfg.nx4 == cfg.groups * cfg.consumers)
                 && pf.klo[0] != PHI_BC_CONST && pf.khi[0] != PHI_BC_CONST;
}

__device__ __forceinline__ void groups_tile(ThreadGroups& tg, const RingCfg& cfg, const DGrid& g, const DField& pf, int y0)
{
    const int nx = g.n[0], ny = g.n[1];
#pragma unroll
    for (int k = 0; k < RING_G; ++k) {
        unsigned f = 0;
        if (tg.j[k] >= 0) {
            const int y = y0 + tg.j[k];
            const int x0 = tg.eoff[k] - tg.j[k] * cfg.pitch;
            if (y < ny) {
                f = GF_VALID;
                if (x0 == 0) f |= GF_XLO;
                if (x0 + 4 >= nx) f |= GF_XHI;
                if (y == 0 && pf.klo[1] == PHI_BC_CONST) f |= GF_YLOC;
                if (y == ny - 1 && pf.khi[1] == PHI_BC_CONST) f |= GF_YHIC;
            }
        }
        tg.flags[k] = f;
    }
}

// Epilogues that declare kTwoFields (reaction-diffusion, N7) take the two haloed arrays of a stage as two fields: ring_compute_any
// runs the consumer once per field (field 1 on the stage pointers moved by one haloed array), tells the epilogue the field and the
// group k of each call, and both consumers form the stencil with stencil_ref - so a cell's bits do not depend on the consumer, the
// tile or the variant that computed it.
template <class E, class = void> struct RingTwoFields : std::false_type {};
template <class E> struct RingTwoFields<E, std::void_t<decltype(E::kTwoFields)>> : std::integral_constant<bool, E::kTwoFields> {};
// Epilogues that declare kRefStencil (the wave step, N8) take the one haloed array's laplacian from stencil_ref as well, for the same reason.
template <class E, class = void> struct RingRefStencil : RingTwoFields<E> {};
template <class E> struct RingRefStencil<E, std::void_t<decltype(E::kRefStencil)>> : std::integral_constant<bool, E::kRefStencil> {};

// sum over axes of (lower + upper - 2 c) / dx^2 in oracle_np.laplace's order, each operation rounded on its own (no contraction)
__device__ __forceinline__ float lap_axis(float lo, float hi, float c, float idx2)
{ return __fmul_rn(__fsub_rn(__fadd_rn(lo, hi), __fmul_rn(2.f, c)), idx2); }
template <int DIM>
__device__ __forceinline__ float lap_ref(float c, float l, float r, float ym, float yp, float zm, float zp, float ix2, float iy2, float iz2)
{
    const float s = __fadd_rn(lap_axis(l, r, c, ix2), lap_axis(ym, yp, c, iy2));
    return DIM == 3 ? __fadd_rn(s, lap_axis(zm, zp, c, iz2)) : s;
}
// l4 / r4: the x-1 / x+1 neighbours of the four cells
template <int DIM>
__device__ __forceinline__ float4 stencil_ref(const float4& c, const float4& l4, const float4& r4, const float4& ym, const float4& yp,
                                              const float4& zm, const float4& zp, float ix2, float iy2, float iz2)
{
    return make_float4(lap_ref<DIM>(c.x, l4.x, r4.x, ym.x, yp.x, zm.x, zp.x, ix2, iy2, iz2),
                       lap_ref<DIM>(c.y, l4.y, r4.y, ym.y, yp.y, zm.y, zp.y, ix2, iy2, iz2),
                       lap_ref<DIM>(c.z, l4.z, r4.z, ym.z, yp.z, zm.z, zp.z, ix2, iy2, iz2),
                       lap_ref<DIM>(c.w, l4.w, r4.w, ym.w, yp.w, zm.w, zp.w, ix2, iy2, iz2));
}

// ---- consumer: one plane of one tile ---------------------------------------------------------------------------------
// sm/sc/sp: stages holding planes z-1, z, z+1 (sm/sp unused in 2-D).  Values of the differenced array are h0 (+ beta*h1).
// Operators with an extra haloed slot (cg_op_xslot) run the face-minimum stencil
//   q_c = sum_faces min(w_c, w_nb) * (v_nb - v_c) / dx^2
// on coefficients w of the last haloed slot of a stage, which travel like the values (same staged lines):
//   Masked (N4, static obstacles): w = the accessible mask; a constant ghost counts as accessible (w = 1); obstacle cells take
//     q_c = v_c (fluid.masked_laplace, phi/physics/fluid.py:197-202), and the mask goes to the epilogue (set_acc);
//   HelmholtzVarying (N6): w = fl(od->ndt * k) (ndt = -dt), rounded as the reference rounds k * (-dt); a constant side's ghost
//     coefficient is its boundary constant od->kclo / od->kchi itself (phi/physics/diffuse.py:129-141).
template <int DIM, int NH, int NE, CgOp OP = CgOp::Poisson, class Epi>
__device__ __forceinline__ void ring_compute(const RingCfg& cfg, const DGrid& g, const DField& pf, const ThreadGroups& tg,
                                             const float* sm, const float* sc, const float* sp, float beta,
                                             long long plane_off, int z, Epi& epi, const CgOperator* od)
{
    const int pitch = cfg.pitch;
    const int h1 = (cfg.TY + 2) * pitch;                 // offset of the second haloed array inside a stage
    const int aoff = NH * (cfg.TY + 2) * pitch;          // offset of the operator's coefficients (cg_op_xslot)
    const int e0off = (NH + (cg_op_xslot(OP) ? 1 : 0)) * (cfg.TY + 2) * pitch;
    const int e1off = e0off + cfg.TY * pitch;
    const float ix2 = g.inv_dx2[0], iy2 = g.inv_dx2[1], iz2 = g.inv_dx2[2];
    const bool zm_const = DIM == 3 && z == 0 && pf.klo[2] == PHI_BC_CONST;
    const bool zp_const = DIM == 3 && z == g.n[2] - 1 && pf.khi[2] == PHI_BC_CONST;
    const bool use1 = NH == 2 && beta != 0.f;
    const int lane = threadIdx.x & 31;

    auto val4 = [&](const float* s, int off) -> float4 {
        float4 a = *reinterpret_cast<const float4*>(s + off);
        if (use1) { const float4 o = *reinterpret_cast<const float4*>(s + h1 + off);
                    a.x = fmaf(beta, o.x, a.x); a.y = fmaf(beta, o.y, a.y); a.z = fmaf(beta, o.z, a.z); a.w = fmaf(beta, o.w, a.w); }
        return a;
    };
    auto val1 = [&](const float* s, int off) -> float {
        float a = s[off];
        if (use1) a = fmaf(beta, s[h1 + off], a);
        return a;
    };

#pragma unroll
    for (int k = 0; k < RING_G; ++k) {
        const unsigned f = tg.flags[k];
        const int rc = tg.soff[k];
        const bool valid = (f & GF_VALID) != 0;
        float4 c = f4_splat(0.f);
        if (valid) c = val4(sc, rc);
        float xl, xr;
        if (cfg.shfl_ok) {                                  // whole warp executes the shuffles (uniform branch)
            xl = __shfl_up_sync(0xffffffffu, c.w, 1);
            xr = __shfl_down_sync(0xffffffffu, c.x, 1);
            if (valid && lane == 0 && !(f & GF_XLO)) xl = val1(sc, rc - 1);
            if (valid && lane == 31 && !(f & GF_XHI)) xr = val1(sc, rc + 4);
        } else if (valid) {
            xl = (f & GF_XLO) ? 0.f : val1(sc, rc - 1);
            xr = (f & GF_XHI) ? 0.f : val1(sc, rc + 4);
        }
        if (!valid) continue;
        float4 ym, yp, q;
        int nvalid = 4;
        if (f == GF_VALID) {                                // interior of the line, no constant ghosts in y
            ym = val4(sc, rc - pitch);
            yp = val4(sc, rc + pitch);
        } else {
            const int row = rc - (tg.eoff[k] - tg.j[k] * pitch);          // start of the staged line
            const int nx = g.n[0];
            const int x0 = rc - row;
            nvalid = min(4, nx - x0);
            ym = (f & GF_YLOC) ? f4_splat(pf.clo[1]) : val4(sc, rc - pitch);
            yp = (f & GF_YHIC) ? f4_splat(pf.chi[1]) : val4(sc, rc + pitch);
            if (f & GF_XLO) { const int kx = pf.klo[0]; xl = kx == PHI_BC_PERIODIC ? val1(sc, row + nx - 1) : (kx == PHI_BC_ZERO_GRADIENT ? c.x : pf.clo[0]); }
            if (f & GF_XHI) { const int kx = pf.khi[0]; xr = kx == PHI_BC_PERIODIC ? val1(sc, row) : (kx == PHI_BC_ZERO_GRADIENT ? f4_get(c, nvalid - 1) : pf.chi[0]); }
        }
        float4 r4 = make_float4(c.y, c.z, c.w, xr);
        if (nvalid < 4) f4_set(r4, nvalid - 1, xr);
        if constexpr (cg_op_xslot(OP)) {
            const float* am = sm + aoff; const float* ac_ = sc + aoff; const float* ap = sp + aoff;
            // coefficient of a staged value, ghost coefficients of the constant sides
            auto cw = [od](float v) { return OP == CgOp::Masked ? v : __fmul_rn(od->ndt, v); };
            auto cw4 = [&](const float* p) { const float4 v = *reinterpret_cast<const float4*>(p); return make_float4(cw(v.x), cw(v.y), cw(v.z), cw(v.w)); };
            auto glo = [od](int ax) { return OP == CgOp::Masked ? 1.f : od->kclo[ax]; };
            auto ghi = [od](int ax) { return OP == CgOp::Masked ? 1.f : od->kchi[ax]; };
            const float4 ac = cw4(ac_ + rc);
            const int row = rc - (tg.eoff[k] - tg.j[k] * pitch);
            const int nx = g.n[0];
            float axl = (f & GF_XLO) ? (pf.klo[0] == PHI_BC_PERIODIC ? cw(ac_[row + nx - 1]) : (pf.klo[0] == PHI_BC_ZERO_GRADIENT ? ac.x : glo(0))) : cw(ac_[rc - 1]);
            float axr = (f & GF_XHI) ? (pf.khi[0] == PHI_BC_PERIODIC ? cw(ac_[row]) : (pf.khi[0] == PHI_BC_ZERO_GRADIENT ? f4_get(ac, nvalid - 1) : ghi(0))) : cw(ac_[rc + 4]);
            const float4 al4 = make_float4(axl, ac.x, ac.y, ac.z);
            float4 ar4 = make_float4(ac.y, ac.z, ac.w, axr);
            if (nvalid < 4) f4_set(ar4, nvalid - 1, axr);
            const float4 l4 = make_float4(xl, c.x, c.y, c.z);
            const float4 aym = (f & GF_YLOC) ? f4_splat(glo(1)) : cw4(ac_ + rc - pitch);
            const float4 ayp = (f & GF_YHIC) ? f4_splat(ghi(1)) : cw4(ac_ + rc + pitch);
            auto term = [](float vn, float vc, float an, float a0) { return fminf(an, a0) * (vn - vc); };
            q.x = (term(l4.x, c.x, al4.x, ac.x) + term(r4.x, c.x, ar4.x, ac.x)) * ix2 + (term(ym.x, c.x, aym.x, ac.x) + term(yp.x, c.x, ayp.x, ac.x)) * iy2;
            q.y = (term(l4.y, c.y, al4.y, ac.y) + term(r4.y, c.y, ar4.y, ac.y)) * ix2 + (term(ym.y, c.y, aym.y, ac.y) + term(yp.y, c.y, ayp.y, ac.y)) * iy2;
            q.z = (term(l4.z, c.z, al4.z, ac.z) + term(r4.z, c.z, ar4.z, ac.z)) * ix2 + (term(ym.z, c.z, aym.z, ac.z) + term(yp.z, c.z, ayp.z, ac.z)) * iy2;
            q.w = (term(l4.w, c.w, al4.w, ac.w) + term(r4.w, c.w, ar4.w, ac.w)) * ix2 + (term(ym.w, c.w, aym.w, ac.w) + term(yp.w, c.w, ayp.w, ac.w)) * iy2;
            if (DIM == 3) {
                const float4 zm = zm_const ? f4_splat(pf.clo[2]) : val4(sm, rc);
                const float4 zp = zp_const ? f4_splat(pf.chi[2]) : val4(sp, rc);
                const float4 azm = zm_const ? f4_splat(glo(2)) : cw4(am + rc);
                const float4 azp = zp_const ? f4_splat(ghi(2)) : cw4(ap + rc);
                q.x += (term(zm.x, c.x, azm.x, ac.x) + term(zp.x, c.x, azp.x, ac.x)) * iz2;
                q.y += (term(zm.y, c.y, azm.y, ac.y) + term(zp.y, c.y, azp.y, ac.y)) * iz2;
                q.z += (term(zm.z, c.z, azm.z, ac.z) + term(zp.z, c.z, azp.z, ac.z)) * iz2;
                q.w += (term(zm.w, c.w, azm.w, ac.w) + term(zp.w, c.w, azp.w, ac.w)) * iz2;
            }
            if constexpr (OP == CgOp::Masked) {
                if (ac.x == 0.f) q.x = c.x;
                if (ac.y == 0.f) q.y = c.y;
                if (ac.z == 0.f) q.z = c.z;
                if (ac.w == 0.f) q.w = c.w;
                epi.set_acc(ac);
            }
        } else if constexpr (RingRefStencil<Epi>::value) {
            const float4 zm = DIM == 3 ? (zm_const ? f4_splat(pf.clo[2]) : val4(sm, rc)) : c;
            const float4 zp = DIM == 3 ? (zp_const ? f4_splat(pf.chi[2]) : val4(sp, rc)) : c;
            q = stencil_ref<DIM>(c, make_float4(xl, c.x, c.y, c.z), r4, ym, yp, zm, zp, ix2, iy2, iz2);
        } else {
        q.x = (xl + r4.x - 2.f * c.x) * ix2 + (ym.x + yp.x - 2.f * c.x) * iy2;
        q.y = (c.x + r4.y - 2.f * c.y) * ix2 + (ym.y + yp.y - 2.f * c.y) * iy2;
        q.z = (c.y + r4.z - 2.f * c.z) * ix2 + (ym.z + yp.z - 2.f * c.z) * iy2;
        q.w = (c.z + r4.w - 2.f * c.w) * ix2 + (ym.w + yp.w - 2.f * c.w) * iy2;
        if (DIM == 3) {
            const float4 zm = zm_const ? f4_splat(pf.clo[2]) : val4(sm, rc);
            const float4 zp = zp_const ? f4_splat(pf.chi[2]) : val4(sp, rc);
            q.x += (zm.x + zp.x - 2.f * c.x) * iz2;
            q.y += (zm.y + zp.y - 2.f * c.y) * iz2;
            q.z += (zm.z + zp.z - 2.f * c.z) * iz2;
            q.w += (zm.w + zp.w - 2.f * c.w) * iz2;
        }
        }
        float4 e0 = f4_splat(0.f), e1 = f4_splat(0.f), e2 = f4_splat(0.f);
        if (NE >= 1) e0 = *reinterpret_cast<const float4*>(sc + e0off + tg.eoff[k]);
        if (NE >= 2) e1 = *reinterpret_cast<const float4*>(sc + e1off + tg.eoff[k]);
        if (NE >= 3) e2 = *reinterpret_cast<const float4*>(sc + e1off + cfg.TY * pitch + tg.eoff[k]);
        if constexpr (RingTwoFields<Epi>::value) epi.k = k;
        epi(plane_off + tg.goff[k], c, q, nvalid, e0, e1, e2);
    }
}

// Branch-free variant for tiles that lie completely inside the grid in y, planes without constant z ghosts and
// non-constant x boundaries: every thread owns exactly G full groups.
// In 3-D a thread owns the same cells on every plane of a unit, so the (combined) values of planes z-1 and z are carried
// in registers from plane to plane (ZMarch) and only plane z+1 is read from shared memory.
struct ZMarch { float4 m[2], c[2]; bool have; };      // only used with <= 2 groups per thread (register budget)

template <int DIM, int NH, int NE, int G, bool MARCH, class Epi>
__device__ __forceinline__ void ring_compute_fast(const RingCfg& cfg, const DGrid& g, const ThreadGroups& tg,
                                                  const float* sm, const float* sc, const float* sp, float beta,
                                                  long long plane_off, Epi& epi, ZMarch& zs)
{
    const int pitch = cfg.pitch;
    const int h1 = (cfg.TY + 2) * pitch;
    const int e0off = NH * (cfg.TY + 2) * pitch;
    const int e1off = e0off + cfg.TY * pitch;
    const float ix2 = g.inv_dx2[0], iy2 = g.inv_dx2[1], iz2 = DIM == 3 ? g.inv_dx2[2] : 0.f;
    const float cc = 2.f * (ix2 + iy2 + iz2);
    const bool use1 = NH == 2 && beta != 0.f;
    auto val4 = [&](const float* s, int off) -> float4 {
        float4 a = *reinterpret_cast<const float4*>(s + off);
        if (use1) { const float4 o = *reinterpret_cast<const float4*>(s + h1 + off);
                    a.x = fmaf(beta, o.x, a.x); a.y = fmaf(beta, o.y, a.y); a.z = fmaf(beta, o.z, a.z); a.w = fmaf(beta, o.w, a.w); }
        return a;
    };
#pragma unroll
    for (int k = 0; k < G; ++k) {
        const int rc = tg.soff[k];
        constexpr bool MZ = MARCH && DIM == 3 && G <= 2;
        const float4 c = (MZ && zs.have) ? zs.c[k & 1] : val4(sc, rc);
        const float4 ym = val4(sc, rc - pitch);
        const float4 yp = val4(sc, rc + pitch);
        float xl = __shfl_up_sync(0xffffffffu, c.w, 1);
        float xr = __shfl_down_sync(0xffffffffu, c.x, 1);
        if (MARCH) {        // latency-bound single-CTA kernels: every lane loads (broadcast address for most), then selects
            float el = sc[tg.xlo[k]], er = sc[tg.xro[k]];
            if (use1) { el = fmaf(beta, sc[h1 + tg.xlo[k]], el); er = fmaf(beta, sc[h1 + tg.xro[k]], er); }
            xl = (tg.needl & (1u << k)) ? el : xl;
            xr = (tg.needr & (1u << k)) ? er : xr;
        } else {
            if (tg.needl & (1u << k)) { xl = sc[tg.xlo[k]]; if (use1) xl = fmaf(beta, sc[h1 + tg.xlo[k]], xl); }
            if (tg.needr & (1u << k)) { xr = sc[tg.xro[k]]; if (use1) xr = fmaf(beta, sc[h1 + tg.xro[k]], xr); }
        }
        float4 q;
        if constexpr (RingRefStencil<Epi>::value) {
            const float4 zm = DIM == 3 ? val4(sm, rc) : c, zp = DIM == 3 ? val4(sp, rc) : c;
            q = stencil_ref<DIM>(c, make_float4(xl, c.x, c.y, c.z), make_float4(c.y, c.z, c.w, xr), ym, yp, zm, zp, ix2, iy2, iz2);
        } else {
        q.x = fmaf(ix2, xl + c.y, fmaf(iy2, ym.x + yp.x, -cc * c.x));
        q.y = fmaf(ix2, c.x + c.z, fmaf(iy2, ym.y + yp.y, -cc * c.y));
        q.z = fmaf(ix2, c.y + c.w, fmaf(iy2, ym.z + yp.z, -cc * c.z));
        q.w = fmaf(ix2, c.z + xr, fmaf(iy2, ym.w + yp.w, -cc * c.w));
        if (DIM == 3) {
            const float4 zm = (MZ && zs.have) ? zs.m[k & 1] : val4(sm, rc);
            const float4 zp = val4(sp, rc);
            q.x = fmaf(iz2, zm.x + zp.x, q.x);
            q.y = fmaf(iz2, zm.y + zp.y, q.y);
            q.z = fmaf(iz2, zm.z + zp.z, q.z);
            q.w = fmaf(iz2, zm.w + zp.w, q.w);
            if (MZ) { zs.m[k & 1] = c; zs.c[k & 1] = zp; }
        }
        }
        float4 e0 = f4_splat(0.f), e1 = f4_splat(0.f), e2 = f4_splat(0.f);
        if (NE >= 1) e0 = *reinterpret_cast<const float4*>(sc + e0off + tg.eoff[k]);
        if (NE >= 2) e1 = *reinterpret_cast<const float4*>(sc + e1off + tg.eoff[k]);
        if (NE >= 3) e2 = *reinterpret_cast<const float4*>(sc + e1off + cfg.TY * pitch + tg.eoff[k]);
        if constexpr (RingTwoFields<Epi>::value) epi.k = k;
        epi(plane_off + tg.goff[k], c, q, 4, e0, e1, e2);
    }
    zs.have = MARCH && DIM == 3 && G <= 2;
}

template <bool GENERIC, int DIM, int NH, int NE, bool MARCH, CgOp OP, class Epi>
__device__ __forceinline__ void ring_compute_sel(const RingCfg& cfg, const DGrid& g, const DField& pf, const ThreadGroups& tg,
                                                 bool fast, const float* sm, const float* sc, const float* sp, float beta,
                                                 long long plane_off, int z, Epi& epi, ZMarch& zs, const CgOperator* od)
{
    if (cg_op_xslot(OP)) { zs.have = false; ring_compute<DIM, NH, NE, OP>(cfg, g, pf, tg, sm, sc, sp, beta, plane_off, z, epi, od); return; }
    if (!GENERIC || fast) {
        if (cfg.groups == 4) { ring_compute_fast<DIM, NH, NE, 4, MARCH>(cfg, g, tg, sm, sc, sp, beta, plane_off, epi, zs); return; }
        if (cfg.groups == 2) { ring_compute_fast<DIM, NH, NE, 2, MARCH>(cfg, g, tg, sm, sc, sp, beta, plane_off, epi, zs); return; }
        if (cfg.groups == 1) { ring_compute_fast<DIM, NH, NE, 1, MARCH>(cfg, g, tg, sm, sc, sp, beta, plane_off, epi, zs); return; }
    }
    zs.have = false;
    if (GENERIC) ring_compute<DIM, NH, NE>(cfg, g, pf, tg, sm, sc, sp, beta, plane_off, z, epi, od);
}

template <bool GENERIC, int DIM, int NH, int NE, bool MARCH, CgOp OP, class Epi>
__device__ __forceinline__ void ring_compute_any(const RingCfg& cfg, const DGrid& g, const DField& pf, const ThreadGroups& tg,
                                                 bool fast, const float* sm, const float* sc, const float* sp, float beta,
                                                 long long plane_off, int z, Epi& epi, ZMarch& zs, const CgOperator* od)
{
    if constexpr (RingTwoFields<Epi>::value) {
        static_assert(NH == 2 && NE == 0 && !MARCH && OP == CgOp::Poisson, "two fields: both haloed arrays, nothing else staged");
        const int h1 = (cfg.TY + 2) * cfg.pitch;
        epi.field = 0;
        ring_compute_sel<GENERIC, DIM, NH, NE, MARCH, OP>(cfg, g, pf, tg, fast, sm, sc, sp, 0.f, plane_off, z, epi, zs, od);
        epi.field = 1;
        ring_compute_sel<GENERIC, DIM, NH, NE, MARCH, OP>(cfg, g, pf, tg, fast, sm + h1, sc + h1, sp + h1, 0.f, plane_off, z, epi, zs, od);
    } else {
        ring_compute_sel<GENERIC, DIM, NH, NE, MARCH, OP>(cfg, g, pf, tg, fast, sm, sc, sp, beta, plane_off, z, epi, zs, od);
    }
}

// ---- one unit: producer streams its planes, consumers march through them --------------------------------------------------
struct RingUnit { int b, y0, z0, z1; };

template <int DIM>
__device__ __forceinline__ RingUnit ring_unit(const RingCfg& cfg, const DGrid& g, int unit)
{
    RingUnit u;
    u.b = unit / cfg.units_per_batch;
    const int r = unit - u.b * cfg.units_per_batch;
    if (DIM == 3) { const int zc = r / cfg.nyt, yt = r - zc * cfg.nyt; u.y0 = yt * cfg.TY; u.z0 = zc * cfg.ZC; u.z1 = min(g.n[2], u.z0 + cfg.ZC); }
    else { u.y0 = r * cfg.TY; u.z0 = 0; u.z1 = 1; }
    return u;
}

// k-th unit of this CTA; false when it has no more
template <int DIM>
__device__ __forceinline__ bool ring_next_unit(const RingCfg& cfg, const DGrid& g, int k, RingUnit& u)
{
    if (!cfg.split) {
        const int unit = blockIdx.x + k * gridDim.x;
        if (unit >= cfg.total_units) return false;
        u = ring_unit<DIM>(cfg, g, unit);
        return true;
    }
    if ((int)blockIdx.x < cfg.nyt) {
        if (k > 0) return false;
        u.b = 0; u.y0 = blockIdx.x * cfg.TY; u.z0 = 0; u.z1 = cfg.Zm;
        return true;
    }
    const int t = ((int)blockIdx.x - cfg.nyt) * cfg.split_t + k;
    if (k >= cfg.split_t || t >= cfg.nyt) return false;
    u.b = 0; u.y0 = t * cfg.TY; u.z0 = cfg.Zm; u.z1 = g.n[2];
    return true;
}

// consumers, 3-D: march through the planes of one unit.  G > 0: every plane takes the branch-free path with G groups.
template <bool GENERIC, int NH, int NE, bool MARCH, int G, CgOp OP, class Epi>
__device__ __forceinline__ void ring_consume_planes(Ring& rg, const RingCfg& cfg, const DGrid& g, const DField& pf, const ThreadGroups& tg,
                                                    bool tile_fast, float beta, long long plane_off, const RingUnit& u, Epi& epi,
                                                    const CgOperator* od)
{
    const int nz = u.z1 - u.z0;
    SlotIt a = rg.pos, bq = a; bq.next(cfg.R);
    SlotIt c2 = bq; c2.next(cfg.R);
    ZMarch zs; zs.have = false;
    ring_wait_full(rg, a); ring_wait_full(rg, bq);
    for (int zi = 0; zi < nz; ++zi) {
        const int z = u.z0 + zi;
        ring_wait_full(rg, c2);
        epi.set_plane(z, g.n[2]);
        if (G > 0) {
            ring_compute_fast<3, NH, NE, (G > 0 ? G : 1), MARCH>(cfg, g, tg, ring_ptr(rg, cfg, a), ring_ptr(rg, cfg, bq), ring_ptr(rg, cfg, c2),
                                                                 beta, plane_off, epi, zs);
        } else {
            const bool fast = tile_fast && !(z == 0 && pf.klo[2] == PHI_BC_CONST) && !(z == g.n[2] - 1 && pf.khi[2] == PHI_BC_CONST);
            ring_compute_any<GENERIC, 3, NH, NE, MARCH, OP>(cfg, g, pf, tg, fast, ring_ptr(rg, cfg, a), ring_ptr(rg, cfg, bq), ring_ptr(rg, cfg, c2),
                                                            beta, plane_off, z, epi, zs, od);
        }
        ring_release(rg, a);
        a = bq; bq = c2; c2.next(cfg.R);
        plane_off += pf.sz;
    }
    ring_release(rg, a); ring_release(rg, bq);
    rg.pos = c2;
}

// cg_op_xslot(OP): hsrc[NH] holds the operator's coefficients (the obstacle mask or the diffusivity) in the haloed slot after the
// NH value arrays; the diffusivity is read from batch entry kb (0 when one k serves every entry).  od: the operator's data.
template <bool GENERIC, int DIM, int NH, int NE, bool MARCH = true, CgOp OP = CgOp::Poisson, class Epi>
__device__ __forceinline__ void ring_process_unit(Ring& rg, const RingCfg& cfg, const DGrid& g, const DField& pf,
                                                  ThreadGroups& tg,
                                                  const float* const* hsrc, const float* const* esrc, float beta,
                                                  const RingUnit& u, Epi& epi, int kb = 0, const CgOperator* od = nullptr)
{
    constexpr bool XSLOT = cg_op_xslot(OP);
    const bool producer = (int)threadIdx.x >= cfg.consumers;
    if (producer) {
        const int nh = (NH == 2 && beta == 0.f && !RingTwoFields<Epi>::value) ? 1 : NH;   // first CG iteration: d' = r, old direction not read
        ProdUnit pu;
        prod_unit_setup<DIM, OP == CgOp::HelmholtzVarying>(pu, cfg, g, pf, ((1u << nh) - 1u) | (XSLOT ? (1u << NH) : 0u), NH + (XSLOT ? 1 : 0), NE, hsrc, esrc, u.b, u.y0, kb);
        if (DIM == 3) {
            const int nz = u.z1 - u.z0;
            for (int p = 0; p < nz + 2; ++p)
                ring_produce<DIM>(rg, cfg, pf, pu, u.z0 - 1 + p, p >= 1 && p <= nz);
        } else {
            ring_produce<DIM>(rg, cfg, pf, pu, 0, true);
        }
        return;
    }
    const int ny = g.n[1];
    const bool tile_fast = !XSLOT && (!GENERIC || tg.fast_ok && u.y0 + cfg.TY <= ny
                           && !(u.y0 == 0 && pf.klo[1] == PHI_BC_CONST) && !(u.y0 + cfg.TY == ny && pf.khi[1] == PHI_BC_CONST));
    if (GENERIC) groups_tile(tg, cfg, g, pf, u.y0);      // also needed on fast tiles: planes with constant z ghosts take the slow path
    long long plane_off = (long long)u.b * pf.sb + (long long)u.y0 * pf.sy + (DIM == 3 ? (long long)u.z0 * pf.sz : 0);
    if (DIM == 3) {
        // kernels that contain only the branch-free path pick the group count once per unit, not once per plane (two-field
        // epilogues go through ring_compute_any, which runs the consumer once per field)
        if constexpr (RingTwoFields<Epi>::value) ring_consume_planes<GENERIC, NH, NE, MARCH, 0, OP>(rg, cfg, g, pf, tg, tile_fast, beta, plane_off, u, epi, od);
        else if (!GENERIC && cfg.groups == 2) ring_consume_planes<GENERIC, NH, NE, MARCH, 2, OP>(rg, cfg, g, pf, tg, tile_fast, beta, plane_off, u, epi, od);
        else if (!GENERIC && cfg.groups == 4) ring_consume_planes<GENERIC, NH, NE, MARCH, 4, OP>(rg, cfg, g, pf, tg, tile_fast, beta, plane_off, u, epi, od);
        else if (!GENERIC) ring_consume_planes<GENERIC, NH, NE, MARCH, 1, OP>(rg, cfg, g, pf, tg, tile_fast, beta, plane_off, u, epi, od);
        else ring_consume_planes<GENERIC, NH, NE, MARCH, 0, OP>(rg, cfg, g, pf, tg, tile_fast, beta, plane_off, u, epi, od);
    } else {
        const SlotIt a = rg.pos;
        ring_wait_full(rg, a);
        const float* sc = ring_ptr(rg, cfg, a);
        epi.set_plane(-1, 0);
        ZMarch zs; zs.have = false;
        ring_compute_any<GENERIC, DIM, NH, NE, MARCH, OP>(cfg, g, pf, tg, tile_fast, sc, sc, sc, beta, plane_off, 0, epi, zs, od);
        ring_release(rg, a);
        rg.pos.next(cfg.R);
    }
}

// ---- epilogues (values of element-wise arrays arrive from shared memory) -------------------------------------------------
// Multi-GPU: an epilogue that updates a vector whose halo the neighbouring slab needs also stores the first / last owned
// plane into that neighbour's halo plane through a peer pointer (NVLink).  plo / phi are pre-offset so that the same
// element offset `off` addresses the right halo plane; zf says whether the current plane is the first (1) / last (2).
struct NoPeerHalo {            // single-GPU kernels: nothing to store, nothing to test
    int zf;
    __device__ __forceinline__ void set_plane(int, int) {}
    __device__ __forceinline__ void put4(long long, const float4&) const {}
    __device__ __forceinline__ void put1(long long, float) const {}
};

struct PeerHalo {
    float* plo; float* phi; int zf;
    __device__ __forceinline__ void set_plane(int z, int nz) { zf = ((z == 0 && plo) ? 1 : 0) | ((z == nz - 1 && phi) ? 2 : 0); }
    __device__ __forceinline__ void put4(long long off, const float4& v) const
    {
        if (zf & 1) *reinterpret_cast<float4*>(plo + off) = v;
        if (zf & 2) *reinterpret_cast<float4*>(phi + off) = v;
    }
    __device__ __forceinline__ void put1(long long off, float v) const
    {
        if (zf & 1) plo[off] = v;
        if (zf & 2) phi[off] = v;
    }
};

template <bool AXPY>
struct REpiLaplace {
    float* y; float coeff;
    __device__ __forceinline__ void set_plane(int, int) {}
    __device__ __forceinline__ void set_acc(const float4&) {}
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid, const float4&, const float4&, const float4&)
    {
        float4 o = q;
        if (AXPY) { o.x = c.x + coeff * q.x; o.y = c.y + coeff * q.y; o.z = c.z + coeff * q.z; o.w = c.w + coeff * q.w; }
        if (nvalid == 4) *reinterpret_cast<float4*>(y + off) = o;
        else for (int j = 0; j < nvalid; ++j) y[off + j] = f4_get(o, j);
    }
};

template <class PH>
struct REpiResidual0 {          // e0 = rhs
    float* r; float mean, offs; float acc0, acc1; PH ph; bool tol_from_y;   // CG-adaptive: tolerance relative to |y|^2
    float4 am = make_float4(1.f, 1.f, 1.f, 1.f);      // obstacles: balanced rhs = y - mean * accessible (fluid.py:205-209)
    __device__ __forceinline__ void set_plane(int z, int nz) { ph.set_plane(z, nz); }
    __device__ __forceinline__ void set_acc(const float4& a) { am = a; }
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid, const float4& y, const float4&, const float4&)
    {
        float4 rt = make_float4((y.x - mean * am.x) - q.x, (y.y - mean * am.y) - q.y, (y.z - mean * am.z) - q.z, (y.w - mean * am.w) - q.w);
        float4 rr = make_float4(rt.x - offs, rt.y - offs, rt.z - offs, rt.w - offs);
        if (tol_from_y) rt = make_float4(y.x - mean * am.x, y.y - mean * am.y, y.z - mean * am.z, y.w - mean * am.w);
        if (nvalid == 4) {
            *reinterpret_cast<float4*>(r + off) = rr;
            if (ph.zf) ph.put4(off, rr);
            acc0 += rr.x * rr.x + rr.y * rr.y + rr.z * rr.z + rr.w * rr.w;
            acc1 += rt.x * rt.x + rt.y * rt.y + rt.z * rt.z + rt.w * rt.w;
        } else for (int j = 0; j < nvalid; ++j) { const float a = f4_get(rr, j), t = f4_get(rt, j); r[off + j] = a; if (ph.zf) ph.put1(off + j, a); acc0 += a * a; acc1 += t * t; }
    }
};

// pass A: stores d', sums d'.Ad' and sum d'; ADAPT (CG-adaptive): the second sum is d'.r (e0 = r, element-wise), _linalg.py:113
template <class PH, bool ADAPT>
struct REpiPassA {
    __device__ __forceinline__ void set_acc(const float4&) {}
    float* dnew; float acc0, acc1; PH ph;
    __device__ __forceinline__ void set_plane(int z, int nz) { ph.set_plane(z, nz); }
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid, const float4& re, const float4&, const float4&)
    {
        if (nvalid == 4) {
            *reinterpret_cast<float4*>(dnew + off) = c;
            if (ph.zf) ph.put4(off, c);
            acc0 += c.x * q.x + c.y * q.y + c.z * q.z + c.w * q.w;
            if (ADAPT) acc1 += c.x * re.x + c.y * re.y + c.z * re.z + c.w * re.w;
            else acc1 += (c.x + c.y) + (c.z + c.w);
        } else for (int j = 0; j < nvalid; ++j) {
            const float v = f4_get(c, j); dnew[off + j] = v; if (ph.zf) ph.put1(off + j, v); acc0 += v * f4_get(q, j);
            if (ADAPT) acc1 += v * f4_get(re, j); else acc1 += v;
        }
    }
};

// The solution update is applied every second iteration only: x_{k+1} = x_{k-1} + alpha_{k-1} d_{k-1} + alpha_k d_k needs
// the previous direction (still intact in the other d buffer) but saves one read+write of x: 30 instead of 32 B/cell/it.
template <class PH, bool RQ = false>      // RQ (CG-adaptive): the second sum is r_new . q (_linalg.py:119)
struct REpiPassBr {
    __device__ __forceinline__ void set_acc(const float4&) {}             // odd iterations: e0 = r; x is left alone
    float* r; float alpha, offs; float acc0, acc1; PH ph;
    __device__ __forceinline__ void set_plane(int z, int nz) { ph.set_plane(z, nz); }
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid, const float4& re, const float4&, const float4&)
    {
        float4 rv = re;
        rv.x -= alpha * (q.x + offs); rv.y -= alpha * (q.y + offs); rv.z -= alpha * (q.z + offs); rv.w -= alpha * (q.w + offs);
        if (nvalid == 4) {
            *reinterpret_cast<float4*>(r + off) = rv;
            if (ph.zf) ph.put4(off, rv);
            acc0 += rv.x * rv.x + rv.y * rv.y + rv.z * rv.z + rv.w * rv.w;
            if (RQ) acc1 += rv.x * q.x + rv.y * q.y + rv.z * q.z + rv.w * q.w;
        } else for (int j = 0; j < nvalid; ++j) { const float t = f4_get(rv, j); r[off + j] = t; if (ph.zf) ph.put1(off + j, t); acc0 += t * t; if (RQ) acc1 += t * f4_get(q, j); }
    }
};

template <class PH, bool RQ = false>
struct REpiPassB {
    __device__ __forceinline__ void set_acc(const float4&) {}              // even iterations: e0 = x, e1 = r, e2 = previous direction
    float* x; float* r; float alpha, aprev, offs; float acc0, acc1; PH ph;
    __device__ __forceinline__ void set_plane(int z, int nz) { ph.set_plane(z, nz); }
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid, const float4& xe, const float4& re, const float4& dp)
    {
        float4 xv = xe, rv = re;
        xv.x += aprev * dp.x; xv.y += aprev * dp.y; xv.z += aprev * dp.z; xv.w += aprev * dp.w;
        xv.x += alpha * c.x; xv.y += alpha * c.y; xv.z += alpha * c.z; xv.w += alpha * c.w;
        rv.x -= alpha * (q.x + offs); rv.y -= alpha * (q.y + offs); rv.z -= alpha * (q.z + offs); rv.w -= alpha * (q.w + offs);
        if (nvalid == 4) {
            *reinterpret_cast<float4*>(x + off) = xv;
            *reinterpret_cast<float4*>(r + off) = rv;
            if (ph.zf) ph.put4(off, rv);
            acc0 += rv.x * rv.x + rv.y * rv.y + rv.z * rv.z + rv.w * rv.w;
            if (RQ) acc1 += rv.x * q.x + rv.y * q.y + rv.z * q.z + rv.w * q.w;
        } else for (int j = 0; j < nvalid; ++j) { x[off + j] = f4_get(xv, j); const float t = f4_get(rv, j); r[off + j] = t; if (ph.zf) ph.put1(off + j, t); acc0 += t * t; if (RQ) acc1 += t * f4_get(q, j); }
    }
};

// diffuse.implicit (N5): the stencil result q = L0 c of the value c becomes M c = c - a L0 c right before the wrapped epilogue,
// so the residual sweep and both CG passes (d.Md, r -= alpha Md) see the Helmholtz operator M = I - a L0.
template <class Epi>
struct REpiHelm {
    Epi& e; float a;
    __device__ __forceinline__ void set_plane(int z, int nz) { e.set_plane(z, nz); }
    __device__ __forceinline__ void set_acc(const float4& m) { e.set_acc(m); }
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid, const float4& e0, const float4& e1, const float4& e2)
    {
        const float4 m = make_float4(fmaf(-a, q.x, c.x), fmaf(-a, q.y, c.y), fmaf(-a, q.z, c.z), fmaf(-a, q.w, c.w));
        e(off, c, m, nvalid, e0, e1, e2);
    }
};

// diffuse.implicit with a varying diffusivity (N6): the HelmholtzVarying consumer delivers q = D0 c, the face-minimum stencil on
// the coefficients w = fl(ndt k), so that M c = c + q (sharpen = explicit(x, k, -dt), phi/physics/diffuse.py:90-95).  No rhs
// balancing: set_acc is not forwarded.
template <class Epi>
struct REpiVarHelm {
    Epi& e;
    __device__ __forceinline__ void set_plane(int z, int nz) { e.set_plane(z, nz); }
    __device__ __forceinline__ void set_acc(const float4&) {}
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid, const float4& e0, const float4& e1, const float4& e2)
    {
        const float4 m = make_float4(c.x + q.x, c.y + q.y, c.z + q.z, c.w + q.w);
        e(off, c, m, nvalid, e0, e1, e2);
    }
};

// ---- laplace -----------------------------------------------------------------------------------------------------------
template <int DIM, bool AXPY, bool GENERIC>
__global__ void __launch_bounds__(RING_THREADS, 2)
k_laplace_ring(DGrid g, DField f, RingCfg cfg, const float* __restrict__ x, float* __restrict__ y, float coeff)
{
    extern __shared__ __align__(128) unsigned char smem[];
    Ring rg;
    ring_init(rg, smem, cfg);
    ThreadGroups tg;
    groups_init(tg, cfg, g, f);
    const float* hsrc[2] = {x, nullptr};
    const float* esrc[2] = {nullptr, nullptr};
    REpiLaplace<AXPY> epi{y, coeff};
    for (int unit = blockIdx.x; unit < cfg.total_units; unit += gridDim.x) {
        const RingUnit u = ring_unit<DIM>(cfg, g, unit);
        ring_process_unit<GENERIC, DIM, 1, 0, false>(rg, cfg, g, f, tg, hsrc, esrc, 0.f, u, epi);
    }
}

// ---- CG ----------------------------------------------------------------------------------------------------------------
struct CgRingArgs {
    CgArgs a;
    RingCfg cfg;
    int ring_smem_offset;        // byte offset of the ring inside dynamic shared memory (after the CgShared block)
    CommDev cm;
    float* d2;                   // one-sweep CG: third direction buffer
    CgOperator op;               // the mask travels in a.acc
};

// The operator's one dispatch point in the CG: picks the batch entry of the diffusivity, turns the stencil result q into M c
// through the operator's epilogue wrapper and runs the unit.  hsrc[NH]: the obstacle mask or the diffusivity.  The Poisson sweeps
// call ring_process_unit directly: one more inlined call level changes nvcc's register allocation of those kernels.
template <int DIM, bool GENERIC, CgOp OP, int NH, int NE, class Epi>
__device__ __forceinline__ void cg_op_unit(Ring& rg, const CgRingArgs& A, ThreadGroups& tg, const float* const* hsrc,
                                           const float* const* esrc, float beta, const RingUnit& u, Epi& epi)
{
    if constexpr (OP == CgOp::Helmholtz) {
        REpiHelm<Epi> he{epi, A.op.amount};
        ring_process_unit<GENERIC, DIM, NH, NE, true, OP>(rg, A.cfg, A.a.g, A.a.pf, tg, hsrc, esrc, beta, u, he);
    } else if constexpr (OP == CgOp::HelmholtzVarying) {
        REpiVarHelm<Epi> he{epi};
        ring_process_unit<GENERIC, DIM, NH, NE, true, OP>(rg, A.cfg, A.a.g, A.a.pf, tg, hsrc, esrc, beta, u, he, A.op.kbcast ? 0 : u.b, &A.op);
    } else ring_process_unit<GENERIC, DIM, NH, NE, true, OP>(rg, A.cfg, A.a.g, A.a.pf, tg, hsrc, esrc, beta, u, epi);
}

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p)
{
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v)
{
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// All-reduce of the two per-batch sums across the ranks, executed inside the persistent kernel after the local
// reduction: block 0 writes this rank's sums into every rank's mailbox (NVLink peer stores) and raises a flag; every CTA
// of every rank waits for the n flags in its OWN mailbox and adds the n entries in rank order (bitwise identical
// everywhere).  Event `seq` uses mailbox half seq&1; a rank can be at most one event ahead of the slowest one.
__device__ __forceinline__ bool comm_allreduce(const CommDev& cm, const CgShared& sh, int batch, unsigned long long seq)
{
    const int par = (int)(seq & 1ull);
    const size_t stride = 2 * (size_t)CG_MAX_BATCH;
    if (blockIdx.x == 0) {
        for (int q = 0; q < cm.n; ++q) {
            double* dst = cm.mbox[q] + ((size_t)par * PHI_MAX_RANKS + cm.rank) * stride;
            for (int b = threadIdx.x; b < batch; b += blockDim.x) { dst[b] = sh.sum0[b]; dst[CG_MAX_BATCH + b] = sh.sum1[b]; }
        }
        __threadfence_system();
        __syncthreads();
        if ((int)threadIdx.x < cm.n) st_release_sys(cm.flag[threadIdx.x] + par * PHI_MAX_RANKS + cm.rank, seq);
    }
    bool ok = true;
    if ((int)threadIdx.x < cm.n) {
        const unsigned long long* f = cm.flag[cm.rank] + par * PHI_MAX_RANKS + threadIdx.x;
        const long long t0 = clock64();
        while (ld_acquire_sys(f) < seq) {
            if (clock64() - t0 > 40000000000ll) { ok = false; break; }        // ~20 s: a peer died; do not hang the GPU
        }
    }
    ok = __syncthreads_and(ok);
    const double* src = cm.mbox[cm.rank] + (size_t)par * PHI_MAX_RANKS * stride;
    for (int b = threadIdx.x; b < batch; b += blockDim.x) {
        double s0 = 0, s1 = 0;
        for (int q = 0; q < cm.n; ++q) {
            s0 += *(volatile const double*)(src + q * stride + b);
            s1 += *(volatile const double*)(src + q * stride + CG_MAX_BATCH + b);
        }
        sh.sum0[b] = s0; sh.sum1[b] = s1;
    }
    __syncthreads();
    return ok;
}

template <int DIM, class F>
__device__ __forceinline__ void ring_unit_cells(const RingCfg& cfg, const DGrid& g, const DField& pf, const ThreadGroups& tg,
                                                const RingUnit& u, F&& fn)
{
    // plain element-wise traversal of a unit by the consumer threads (sums, mean removal); no staging
    if ((int)threadIdx.x >= cfg.consumers) return;
    long long plane_off = (long long)u.b * pf.sb + (long long)u.y0 * pf.sy + (DIM == 3 ? (long long)u.z0 * pf.sz : 0);
    for (int z = u.z0; z < u.z1; ++z, plane_off += pf.sz)
#pragma unroll
        for (int k = 0; k < RING_G; ++k) {
            if (tg.j[k] < 0 || u.y0 + tg.j[k] >= g.n[1]) continue;
            const int x0 = tg.eoff[k] - tg.j[k] * cfg.pitch;
            fn(plane_off + tg.goff[k], min(4, g.n[0] - x0));
        }
}

// ---- one-sweep CG (pass F) -----------------------------------------------------------------------------------------------
// CG needs two sweeps per iteration only because beta = |r'|^2 / |r|^2 is a global sum that must be known before d' = r' + beta d
// can be formed.  Pass F computes that beta one step ahead instead.  Iteration k starts with r_k, d_k in memory and alpha_k,
// beta_{k+1} known, and in ONE sweep forms, per plane,
//   q_k = A d_k, r_{k+1} = r_k - alpha_k q_k, d_{k+1} = r_{k+1} + beta_{k+1} d_k   on the tile plus one halo line / plane,
//   q_{k+1} = A d_{k+1}                                                        on the tile,
// and sums d_{k+1}.q_{k+1}, |r_{k+1}|^2, r_{k+1}.q_{k+1}, |q_{k+1}|^2.  After the one grid barrier alpha_{k+1} = |r_{k+1}|^2 / d.q and
// beta_{k+2} = (|r_{k+1}|^2 - 2 alpha r.q + alpha^2 |q|^2) / |r_{k+1}|^2 (= |r_{k+2}|^2 / |r_{k+1}|^2 in exact arithmetic).  The
// stopping rule still uses the true |r_{k+1}|^2, and the look-ahead is rebuilt from it every iteration, so its rounding does not
// accumulate.  r is not stored: the previous pass formed d_k = r_k + beta_k d_{k-1}, so r_k = d_k - beta_k d_{k-1} is recovered in
// registers (its rounding error is relative to |d_k|, a small multiple of |r_k|, and does not grow with k; r_0 = d_0).
// x is read and written every third iteration: sweep k then applies alpha_{k-2} d_{k-2} + alpha_{k-1} d_{k-1} + alpha_k d_k.  d_{k-2}
// is not read back (other CTAs overwrite its buffer with d_{k+1}) but rebuilt from what is staged: d_{k-1} = r_{k-1} + beta_{k-1}
// d_{k-2} and r_{k-1} = r_k + alpha_{k-1} A d_{k-1}, with r_k = d_k - beta_k d_{k-1}, so the update is
//   x += (alpha_{k-1} + g (1 + beta_k)) d_{k-1} + (alpha_k - g) d_k - g alpha_{k-1} A d_{k-1},   g = alpha_{k-2} / beta_{k-1},
// with A d_{k-1} formed on the owned cells from the d_{k-1} stage.  Guard (fused_xmode): a sweep that starts owing one direction
// while its beta_k (the divisor of the next sweep) is below FUSED_XBETA_MIN applies alpha_{k-1} d_{k-1} + alpha_k d_k at once.  An
// entry that stops owing steps gets them after the loop.  Bytes per iteration: d_k, d_{k-1} read, d_{k+1} written (12 B/cell) + the
// x read and write every third iteration (8/3 B/cell) = 14.7 B/cell, against 30 for the two sweeps of k_cg_ring.
// Stage layout: d_k (TY+4 lines: halo 2 in y, because d_{k+1} is needed on the halo lines), d_{k-1} (TY+2 lines, not fetched in
// iteration 0).  x has no halo and is read only on owned cells of every third iteration, so it does not travel through the ring:
// consumers load it from global memory one plane ahead.  d_{k+1} of each plane goes to a triple-buffered shared tile (TY+2 lines)
// from which the q_{k+1} stencil takes its y and warp-edge x neighbours; consumers sync on a named barrier once per plane.
// Only for 3-D, the branch-free tiling, periodic y and z, one GPU, CG without matrix offset or obstacles (phi_launch_cg_ring).
#define FUSED_GI 2               // owned groups per consumer thread: TY * nx4 <= FUSED_GI * consumers
#define FUSED_GH 2               // groups per consumer thread on the two halo lines: 2 * nx4 <= FUSED_GH * consumers
#define FUSED_TILE_BUFS 3

// A thread's groups come in two kinds with fixed register slots: owned groups (lines 1 .. TY of the d_{k+1} tile) carry d_k, d_{k+1}
// and r_{k+1} from plane to plane, halo groups (lines 0 and TY+1) only d_k.  Group k of a kind is group threadIdx.x + k * consumers
// of that kind's lines; with nx4 % 32 == 0 (shfl_ok) every warp's 32 groups lie on one line, so validity is warp-uniform, and
// lane 0 / lane 31 are the only lanes whose x-1 / x+4 neighbour is not a shuffle away.
struct FusedGroups {
    int ti[FUSED_GI], th[FUSED_GH];   // jj * pitch + x0: offset in the d_{k+1} tile (line jj); in the d stage + pitch
    int ei[FUSED_GI], eh[FUSED_GH];   // tile offset of the x neighbour lane 0 (x-1) or lane 31 (x+4) reads; other lanes 0 (broadcast)
    int gi[FUSED_GI];                       // (jj - 1) * sy + x0: element offset of an owned group relative to (y0, x = 0) of the plane
    unsigned vi, vh;                  // bit k: owned / halo group k exists (warp-uniform)
};

__device__ __forceinline__ void fused_groups_init(FusedGroups& fg, const RingCfg& cfg, const DGrid& g, const DField& pf)
{
    const int lane = threadIdx.x & 31, nx = g.n[0], pitch = cfg.pitch, nx4 = cfg.nx4;
    // tile offset of the x neighbour this lane reads for the group at line jj, x0 (lane 0: x-1, lane 31: x+4, ghosts resolved)
    auto edge = [&](int jj, int x0) -> int {
        const int row = jj * pitch;
        if (lane == 0) return x0 == 0 ? (pf.klo[0] == PHI_BC_PERIODIC ? row + nx - 1 : row) : row + x0 - 1;
        if (lane == 31) return x0 + 4 >= nx ? (pf.khi[0] == PHI_BC_PERIODIC ? row : row + nx - 1) : row + x0 + 4;
        return 0;
    };
    fg.vi = fg.vh = 0;
#pragma unroll
    for (int k = 0; k < FUSED_GI; ++k) {
        const int ge = threadIdx.x + k * cfg.consumers;
        const int j = ge / nx4, x0 = (ge - j * nx4) * 4;
        if (j < cfg.TY) fg.vi |= 1u << k;
        fg.ti[k] = (j + 1) * pitch + x0;
        fg.ei[k] = edge(j + 1, x0);
        fg.gi[k] = j * (int)pf.sy + x0;
    }
#pragma unroll
    for (int k = 0; k < FUSED_GH; ++k) {
        const int ge = threadIdx.x + k * cfg.consumers;
        const int h = ge / nx4, x0 = (ge - h * nx4) * 4;
        const int jj = h == 0 ? 0 : cfg.TY + 1;
        if (h < 2) fg.vh |= 1u << k;
        fg.th[k] = jj * pitch + x0;
        fg.eh[k] = edge(jj, x0);
    }
}

// Producer of pass F: the haloed lines (hmask, tot_h) are d_k (TY+4 lines from y0-2), fetched on every plane of the unit; the
// element-wise ones (emask, tot_e) are d_{k-1} (TY+2 lines from y0-1), fetched on planes z0-1 .. z1.  A null source (d_{k-1} in
// iteration 0) is not fetched.  y and z are periodic, so every line and plane is a stored one and ring_produce<3> streams them.
__device__ __forceinline__ void prod_fused_setup(ProdUnit& pu, const RingCfg& cfg, const DField& pf, const float* d, const float* dprev,
                                                 int b, int y0)
{
    const int lane = threadIdx.x & 31, TY = cfg.TY;
    const uint32_t row_bytes = (uint32_t)cfg.pitch * 4u;
    const bool mergeable = pf.sy == cfg.pitch;
    const int rows[2] = {TY + 4, TY + 2};
    const int ylo[2] = {y0 - 2, y0 - 1};
    const float* src[2] = {d, dprev};
    int cnt[2] = {0, 0};
    pu.hmask = pu.emask = 0;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int line = lane + 32 * it;
        pu.yoff[it] = 0; pu.base[it] = nullptr; pu.dsto[it] = 0; pu.nbytes[it] = row_bytes;
        int key = -1, yv = 0, first = 0;
#pragma unroll
        for (int arr = 0; arr < 2; ++arr) {
            if (key < 0 && line >= first && line < first + rows[arr] && src[arr]) {
                int yy = ylo[arr] + (line - first); float cv;
                phi_resolve(yy, pf, 1, cv);                         // periodic in y: always a stored line
                pu.yoff[it] = (long long)b * pf.sb + (long long)yy * pf.sy;
                pu.base[it] = src[arr];
                pu.dsto[it] = 4u * (uint32_t)(line * cfg.pitch);
                key = arr; yv = yy;
            }
            first += rows[arr];
        }
        cnt[0] += key == 0; cnt[1] += key == 1;
        if (prod_merge_lines(key, yv, mergeable, row_bytes, pu.nbytes[it])) {
            if (key == 0) pu.hmask |= 1u << it; else pu.emask |= 1u << it;
        }
    }
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cnt[c] += __shfl_xor_sync(0xffffffffu, cnt[c], o);
    pu.tot_h = cnt[0]; pu.tot_e = cnt[1];
}

__device__ __forceinline__ float4 lds4(const float* s, int off) { return *reinterpret_cast<const float4*>(s + off); }
__device__ __forceinline__ float dot4(const float4& a, const float4& b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }

// 7-point stencil of the branch-free consumer (ring_compute_fast), same operation order
__device__ __forceinline__ float4 stencil7(const float4& c, float xl, float xr, const float4& ym, const float4& yp, const float4& zm, const float4& zp,
                                           float ix2, float iy2, float iz2, float cc)
{
    float4 q;
    q.x = fmaf(ix2, xl + c.y, fmaf(iy2, ym.x + yp.x, -cc * c.x));
    q.y = fmaf(ix2, c.x + c.z, fmaf(iy2, ym.y + yp.y, -cc * c.y));
    q.z = fmaf(ix2, c.y + c.w, fmaf(iy2, ym.z + yp.z, -cc * c.z));
    q.w = fmaf(ix2, c.z + xr, fmaf(iy2, ym.w + yp.w, -cc * c.w));
    q.x = fmaf(iz2, zm.x + zp.x, q.x);
    q.y = fmaf(iz2, zm.y + zp.y, q.y);
    q.z = fmaf(iz2, zm.z + zp.z, q.z);
    q.w = fmaf(iz2, zm.w + zp.w, q.w);
    return q;
}

struct FusedPass {
    const float* d; const float* dprev;                   // d_k, d_{k-1} (nullptr in iteration 0, where r_0 = d_0)
    float* dn; float* x;                                  // d_{k+1}, solution (x == nullptr: no x update this iteration)
    float alpha, aprev, beta, bprev;                      // alpha_k, alpha_{k-1}, beta_{k+1}, beta_k
    float xd, xdp, xq;                                    // three-direction sweep: x += xd d_k + xdp d_{k-1} + xq A d_{k-1}
};

// beta_{k-1} below this is not divided by: the x step of a sweep that starts owing one direction is then applied at once (two
// directions) instead of being deferred to a three-direction sweep.  The rebuilt d_{k-2} carries a rounding error of about
// eps / sqrt(beta_{k-1}) relative to |d_{k-2}|; 1e-2 bounds that at ten times the rounding of a stored direction.
#define FUSED_XBETA_MIN 1e-2f

// x update of a pass F sweep from the directions x owes at its start and beta_k (its bprev): 0 none (the step of d_k is deferred),
// 2 x += alpha_{k-1} d_{k-1} + alpha_k d_k, 3 the same + alpha_{k-2} d_{k-2}.  The same on every CTA: both inputs are per-entry
// state that every CTA reduces alike.
__device__ __forceinline__ int fused_xmode(int owed, float bprev)
{
    return owed == 2 ? 3 : (owed == 1 && !(fabsf(bprev) >= FUSED_XBETA_MIN)) ? 2 : 0;
}

// One unit of pass F: producer warp streams planes z0-2 .. z1+1, consumers march planes p = z0-1 .. z1 (d_{k+1} on the haloed
// region) and, one plane behind, q_{k+1} on the owned planes.  acc: d.q, |r|^2, r.q, |q|^2 of this thread.  X3: a three-direction
// sweep, which also forms A d_{k-1} on the owned planes; it releases the stage of each plane one plane later, so that d_{k-1} of
// plane p-1 is still staged (pass F runs with at least 4 stages).  That allocates better than carrying the plane in registers.
template <bool X3>
__device__ __forceinline__ void ring_fused_unit(Ring& rg, const RingCfg& cfg, const DGrid& g, const DField& pf, const FusedGroups& fg,
                                                const FusedPass& P, float* tile, const RingUnit& u, float (&acc)[4])
{
    const int nz = u.z1 - u.z0;
    if ((int)threadIdx.x >= cfg.consumers) {
        ProdUnit pu;
        prod_fused_setup(pu, cfg, pf, P.d, P.dprev, u.b, u.y0);
        for (int p = 0; p < nz + 4; ++p)
            ring_produce<3>(rg, cfg, pf, pu, u.z0 - 2 + p, p >= 1 && p <= nz + 2);
        return;
    }
    const int pitch = cfg.pitch, TY = cfg.TY;
    const int pb = (TY + 4) * pitch;
    const int tsz = (TY + 2) * pitch;
    const int lane = threadIdx.x & 31;
    const float ix2 = g.inv_dx2[0], iy2 = g.inv_dx2[1], iz2 = g.inv_dx2[2];
    const float cc = 2.f * (ix2 + iy2 + iz2);
    const float alpha = P.alpha, aprev = P.aprev, beta = P.beta, bprev = P.bprev;
    const bool has_prev = P.dprev != nullptr;
    long long plane_off = (long long)u.b * pf.sb + (long long)u.y0 * pf.sy + (long long)u.z0 * pf.sz - pf.sz;   // plane z0 - 1

    // d_{k+1} of the group at stage offset o (= pitch + tile offset) of plane p; c = d_k on p, zm = d_k on p-1, e = tile offset of
    // this lane's x neighbour.  rv: r_{k+1}, dp: d_{k-1}.
    auto dnew = [&](const float* sc, const float* sn, int o, int e, const float4& c, const float4& zm, float4& rv, float4& dp, float4& zp) {
        const float4 ym = lds4(sc, o - pitch), yp = lds4(sc, o + pitch);
        zp = lds4(sn, o);
        float xl = __shfl_up_sync(0xffffffffu, c.w, 1), xr = __shfl_down_sync(0xffffffffu, c.x, 1);
        const float ev = sc[pitch + e];
        if (lane == 0) xl = ev;
        if (lane == 31) xr = ev;
        const float4 q = stencil7(c, xl, xr, ym, yp, zm, zp, ix2, iy2, iz2, cc);
        rv = c; dp = f4_splat(0.f);                          // r_k = d_k - beta_k d_{k-1}; r_0 = d_0 (d_{k-1} slot not staged)
        if (has_prev) {
            dp = lds4(sc, pb + o - pitch);
            rv = make_float4(fmaf(-bprev, dp.x, c.x), fmaf(-bprev, dp.y, c.y), fmaf(-bprev, dp.z, c.z), fmaf(-bprev, dp.w, c.w));
        }
        rv.x = fmaf(-alpha, q.x, rv.x); rv.y = fmaf(-alpha, q.y, rv.y); rv.z = fmaf(-alpha, q.z, rv.z); rv.w = fmaf(-alpha, q.w, rv.w);
        return make_float4(fmaf(beta, c.x, rv.x), fmaf(beta, c.y, rv.y), fmaf(beta, c.z, rv.z), fmaf(beta, c.w, rv.w));
    };

    float4 dm[FUSED_GI], dc[FUSED_GI];           // d_k on planes p-1, p (owned groups)
    float4 hm[FUSED_GH], hc[FUSED_GH];           // the same on the halo groups
    float4 n2[FUSED_GI], n1[FUSED_GI];           // d_{k+1} on planes p-2, p-1
    float4 r1[FUSED_GI];                         // r_{k+1} on plane p-1
    float4 xv[FUSED_GI];                         // x on plane p (x-update iterations), loaded during plane p-1
    SlotIt cur = rg.pos, nxt = cur, prv = cur; nxt.next(cfg.R);   // prv (X3): the plane before cur, still held
    ring_wait_full(rg, cur); ring_wait_full(rg, nxt);
    {
        const float* s0 = ring_ptr(rg, cfg, cur);
        const float* s1 = ring_ptr(rg, cfg, nxt);
#pragma unroll
        for (int k = 0; k < FUSED_GI; ++k) {
            dm[k] = dc[k] = n2[k] = n1[k] = r1[k] = xv[k] = f4_splat(0.f);
            if (fg.vi & (1u << k)) { dm[k] = lds4(s0, pitch + fg.ti[k]); dc[k] = lds4(s1, pitch + fg.ti[k]); }
        }
#pragma unroll
        for (int k = 0; k < FUSED_GH; ++k) {
            hm[k] = hc[k] = f4_splat(0.f);
            if (fg.vh & (1u << k)) { hm[k] = lds4(s0, pitch + fg.th[k]); hc[k] = lds4(s1, pitch + fg.th[k]); }
        }
    }
    ring_release(rg, cur);
    cur = nxt; nxt.next(cfg.R);
    for (int i = 0; i < nz + 2; ++i) {               // plane p = z0 - 1 + i
        const bool own = i >= 1 && i <= nz;
        ring_wait_full(rg, nxt);
        const float* sc = ring_ptr(rg, cfg, cur);
        const float* sn = ring_ptr(rg, cfg, nxt);
        float* tw = tile + (i % FUSED_TILE_BUFS) * tsz;
#pragma unroll
        for (int k = 0; k < FUSED_GH; ++k) {
            if (!(fg.vh & (1u << k))) continue;
            float4 rv, dp, zp;
            const float4 dv = dnew(sc, sn, pitch + fg.th[k], fg.eh[k], hc[k], hm[k], rv, dp, zp);
            *reinterpret_cast<float4*>(tw + fg.th[k]) = dv;
            hm[k] = hc[k]; hc[k] = zp;
        }
        float4 n0[FUSED_GI], r0[FUSED_GI];
        float* const dnp = P.dn + plane_off;
        float* const xp = P.x ? P.x + plane_off : nullptr;
#pragma unroll
        for (int k = 0; k < FUSED_GI; ++k) {
            n0[k] = r0[k] = f4_splat(0.f);
            if (!(fg.vi & (1u << k))) continue;
            const float4 c = dc[k];
            float4 rv, dp, zp;
            const float4 dv = dnew(sc, sn, pitch + fg.ti[k], fg.ei[k], c, dm[k], rv, dp, zp);
            *reinterpret_cast<float4*>(tw + fg.ti[k]) = dv;
            if (own) {
                *reinterpret_cast<float4*>(dnp + fg.gi[k]) = dv;
                acc[1] += dot4(rv, rv);
                if constexpr (X3) {                          // A d_{k-1} from the d_{k-1} stages of planes p-1, p, p+1
                    const int od = pb + fg.ti[k];
                    const float4 ym = lds4(sc, od - pitch), yp = lds4(sc, od + pitch), zpp = lds4(sn, od);
                    float xl = __shfl_up_sync(0xffffffffu, dp.w, 1), xr = __shfl_down_sync(0xffffffffu, dp.x, 1);
                    const float ev = sc[pb + fg.ei[k]];
                    if (lane == 0) xl = ev;
                    if (lane == 31) xr = ev;
                    const float4 q = stencil7(dp, xl, xr, ym, yp, lds4(ring_ptr(rg, cfg, prv), od), zpp, ix2, iy2, iz2, cc);
                    float4 x4 = xv[k];
                    x4.x = fmaf(P.xq, q.x, fmaf(P.xdp, dp.x, fmaf(P.xd, c.x, x4.x)));
                    x4.y = fmaf(P.xq, q.y, fmaf(P.xdp, dp.y, fmaf(P.xd, c.y, x4.y)));
                    x4.z = fmaf(P.xq, q.z, fmaf(P.xdp, dp.z, fmaf(P.xd, c.z, x4.z)));
                    x4.w = fmaf(P.xq, q.w, fmaf(P.xdp, dp.w, fmaf(P.xd, c.w, x4.w)));
                    *reinterpret_cast<float4*>(xp + fg.gi[k]) = x4;
                } else if (xp) {                             // two directions: d_{k-1} is staged
                    float4 x4 = xv[k];
                    x4.x += aprev * dp.x; x4.y += aprev * dp.y; x4.z += aprev * dp.z; x4.w += aprev * dp.w;
                    x4.x += alpha * c.x; x4.y += alpha * c.y; x4.z += alpha * c.z; x4.w += alpha * c.w;
                    *reinterpret_cast<float4*>(xp + fg.gi[k]) = x4;
                }
            }
            n0[k] = dv; r0[k] = rv;
            dm[k] = c; dc[k] = zp;
        }
        if constexpr (X3) { if (i > 0) ring_release(rg, prv); prv = cur; }
        else ring_release(rg, cur);
        if (xp && i < nz) {                          // x of the next owned plane, in flight while q_{k+1} is formed
#pragma unroll
            for (int k = 0; k < FUSED_GI; ++k)
                if (fg.vi & (1u << k)) xv[k] = __ldcs(reinterpret_cast<const float4*>(xp + pf.sz + fg.gi[k]));
        }
        asm volatile("bar.sync 1, %0;" ::"r"(cfg.consumers) : "memory");      // the tile of plane p is complete
        if (i >= 2) {                                // q_{k+1} on plane p - 1 (owned: i - 1 in 1 .. nz)
            const float* tp = tile + ((i - 1) % FUSED_TILE_BUFS) * tsz;
#pragma unroll
            for (int k = 0; k < FUSED_GI; ++k) {
                if (!(fg.vi & (1u << k))) continue;
                const float4 c = n1[k];
                const float4 ym = lds4(tp, fg.ti[k] - pitch), yp = lds4(tp, fg.ti[k] + pitch);
                float xl = __shfl_up_sync(0xffffffffu, c.w, 1), xr = __shfl_down_sync(0xffffffffu, c.x, 1);
                const float ev = tp[fg.ei[k]];
                if (lane == 0) xl = ev;
                if (lane == 31) xr = ev;
                const float4 q = stencil7(c, xl, xr, ym, yp, n2[k], n0[k], ix2, iy2, iz2, cc);
                acc[0] += dot4(c, q);
                acc[2] += dot4(r1[k], q);
                acc[3] += dot4(q, q);
            }
        }
#pragma unroll
        for (int k = 0; k < FUSED_GI; ++k) { n2[k] = n1[k]; n1[k] = n0[k]; r1[k] = r0[k]; }
        cur = nxt; nxt.next(cfg.R);
        plane_off += pf.sz;
    }
    if constexpr (X3) ring_release(rg, prv);
    ring_release(rg, cur);
    rg.pos = nxt;
    asm volatile("bar.sync 1, %0;" ::"r"(cfg.consumers) : "memory");          // the next unit rewrites the tile
}

// prologue of the one-sweep solve: d_0 = r_0 is stored, sums d_0.A d_0 and |A d_0|^2 (alpha_0 and beta_1)
struct REpiFusedStart {
    float* d; float acc0, acc1;
    __device__ __forceinline__ void set_plane(int, int) {}
    __device__ __forceinline__ void set_acc(const float4&) {}
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int, const float4&, const float4&, const float4&)
    {
        *reinterpret_cast<float4*>(d + off) = c;
        acc0 += dot4(c, q);
        acc1 += dot4(q, q);
    }
};

// OP (cg_op_unit): Masked (N4): static obstacles - a.acc is the accessible mask, staged as an extra haloed array (always the
// GENERIC consumer).  Helmholtz (N5, diffuse.implicit): two-sweep CG on M = I - A.op.amount * L0 (REpiHelm); every batch entry is
// its own system.  HelmholtzVarying (N6): M = I + D0 of a varying diffusivity A.op.k (REpiVarHelm, the face-minimum consumer).
// FUSED: the one-sweep iteration (pass F above) replaces passes A and B.
template <int DIM, bool GENERIC, bool DIST, bool ADAPT, CgOp OP = CgOp::Poisson, bool FUSED = false>
__global__ void __launch_bounds__(RING_THREADS, 1)
k_cg_ring(CgRingArgs A)
{
    constexpr bool MASK = OP == CgOp::Masked;
    static_assert((OP != CgOp::Helmholtz && OP != CgOp::HelmholtzVarying) || (!DIST && !ADAPT && !FUSED),
                  "the Helmholtz operators run on the single-GPU two-sweep CG only");
    static_assert(!MASK || !ADAPT || (!DIST && !FUSED), "CG-adaptive with obstacles runs on the single-GPU two-sweep CG only");
    static_assert(!cg_op_xslot(OP) || GENERIC, "the face-minimum stencil runs on the generic consumer");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const CgArgs& a = A.a;
    const RingCfg& cfg = A.cfg;
    CgShared sh = cg_carve(smem_raw, a.g.batch);
    Ring rg;
    ring_init(rg, smem_raw + A.ring_smem_offset, cfg);
    cg::grid_group grid = cg::this_grid();
    const DGrid& g = a.g;
    const int batch = g.batch;
    const double cells = (double)g.n[0] * g.n[1] * g.n[2] * (A.cm.n > 1 ? A.cm.n : 1);   // global cell count (equal slabs)
    const float coffs = a.prm.matrix_offset;
    constexpr bool adaptive = ADAPT;                 // a.prm.method == PHI_SOLVER_CG_ADAPTIVE, chosen by the launcher
    int region = 0;
    ThreadGroups tg;
    groups_init(tg, cfg, g, a.pf);
    // the operator's haloed array after the CG vectors (cg_op_xslot): the obstacle mask or the diffusivity
    const float* const xsrc = OP == CgOp::Masked ? a.acc : (OP == CgOp::HelmholtzVarying ? A.op.k : nullptr);

    auto sweep = [&](const unsigned char* active, auto&& body) {
        int cur_b = cfg.split ? 0 : -1; float acc0 = 0.f, acc1 = 0.f;      // split mode: every CTA reports for the one batch entry
        RingUnit u;
        for (int k = 0; ring_next_unit<DIM>(cfg, g, k, u); ++k) {
            if (active && !active[u.b]) continue;
            if (u.b != cur_b) {
                if (cur_b >= 0) flush_partials(sh, a.partials, region, batch, cur_b, acc0, acc1);
                cur_b = u.b; acc0 = 0.f; acc1 = 0.f;
            }
            body(u, acc0, acc1);
        }
        if (cur_b >= 0) flush_partials(sh, a.partials, region, batch, cur_b, acc0, acc1);
    };
    const CommDev& cm = A.cm;
    unsigned long long seq = cm.n > 1 ? *cm.seq : 0ull;
    bool comm_ok = true;
    auto barrier_and_reduce = [&](const unsigned char* active) {
        fence_proxy_async();                       // generic-proxy stores of this pass -> later TMA (async proxy) loads
        if (cm.n > 1) __threadfence_system();      // halo planes stored into the neighbours' memory
        grid.sync();
        fence_proxy_async();
        reduce_partials(sh, a.partials, region, batch, cfg.split ? (int)gridDim.x : cfg.units_per_batch, active);
        region ^= 1;
        if (cm.n > 1) {
            comm_ok = comm_allreduce(cm, sh, batch, ++seq) && comm_ok;
            fence_proxy_async();
        }
    };
    const long long nzsz = (long long)g.n[2] * a.pf.sz;
    using PH = typename std::conditional<DIST, PeerHalo, NoPeerHalo>::type;
    auto peer_halo = [&](float* lo_arr, float* hi_arr) {
        PH ph;
        if constexpr (DIST) {
            ph.plo = cm.lower >= 0 ? lo_arr + nzsz : nullptr;
            ph.phi = cm.upper >= 0 ? hi_arr - nzsz : nullptr;
        }
        ph.zf = 0;
        return ph;
    };

    for (int b = threadIdx.x; b < batch; b += blockDim.x) { sh.mean[b] = 0.f; sh.offs[b] = 0.f; }
    __syncthreads();

    if (a.prm.balance_rhs || coffs != 0.f) {
        sweep(nullptr, [&](const RingUnit& u, float& acc0, float& acc1) {
            ring_unit_cells<DIM>(cfg, g, a.pf, tg, u, [&](long long off, int nvalid) {
                for (int j = 0; j < nvalid; ++j) { acc0 += a.rhs[off + j]; acc1 += MASK ? a.acc[off + j] : a.x[off + j]; }
            });
        });
        barrier_and_reduce(nullptr);
        for (int b = threadIdx.x; b < batch; b += blockDim.x) cg_balance<MASK>(sh, a.prm, b, cells);
        __syncthreads();
    }

    {   // r0 = y - (A + c 11^T) x0
        const float* hsrc[2] = {a.x, xsrc};
        const float* esrc[2] = {a.rhs, nullptr};
        sweep(nullptr, [&](const RingUnit& u, float& acc0, float& acc1) {
            REpiResidual0<PH> epi{a.r, sh.mean[u.b], sh.offs[u.b], 0.f, 0.f, peer_halo(cm.lo_r, cm.hi_r), adaptive};
            if constexpr (OP == CgOp::Poisson) ring_process_unit<GENERIC, DIM, 1, 1>(rg, cfg, g, a.pf, tg, hsrc, esrc, 0.f, u, epi);
            else cg_op_unit<DIM, GENERIC, OP, 1, 1>(rg, A, tg, hsrc, esrc, 0.f, u, epi);
            acc0 += epi.acc0; acc1 += epi.acc1;
        });
    }
    barrier_and_reduce(nullptr);
    cg_start(sh, a.prm, batch);

    // one-sweep CG: d_k lives in D[k % 3]: pass k reads d_k and d_{k-1} with halos while other CTAs write d_{k+1}.  a.r holds r_0 only.
    float* const D[3] = {a.d0, a.d1, A.d2};
    if constexpr (FUSED) {
        static_assert(DIM == 3 && !GENERIC && !DIST && !ADAPT && OP == CgOp::Poisson, "the one-sweep CG is 3-D, branch-free, single-GPU CG only");
        float* const tile = rg.stage0 + (size_t)cfg.R * cfg.stage_floats;
        FusedGroups fg;
        fused_groups_init(fg, cfg, g, a.pf);
        for (int b = threadIdx.x; b < batch; b += blockDim.x) sh.owed[b] = 0;
        __syncthreads();
        if (*sh.any_cont) {                          // d_0 = r_0; alpha_0 = |r_0|^2 / d_0.A d_0, beta_1 from |A d_0|^2
            const float* hsrc[2] = {a.r, nullptr};
            const float* esrc[2] = {nullptr, nullptr};
            sweep(sh.cont, [&](const RingUnit& u, float& acc0, float& acc1) {
                REpiFusedStart epi{D[0], 0.f, 0.f};
                ring_process_unit<false, 3, 1, 0, true>(rg, cfg, g, a.pf, tg, hsrc, esrc, 0.f, u, epi);
                acc0 += epi.acc0; acc1 += epi.acc1;
            });
            barrier_and_reduce(sh.cont);
            for (int b = threadIdx.x; b < batch; b += blockDim.x) {
                if (!sh.cont[b]) continue;
                const double dl = sh.delta[b], dq = sh.sum0[b];
                const float al = (dq != 0.0) ? (float)(dl / dq) : 0.f;
                const double nxt = dl - 2.0 * al * dq + (double)al * al * sh.sum1[b];
                sh.alpha[b] = al;
                sh.beta[b] = (dl != 0.0) ? (float)(nxt / dl) : 0.f;
                sh.bprev[b] = 0.f;
            }
            __syncthreads();
        }
        const int upb = cfg.split ? (int)gridDim.x : cfg.units_per_batch;
        int reg = 1;                                 // pass F sums go to partial slots 4 reg .. 4 reg + 3; the 2-sum sweeps used 0 .. 3
        for (int k = 0; *sh.any_cont; ++k) {
            FusedPass P;
            P.d = D[k % 3]; P.dprev = k > 0 ? D[(k + 2) % 3] : nullptr;
            P.dn = D[(k + 1) % 3];
            int cur_b = cfg.split ? 0 : -1;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            RingUnit u;
            for (int j = 0; ring_next_unit<3>(cfg, g, j, u); ++j) {
                if (!sh.cont[u.b]) continue;
                if (u.b != cur_b) {
                    if (cur_b >= 0) { flush_partials(sh, a.partials, 2 * reg, batch, cur_b, acc[0], acc[1]);
                                      flush_partials(sh, a.partials, 2 * reg + 1, batch, cur_b, acc[2], acc[3]); }
                    cur_b = u.b; acc[0] = acc[1] = acc[2] = acc[3] = 0.f;
                }
                P.alpha = sh.alpha[u.b]; P.aprev = sh.aprev[u.b]; P.beta = sh.beta[u.b]; P.bprev = sh.bprev[u.b];
                const int xm = fused_xmode(sh.owed[u.b], P.bprev);
                P.x = xm ? a.x : nullptr;
                if (xm == 3) {                       // d_{k-2} = ((1 + beta_k) d_{k-1} - d_k - alpha_{k-1} A d_{k-1}) / beta_{k-1}
                    const double gam = (double)sh.aprev2[u.b] / sh.bprev2[u.b];
                    P.xd = (float)(P.alpha - gam);
                    P.xdp = (float)(P.aprev + gam * (1.0 + P.bprev));
                    P.xq = (float)(-gam * P.aprev);
                    ring_fused_unit<true>(rg, cfg, g, a.pf, fg, P, tile, u, acc);
                } else ring_fused_unit<false>(rg, cfg, g, a.pf, fg, P, tile, u, acc);
            }
            if (cur_b >= 0) { flush_partials(sh, a.partials, 2 * reg, batch, cur_b, acc[0], acc[1]);
                              flush_partials(sh, a.partials, 2 * reg + 1, batch, cur_b, acc[2], acc[3]); }
            fence_proxy_async();
            grid.sync();
            fence_proxy_async();
            reduce_partials(sh, a.partials, 2 * reg, batch, upb, sh.cont);
            for (int b = threadIdx.x; b < batch; b += blockDim.x) {
                if (!sh.cont[b]) continue;
                const double dn = sh.sum1[b], dq = sh.sum0[b];
                const int ow = sh.owed[b];
                sh.owed[b] = fused_xmode(ow, sh.bprev[b]) ? 0 : ow + 1;
                if (cg_iteration_done(sh, a.prm, b, dn)) {       // an entry that stops keeps alpha_k, alpha_{k-1}: the steps it owes
                    sh.aprev2[b] = sh.aprev[b];
                    sh.bprev2[b] = sh.bprev[b];
                    sh.aprev[b] = sh.alpha[b];
                    sh.bprev[b] = sh.beta[b];
                    sh.alpha[b] = (dq != 0.0) ? (float)(dn / dq) : 0.f;
                }
            }
            __syncthreads();
            reduce_partials(sh, a.partials, 2 * reg + 1, batch, upb, sh.cont);
            for (int b = threadIdx.x; b < batch; b += blockDim.x) {
                if (!sh.cont[b]) continue;
                const double dn = sh.delta[b], al = sh.alpha[b];
                const double nxt = dn - 2.0 * al * sh.sum0[b] + al * al * sh.sum1[b];
                sh.beta[b] = (dn != 0.0) ? (float)(nxt / dn) : 0.f;
            }
            cg_count_running(sh, batch);
            reg ^= 1;
        }
        region = reg == 1 ? 2 : 0;                   // 2-sum slots that the last pass F did not use
    }

    // a.prm.method == PHI_SOLVER_CG_ADAPTIVE (_linalg.py:93-128) reuses both passes: pass A forms d' = r - c d (beta = -c) and
    // sums d'.Ad' and d'.r, pass B applies the step (d'.r)/(d'.Ad') and sums |r|^2 and r.Ad' for the next c.
    float* dold = a.d0; float* dnew = a.d1;
    float* lo_dnew = cm.lo_d1; float* hi_dnew = cm.hi_d1; float* lo_dold = cm.lo_d0; float* hi_dold = cm.hi_d0;
    bool x_pending = false;      // all running entries are at the same iteration, so one flag describes them all
    while (!FUSED && *sh.any_cont && comm_ok) {
        {   // pass A; CG-adaptive also sums d'.r (r once more, element-wise)
            const float* hsrc[3] = {a.r, dold, xsrc};
            const float* esrc[2] = {ADAPT ? a.r : nullptr, nullptr};
            sweep(sh.cont, [&](const RingUnit& u, float& acc0, float& acc1) {
                REpiPassA<PH, ADAPT> epi{dnew, 0.f, 0.f, peer_halo(lo_dnew, hi_dnew)};
                if constexpr (OP == CgOp::Poisson) ring_process_unit<GENERIC, DIM, 2, ADAPT ? 1 : 0>(rg, cfg, g, a.pf, tg, hsrc, esrc, sh.beta[u.b], u, epi);
                else cg_op_unit<DIM, GENERIC, OP, 2, ADAPT ? 1 : 0>(rg, A, tg, hsrc, esrc, sh.beta[u.b], u, epi);
                acc0 += epi.acc0; acc1 += epi.acc1;
            });
        }
        barrier_and_reduce(sh.cont);
        for (int b = threadIdx.x; b < batch; b += blockDim.x) {
            if (!sh.cont[b]) continue;
            sh.aprev[b] = sh.alpha[b];
            if (adaptive) {                          // step = (d.r) / (d.Ad), divide_no_nan (_linalg.py:113-114)
                const double dq = sh.sum0[b];
                sh.alpha[b] = (dq != 0.0) ? (float)(sh.sum1[b] / dq) : 0.f;
                sh.delta[b] = dq;                    // kept for the direction update after pass B
                sh.offs[b] = 0.f;
                continue;
            }
            const double S = sh.sum1[b];
            const double dq = sh.sum0[b] + (double)coffs * S * S;
            sh.alpha[b] = (dq != 0.0) ? (float)(sh.delta[b] / dq) : 0.f;
            sh.offs[b] = coffs * (float)S;
        }
        __syncthreads();
        if (!x_pending) {                           // pass B, odd iteration: r only, the x update is deferred
            const float* hsrc[2] = {dnew, xsrc};
            const float* esrc[3] = {a.r, nullptr, nullptr};
            sweep(sh.cont, [&](const RingUnit& u, float& acc0, float& acc1) {
                REpiPassBr<PH, ADAPT> epi{a.r, sh.alpha[u.b], ADAPT ? 0.f : sh.offs[u.b], 0.f, 0.f, peer_halo(cm.lo_r, cm.hi_r)};
                if constexpr (OP == CgOp::Poisson) ring_process_unit<GENERIC, DIM, 1, 1>(rg, cfg, g, a.pf, tg, hsrc, esrc, 0.f, u, epi);
                else cg_op_unit<DIM, GENERIC, OP, 1, 1>(rg, A, tg, hsrc, esrc, 0.f, u, epi);
                acc0 += epi.acc0; if (ADAPT) acc1 += epi.acc1;
            });
        } else {            // pass B, even iteration: x += alpha_prev d_prev + alpha d
            const float* hsrc[2] = {dnew, xsrc};
            const float* esrc[3] = {a.x, a.r, dold};
            sweep(sh.cont, [&](const RingUnit& u, float& acc0, float& acc1) {
                REpiPassB<PH, ADAPT> epi{a.x, a.r, sh.alpha[u.b], sh.aprev[u.b], ADAPT ? 0.f : sh.offs[u.b], 0.f, 0.f, peer_halo(cm.lo_r, cm.hi_r)};
                if constexpr (OP == CgOp::Poisson) ring_process_unit<GENERIC, DIM, 1, 3>(rg, cfg, g, a.pf, tg, hsrc, esrc, 0.f, u, epi);
                else cg_op_unit<DIM, GENERIC, OP, 1, 3>(rg, A, tg, hsrc, esrc, 0.f, u, epi);
                acc0 += epi.acc0; if (ADAPT) acc1 += epi.acc1;
            });
        }
        x_pending = !x_pending;
        barrier_and_reduce(sh.cont);
        for (int b = threadIdx.x; b < batch; b += blockDim.x) {
            if (!sh.cont[b]) continue;
            const double dn = sh.sum0[b];
            const double dprev = sh.delta[b];                 // CG: previous |r|^2;  CG-adaptive: d.Ad of this iteration
            // CG: d' = r + (|r'|^2 / |r|^2) d;  CG-adaptive: d' = r - ((r.Ad) / (d.Ad)) d  (_linalg.py:120)
            if (adaptive) sh.beta[b] = (dprev != 0.0) ? -(float)(sh.sum1[b] / dprev) : 0.f;
            else sh.beta[b] = (dprev != 0.0) ? (float)(dn / dprev) : 0.f;
            cg_iteration_done(sh, a.prm, b, dn);
        }
        cg_count_running(sh, batch);
        float* t = dold; dold = dnew; dnew = t;
        t = lo_dold; lo_dold = lo_dnew; lo_dnew = t;
        t = hi_dold; hi_dold = hi_dnew; hi_dnew = t;
    }

    // entries that stopped after an odd number of iterations (two sweeps) still owe x the step alpha d of their last iteration,
    // whose direction is in d1 (odd iterations write d1).  Pass F entries owe up to two steps (sh.owed): alpha_k d_k of their last
    // iteration k = it - 1, in D[(it - 1) % 3], and alpha_{k-1} d_{k-1}, in D[(it + 1) % 3].  Pass F tiles hold whole float4 groups;
    // keeping the partial-group path out of the one-sweep kernel keeps its register allocation (24 B more spill loads with it).
    RingUnit u;
    for (int k = 0; ring_next_unit<DIM>(cfg, g, k, u); ++k) {
        const int it = sh.iters[u.b];
        const int owe = FUSED ? sh.owed[u.b] : (it & 1);
        if (!owe) continue;
        const float al = sh.alpha[u.b];
        const float* dl = FUSED ? D[(it - 1) % 3] : a.d1;
        const float ap = sh.aprev[u.b];
        const float* dl2 = D[(it + 1) % 3];
        ring_unit_cells<DIM>(cfg, g, a.pf, tg, u, [&](long long off, int nvalid) {
            if (FUSED || nvalid == 4) {
                float4 xv = *reinterpret_cast<const float4*>(a.x + off);
                if (FUSED && owe == 2) {
                    const float4 dp = *reinterpret_cast<const float4*>(dl2 + off);
                    xv.x += ap * dp.x; xv.y += ap * dp.y; xv.z += ap * dp.z; xv.w += ap * dp.w;
                }
                const float4 dv = *reinterpret_cast<const float4*>(dl + off);
                xv.x += al * dv.x; xv.y += al * dv.y; xv.z += al * dv.z; xv.w += al * dv.w;
                *reinterpret_cast<float4*>(a.x + off) = xv;
            } else for (int j = 0; j < nvalid; ++j) a.x[off + j] += al * dl[off + j];
        });
    }

    if (a.prm.project_mean) {
        sweep(nullptr, [&](const RingUnit& u, float& acc0, float& acc1) {
            ring_unit_cells<DIM>(cfg, g, a.pf, tg, u, [&](long long off, int nvalid) {
                for (int j = 0; j < nvalid; ++j) { if (MASK) { acc0 += a.x[off + j] * a.acc[off + j]; acc1 += a.acc[off + j]; } else acc0 += a.x[off + j]; }
            });
        });
        barrier_and_reduce(nullptr);
        for (int k = 0; ring_next_unit<DIM>(cfg, g, k, u); ++k) {
            const float m = cg_projection_mean<MASK>(sh, u.b, cells);
            ring_unit_cells<DIM>(cfg, g, a.pf, tg, u, [&](long long off, int nvalid) {
                for (int j = 0; j < nvalid; ++j) a.x[off + j] -= MASK ? m * a.acc[off + j] : m;
            });
        }
    }

    if (cm.n > 1 && blockIdx.x == 0 && threadIdx.x == 0) *cm.seq = seq;
    cg_write_result(sh, a.result, batch, comm_ok);
}

// ---- host side ------------------------------------------------------------------------------------------------------------
static const int kSmemBudget = 227 * 1024;           // opt-in shared memory per block on H100
// cost of starting a unit, in plane loads (two halo planes are counted separately)
#define RING_UNIT_OVERHEAD 2.5

// lines staged per stage = lines_a * TY + lines_b; returns false when the grid lines are too long for a useful ring
// zhalo: halo planes a unit stages in z besides its own (2 for the stencil, 4 for the one-sweep CG)
static bool ring_config(const DGrid& g, int lines_a, int lines_b, int reserve_bytes, int min_stages, int max_stages,
                        int target_units, RingCfg* out, int consumers = RING_CONSUMERS, int zhalo = 2)
{
    RingCfg c;
    c.split = 0; c.Zm = 0; c.split_t = 0;
    c.consumers = consumers;
    c.pitch = g.cext[0]; c.nx4 = g.cext[0] / 4;
    const int row_bytes = c.pitch * 4;
    // smaller stages -> deeper ring; the extra y-halo lines are served by L2 (tools/sweep_ring.py sweeps TY and the ring depth)
    int ty = g.dim == 3 ? 4 : 16;
    if (g.dim == 3) {
        // a CTA wants >= 2048 cells per staged plane: the per-plane mbarrier bookkeeping is amortised over TY * nx cells.
        // 512 -> 4, 256 -> 8, ...
        const int want = 2048 / (g.cext[0] > 0 ? g.cext[0] : 1);
        ty = 1;
        while (ty * 2 <= want && ty < 16) ty *= 2;
        while (ty > 1 && ty / 2 >= g.n[1]) ty /= 2;
    }
    if (const char* e = getenv("PHICUDA_RING_TY")) { const int v = atoi(e); if (v >= 1 && v <= 32) ty = v; }     // tuning knob
    for (;; ty /= 2) {
        if (ty < 1) return false;
        if (ty * c.nx4 > RING_G * consumers) continue;                    // <= RING_G groups per thread
        if (lines_a * ty + lines_b > 128) continue;                            // <= 4 lines per producer lane
        const int stage_bytes = (lines_a * ty + lines_b) * row_bytes;
        const int r = (kSmemBudget - reserve_bytes - 128) / stage_bytes;
        if (const char* e = getenv("PHICUDA_RING_R")) { const int v = atoi(e); if (v >= min_stages && v < max_stages) max_stages = v; }   // tuning knob
        if (r >= min_stages) { c.TY = ty; c.R = r > max_stages ? max_stages : r; c.stage_floats = stage_bytes / 4; break; }
    }
    while (g.dim == 2 && c.TY > 1 && c.TY / 2 >= g.n[1]) c.TY /= 2;
    c.groups = (c.TY * c.nx4 + consumers - 1) / consumers;
    c.shfl_ok = (c.nx4 % 32 == 0) ? 1 : 0;
    if (g.dim == 3) {
        c.nyt = (g.n[1] + c.TY - 1) / c.TY;
        // z chunking: every unit pays two halo planes plus a pipeline start (~2.5 plane loads, RING_UNIT_OVERHEAD), and
        // the persistent grid of `ctas` CTAs is only fully busy when the unit count is close to a multiple of it -> maximise
        //   utilisation(units, ctas) / (1 + (2 + overhead)/ZC)
        const int ctas = target_units;
        double best = -1.0; int best_nzc = 1;
        const int max_nzc = g.n[2] >= 4 ? g.n[2] / 4 : 1;
        for (int nzc = 1; nzc <= max_nzc; ++nzc) {
            const int zc = (g.n[2] + nzc - 1) / nzc;
            if ((g.n[2] + zc - 1) / zc != nzc) continue;
            const long long units = (long long)c.nyt * nzc * g.batch;
            const long long rounds = (units + ctas - 1) / ctas;
            const double util = (double)units / (double)(rounds * ctas);
            const double score = util / (1.0 + (zhalo + RING_UNIT_OVERHEAD) / zc);
            if (score > best + 1e-9) { best = score; best_nzc = nzc; }
        }
        if (const char* e = getenv("PHICUDA_RING_NZC")) {                     // tuning knob
            const int v = atoi(e);
            if (v >= 1 && v <= g.n[2]) { const int zc = (g.n[2] + v - 1) / v; best_nzc = (g.n[2] + zc - 1) / zc; }
        }
        c.nzc = best_nzc; c.ZC = (g.n[2] + best_nzc - 1) / best_nzc;
        c.units_per_batch = c.nyt * c.nzc;
        c.total_units = c.units_per_batch * g.batch;
    } else {
        c.nyt = (g.n[1] + c.TY - 1) / c.TY; c.nzc = 1; c.ZC = 1;
        c.units_per_batch = c.nyt; c.total_units = c.nyt * g.batch;
    }
    *out = c;
    return true;
}

// every tile and plane of the grid qualifies for the branch-free consumer path
static bool ring_all_fast(const DGrid& g, const DField& f, const RingCfg& c)
{
    if (!c.shfl_ok || c.nx4 * 4 != g.n[0] || c.TY * c.nx4 != c.groups * c.consumers || g.n[1] % c.TY != 0) return false;
    for (int a = 0; a < g.dim; ++a) if (f.klo[a] == PHI_BC_CONST || f.khi[a] == PHI_BC_CONST) return false;
    return c.groups == 1 || c.groups == 2 || c.groups == 4;
}

static void note_ring_launch(int kernel, const RingCfg& c, bool generic, bool dist, bool adaptive, int grid, bool masked = false)
{
    PhiLaunchInfo li; memset(&li, 0, sizeof(li));
    li.kernel = kernel; li.generic = generic; li.dist = dist; li.adaptive = adaptive; li.masked = masked;
    li.TY = c.TY; li.stages = c.R; li.ZC = c.ZC; li.nzc = c.nzc; li.groups = c.groups; li.total_units = c.total_units; li.grid_ctas = grid; li.split = c.split;
    phi_note_launch(li);
}

// returns -100 when the ring does not apply (caller falls back to the register-marching kernel)
int phi_launch_laplace_ring(const DGrid& g, const DField& f, const float* x, float* y, float coeff, bool axpy, cudaStream_t s)
{
    RingCfg cfg;
    const int sms = phi_sm_count();
    // two CTAs per SM: each gets half of the shared memory
    if (!ring_config(g, 1, 2, kSmemBudget / 2 + 1024, g.dim == 3 ? 4 : 2, 6, sms * 2, &cfg)) return -100;
    const size_t smem = 128 + (size_t)cfg.R * cfg.stage_floats * 4;
    int grid = sms * 2;
    if (grid > cfg.total_units) grid = cfg.total_units;
    cudaError_t e;
    const bool generic = !ring_all_fast(g, f, cfg);
#define LAUNCH_LAP(D, AX, GEN) do { \
        e = cudaFuncSetAttribute(k_laplace_ring<D, AX, GEN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
        if (e == cudaSuccess) k_laplace_ring<D, AX, GEN><<<grid, RING_THREADS, smem, s>>>(g, f, cfg, x, y, coeff); } while (0)
#define LAUNCH_LAP2(D, AX) do { if (generic) LAUNCH_LAP(D, AX, true); else LAUNCH_LAP(D, AX, false); } while (0)
    if (g.dim == 3) { if (axpy) LAUNCH_LAP2(3, true); else LAUNCH_LAP2(3, false); }
    else            { if (axpy) LAUNCH_LAP2(2, true); else LAUNCH_LAP2(2, false); }
#undef LAUNCH_LAP2
#undef LAUNCH_LAP
    if (e != cudaSuccess) return (int)e;
    note_ring_launch(PHI_KERNEL_LAPLACE_RING, cfg, generic, false, false, grid);
    return (int)cudaGetLastError();
}

// ring of the two-sweep CG; lines staged per stage: pass B (even) = 1 haloed + 3 element-wise arrays = 4 TY + 2; with the
// operator's coefficients (cg_op_xslot: the obstacle mask or the diffusivity) as an extra haloed array 5 TY + 4 (pass A: 3 haloed = 3 TY + 6;
// pass A of CG-adaptive with obstacles: r, d, mask haloed + r element-wise = 4 TY + 6), reserved as 5 TY + 6
static bool cg_ring_config(const DGrid& g, CgOp op, int cgs, int target_units, RingCfg* c)
{
    const bool xslot = cg_op_xslot(op);
    return ring_config(g, xslot ? 5 : 4, xslot ? 6 : 2, cgs, g.dim == 3 ? (xslot ? 3 : 4) : 2, RING_MAX_STAGES, target_units, c);
}

// The k_cg_ring instantiation of an operator and solver variant; nullptr: the combination has none.
using CgRingKernel = void (*)(CgRingArgs);
static CgRingKernel cg_ring_kernel(CgOp op, int dim, bool generic, bool dist, bool adapt, bool fused)
{
    constexpr CgOp P = CgOp::Poisson, M = CgOp::Masked, H = CgOp::Helmholtz, V = CgOp::HelmholtzVarying;
    const bool d3 = dim == 3;
    switch (op) {
    case P:
        if (fused)              // the one-sweep CG: 3-D, branch-free, single-GPU CG
            return d3 && !generic && !dist && !adapt ? k_cg_ring<3, false, false, false, P, true> : nullptr;
        if (d3) return generic ? (dist ? (adapt ? k_cg_ring<3, true, true, true> : k_cg_ring<3, true, true, false>)
                                       : (adapt ? k_cg_ring<3, true, false, true> : k_cg_ring<3, true, false, false>))
                               : (dist ? (adapt ? k_cg_ring<3, false, true, true> : k_cg_ring<3, false, true, false>)
                                       : (adapt ? k_cg_ring<3, false, false, true> : k_cg_ring<3, false, false, false>));
        return generic ? (dist ? (adapt ? k_cg_ring<2, true, true, true> : k_cg_ring<2, true, true, false>)
                               : (adapt ? k_cg_ring<2, true, false, true> : k_cg_ring<2, true, false, false>))
                       : (dist ? (adapt ? k_cg_ring<2, false, true, true> : k_cg_ring<2, false, true, false>)
                               : (adapt ? k_cg_ring<2, false, false, true> : k_cg_ring<2, false, false, false>));
    case M:                     // the generic consumer; CG-adaptive on one GPU only
        if (!generic || fused || (adapt && dist)) return nullptr;
        if (adapt) return d3 ? k_cg_ring<3, true, false, true, M> : k_cg_ring<2, true, false, true, M>;
        return d3 ? (dist ? k_cg_ring<3, true, true, false, M> : k_cg_ring<3, true, false, false, M>)
                  : (dist ? k_cg_ring<2, true, true, false, M> : k_cg_ring<2, true, false, false, M>);
    case H:                     // the Helmholtz operators: single-GPU two-sweep CG
        if (dist || adapt || fused) return nullptr;
        return d3 ? (generic ? k_cg_ring<3, true, false, false, H> : k_cg_ring<3, false, false, false, H>)
                  : (generic ? k_cg_ring<2, true, false, false, H> : k_cg_ring<2, false, false, false, H>);
    case V:
        if (dist || adapt || fused || !generic) return nullptr;
        return d3 ? k_cg_ring<3, true, false, false, V> : k_cg_ring<2, true, false, false, V>;
    }
    return nullptr;
}

int phi_launch_cg_ring(const CgLaunch& l, const CommDev* cm, cudaStream_t s)
{
    const DGrid& g = l.g;
    const CgOp op = l.op.kind;
    if (g.batch > CG_MAX_BATCH) return -100;
    if (op == CgOp::Masked && l.prm.matrix_offset != 0.f) return -100;
    const bool xslot = cg_op_xslot(op);
    CgRingArgs A;
    const int cgs = (int)((cg_smem_bytes(g.batch) + 127) / 128 * 128);
    const int sms = phi_sm_count();
    if (!cg_ring_config(g, op, cgs, sms, &A.cfg)) return -100;
    // pass A of CG-adaptive stages 2 haloed + 1 element-wise array = 3 TY + 4 lines: one line more than 4 TY + 2 at TY = 1 (with
    // obstacles 4 TY + 6 lines, inside the 5 TY + 6 of cg_ring_config)
    if (l.prm.method == PHI_SOLVER_CG_ADAPTIVE && !xslot && A.cfg.TY == 1
        && !ring_config(g, 4, 3, cgs, g.dim == 3 ? 4 : 2, RING_MAX_STAGES, sms, &A.cfg)) return -100;
    A.ring_smem_offset = cgs;
    int per_sm = 0;
    cudaError_t e;
    const bool generic = xslot || !ring_all_fast(g, l.pf, A.cfg);
    const bool dist = cm && cm->n > 1;
    const bool adapt = l.prm.method == PHI_SOLVER_CG_ADAPTIVE;
    // one-sweep CG (pass F): 3-D, branch-free tiling, periodic y and z, one GPU, plain CG without matrix offset or obstacles.
    // PHICUDA_CG_PASSES=2 forces the two-sweep kernel (A/B timing, tools/cg_passes_bench.py).
    bool fused = false;
    size_t tile_bytes = 0;
    {
        const char* e = getenv("PHICUDA_CG_PASSES");
        const DField& pf = l.pf;
        if (!(e && atoi(e) == 2) && g.dim == 3 && !generic && !dist && !adapt && op == CgOp::Poisson && l.prm.matrix_offset == 0.f
            && pf.klo[1] == PHI_BC_PERIODIC && pf.khi[1] == PHI_BC_PERIODIC && pf.klo[2] == PHI_BC_PERIODIC && pf.khi[2] == PHI_BC_PERIODIC) {
            // stage = d_k (TY+4) + d_{k-1} (TY+2) lines; the tile is chosen with TY more lines per stage (3 TY + 6), which keeps the
            // tiling pass F had while it staged x (lines up to 1024 cells at TY 1).  The d_{k+1} tile is reserved at the largest TY
            // ring_config may pick.
            RingCfg fc;
            if (ring_config(g, 3, 6, cgs, 4, RING_MAX_STAGES, sms, &fc, RING_CONSUMERS, 4)
                && ring_config(g, 3, 6, cgs + FUSED_TILE_BUFS * (fc.TY + 2) * fc.pitch * 4, 4, RING_MAX_STAGES, sms, &fc, RING_CONSUMERS, 4)
                && ring_all_fast(g, pf, fc) && fc.TY * fc.nx4 <= FUSED_GI * fc.consumers && 2 * fc.nx4 <= FUSED_GH * fc.consumers) {
                fused = true;
                A.cfg = fc;
                tile_bytes = (size_t)FUSED_TILE_BUFS * (fc.TY + 2) * fc.pitch * 4;
            }
        }
    }
    const int threads = RING_THREADS;
    const size_t smem = (size_t)cgs + 128 + (size_t)A.cfg.R * A.cfg.stage_floats * 4 + tile_bytes;
    const void* fn = (const void*)cg_ring_kernel(op, g.dim, generic, dist, adapt, fused);
    if (!fn) return -100;
    e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, threads, smem);
    if (e != cudaSuccess || per_sm < 1) return -100;
    int grid = sms * per_sm;
    // tail split (see RingCfg): compare the planes the busiest CTA stages per pass, default decomposition vs split
    A.cfg.split = 0; A.cfg.Zm = 0; A.cfg.split_t = 0;
    {
        const char* e = getenv("PHICUDA_RING_SPLIT");                       // tuning knob: 0 = never, 1 = whenever possible
        const int force = e ? atoi(e) : -1;
        const int nyt = A.cfg.nyt, nz = g.n[2];
        const int zh = fused ? 4 : 2;                                         // z halo planes staged per unit
        if (g.dim == 3 && g.batch == 1 && force != 0 && grid <= CG_MAX_GRID && nyt < grid && nz >= 8) {
            const int spare = grid - nyt, T = (nyt + spare - 1) / spare;
            int best_zm = 0; double best = 1e30;
            for (int zm = 4; zm <= nz - 1; ++zm) {
                const double main_c = zm + zh + RING_UNIT_OVERHEAD, tail_c = T * (nz - zm + zh + RING_UNIT_OVERHEAD);
                const double cost = main_c > tail_c ? main_c : tail_c;
                if (cost < best) { best = cost; best_zm = zm; }
            }
            const long long rounds = ((long long)A.cfg.total_units + grid - 1) / grid;
            const double dflt = rounds * (A.cfg.ZC + zh + RING_UNIT_OVERHEAD);
            if (best_zm > 0 && (force == 1 || best < dflt * 0.97)) {
                A.cfg.split = 1; A.cfg.Zm = best_zm; A.cfg.split_t = T;
                A.cfg.nzc = 2; A.cfg.ZC = best_zm; A.cfg.units_per_batch = A.cfg.total_units = 2 * nyt;
            }
        }
    }
    if (!A.cfg.split && grid > A.cfg.total_units) grid = A.cfg.total_units;
    if (grid > CG_MAX_GRID) grid = CG_MAX_GRID;
    const CgWorkspace w = phi_cg_workspace(g, l.workspace);
    CgArgs& a = A.a;
    a.g = g; a.pf = l.pf; a.um = UnitMap();
    a.rhs = l.rhs; a.x = l.x; a.acc = l.op.mask;
    a.r = w.r; a.d0 = w.d0; a.d1 = w.d1; a.partials = w.partials;
    A.d2 = w.d2;
    A.op = l.op;
    a.result = l.result; a.prm = l.prm;
    if (cm) A.cm = *cm; else { memset(&A.cm, 0, sizeof(A.cm)); A.cm.n = 1; A.cm.lower = A.cm.upper = -1; }
    void* args[] = {&A};
    e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(threads), args, smem, s);
    if (e != cudaSuccess) { phi_set_error("cg ring: cooperative launch failed: %s", cudaGetErrorString(e)); return (int)e; }
    note_ring_launch(PHI_KERNEL_CG_RING, A.cfg, generic, dist, adapt, grid, op == CgOp::Masked);
    phi_note_cg_passes(fused ? 1 : 2);
    phi_note_cg_operator(op == CgOp::HelmholtzVarying ? PHI_CG_OP_HELMHOLTZ_VARYING : (op == CgOp::Helmholtz ? PHI_CG_OP_HELMHOLTZ : PHI_CG_OP_POISSON));
    return 0;
}

// ---- N5 diffuse.implicit --------------------------------------------------------------------------------------------------
// The reference solves sharpen(x) = x - a L_bc(x) = y as the affine system M x = y - bias with M = I - a L0 (L0: L_bc with every
// constant ghost 0) and bias = sharpen(0) = -a L_bc(0) (PhiML/phiml/math/_optimize.py:622, 645).  The bias is non-zero only in
// cells next to a constant side with a non-zero value; this pass forms y' = y - bias = y + a L_bc(0) for every entry, with the
// constants of the entry's component (entry b is component b % C).
struct HelmConsts { float clo[3][3], chi[3][3]; };      // [component][axis]

__global__ void k_helm_bias(DGrid g, DField f, int C, float amount, HelmConsts hc, const float* __restrict__ y, float* __restrict__ out)
{
    const long long plane = (long long)g.n[0] * g.n[1], cells = plane * g.n[2], total = cells * g.batch;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / cells);
        const long long r = i - b * cells;
        const int z = (int)(r / plane), yy = (int)((r - z * plane) / g.n[0]), x = (int)(r - z * plane - (long long)yy * g.n[0]);
        const int idx[3] = {x, yy, z};
        const int c = b % C;
        float lap = 0.f;                        // L_bc(0): sum over axes of (lower ghost + upper ghost) / dx^2
        for (int ax = 0; ax < g.dim; ++ax) {
            float gs = 0.f;
            if (idx[ax] == 0 && f.klo[ax] == PHI_BC_CONST) gs += hc.clo[c][ax];
            if (idx[ax] == g.n[ax] - 1 && f.khi[ax] == PHI_BC_CONST) gs += hc.chi[c][ax];
            lap += gs * g.inv_dx2[ax];
        }
        const long long off = b * f.sb + z * f.sz + (long long)yy * f.sy + x;
        out[off] = fmaf(amount, lap, y[off]);
    }
}

// N6, varying diffusivity: bias = sharpen(0) = sum over constant sides of f_b c / dx^2 with f_b = min(fl(ndt k_edge), c) (the
// coefficient ghost of a constant side is c itself); this pass forms y' = y - bias.  k: entry b, or entry 0 when kbcast.
__global__ void k_helm_bias_var(DGrid g, DField f, float ndt, HelmConsts hc, const float* __restrict__ k, int kbcast,
                                const float* __restrict__ y, float* __restrict__ out)
{
    const long long plane = (long long)g.n[0] * g.n[1], cells = plane * g.n[2], total = cells * g.batch;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / cells);
        const long long r = i - b * cells;
        const int z = (int)(r / plane), yy = (int)((r - z * plane) / g.n[0]), x = (int)(r - z * plane - (long long)yy * g.n[0]);
        const int idx[3] = {x, yy, z};
        const long long cell = z * f.sz + (long long)yy * f.sy + x;
        const float w = __fmul_rn(ndt, k[(kbcast ? 0 : b) * f.sb + cell]);
        float bias = 0.f;
        for (int ax = 0; ax < g.dim; ++ax) {
            float s = 0.f;
            if (idx[ax] == 0 && f.klo[ax] == PHI_BC_CONST) { const float c = hc.clo[0][ax]; s += fminf(w, c) * c; }
            if (idx[ax] == g.n[ax] - 1 && f.khi[ax] == PHI_BC_CONST) { const float c = hc.chi[0][ax]; s += fminf(w, c) * c; }
            bias += s * g.inv_dx2[ax];
        }
        const long long off = b * f.sb + cell;
        out[off] = y[off] - bias;
    }
}

// the grid fits the persistent ring CG with operator op (host-only test, no CUDA call)
bool phi_cg_ring_fits(const DGrid& g, CgOp op)
{
    if (g.batch > CG_MAX_BATCH || g.halo != 0) return false;
    RingCfg c;
    return cg_ring_config(g, op, (int)((cg_smem_bytes(g.batch) + 127) / 128 * 128), 1, &c);
}

// the widest grid line (cells, a multiple of 4, at most g's own) for which fits(h) holds, h being g with that line; 0: none
template <class F>
static int ring_max_width(const DGrid& g, F&& fits)
{
    for (int w = g.cext[0] < 4096 ? g.cext[0] / 4 * 4 : 4096; w >= 4; w -= 4) {       // ty * nx4 <= RING_G * 256: no line beyond 4096
        DGrid h = g; h.n[0] = w; h.cext[0] = w;
        if (fits(h)) return w;
    }
    return 0;
}

// the widest grid line (cells, a multiple of 4) that phi_launch_cg_ring takes for g's other extents and batch with operator op and
// solver method adapt; 0: none (host-only, no CUDA call; for the error message of a refused solve)
int phi_cg_ring_max_width(const DGrid& g, CgOp op, bool adapt)
{
    if (g.batch > CG_MAX_BATCH || g.halo != 0) return 0;
    const int cgs = (int)((cg_smem_bytes(g.batch) + 127) / 128 * 128);
    return ring_max_width(g, [&](const DGrid& h) {
        RingCfg c;
        if (!cg_ring_config(h, op, cgs, 1, &c)) return false;
        return !(adapt && !cg_op_xslot(op) && c.TY == 1) || ring_config(h, 4, 3, cgs, h.dim == 3 ? 4 : 2, RING_MAX_STAGES, 1, &c);
    });
}

// l.pf: boundary kinds with zeroed constants (the value ghosts of L0 / D0); cf[0 .. C-1]: the boundary with its constants of component
// c = entry % C (bias; with a varying diffusivity also the coefficient ghosts l.op.kclo / kchi).  y' = y - bias goes to the
// workspace's d2 (phi_cg_workspace).  The varying pre-pass runs whenever a constant is non-zero - also for dt = 0, where
// f_b = min(-0, c) = c for c < 0.  -100: the grid does not fit.
int phi_launch_diffuse_implicit(const CgLaunch& l, int C, const DField* cf, cudaStream_t s)
{
    const DGrid& g = l.g;
    const bool varying = l.op.kind == CgOp::HelmholtzVarying;
    HelmConsts hc;
    bool bias = false;
    for (int c = 0; c < 3; ++c)
        for (int ax = 0; ax < 3; ++ax) {
            const bool used = c < C && ax < g.dim;
            hc.clo[c][ax] = used && cf[c].klo[ax] == PHI_BC_CONST ? cf[c].clo[ax] : 0.f;
            hc.chi[c][ax] = used && cf[c].khi[ax] == PHI_BC_CONST ? cf[c].chi[ax] : 0.f;
            bias = bias || hc.clo[c][ax] != 0.f || hc.chi[c][ax] != 0.f;
        }
    CgLaunch m = l;
    if (bias && (varying || l.op.amount != 0.f)) {
        float* yb = phi_cg_workspace(g, l.workspace).d2;
        const long long total = (long long)g.n[0] * g.n[1] * g.n[2] * g.batch;
        const long long want = (total + 255) / 256, cap = (long long)phi_sm_count() * 8;
        const int blocks = (int)(want < cap ? want : cap);
        if (varying) k_helm_bias_var<<<blocks, 256, 0, s>>>(g, l.pf, l.op.ndt, hc, l.op.k, l.op.kbcast, l.rhs, yb);
        else k_helm_bias<<<blocks, 256, 0, s>>>(g, l.pf, C, l.op.amount, hc, l.rhs, yb);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
        m.rhs = yb;
    }
    return phi_launch_cg_ring(m, nullptr, s);
}

// ---- persistent steppers (N7, N8): every substep of a call in one cooperative launch ------------------------------------------
// Between two substeps: the generic-proxy stores of one substep must be visible to the TMA (async proxy) loads of the next one, whose
// halo lines other CTAs wrote - the sequence k_cg_ring uses between passes.
__device__ __forceinline__ void step_grid_sync(cg::grid_group& grid)
{
    fence_proxy_async();
    grid.sync();
    fence_proxy_async();
}

// d0 = s0 and, with TWO, d1 = s1 on every cell of this CTA's units
template <int DIM, bool TWO>
__device__ __forceinline__ void step_copy_units(const RingCfg& cfg, const DGrid& g, const DField& f, const ThreadGroups& tg,
                                                float* d0, const float* s0, float* d1 = nullptr, const float* s1 = nullptr)
{
    for (int unit = blockIdx.x; unit < cfg.total_units; unit += gridDim.x)
        ring_unit_cells<DIM>(cfg, g, f, tg, ring_unit<DIM>(cfg, g, unit), [&](long long off, int nvalid) {
            for (int j = 0; j < nvalid; ++j) { d0[off + j] = s0[off + j]; if (TWO) d1[off + j] = s1[off + j]; }
        });
}

// ---- N7 reaction-diffusion (Gray-Scott, the Reaction_Diffusion notebook) ------------------------------------------------------
// One substep of the notebook's step, per cell, in the reference's operation order (field arithmetic, one rounding per operation):
//   uvv = u * v**2;  su = du * laplace(u) - uvv + f * (1 - u);  sv = dv * laplace(v) + uvv - (f + k) * v;  u' = u + dt su, v' = v + dt sv
// u and v are staged as the two haloed arrays of one stage (same boundary kinds, zero constants: the ghosts of both fields are
// fixed points of the reference's extrapolation arithmetic).  The consumer runs once per field (RingTwoFields): field 0 keeps u and
// laplace(u) of each of the thread's groups in registers, field 1 forms both updates.  16 B/cell per substep.
__device__ __forceinline__ void rd_cell(const RdParams& p, float u, float lu, float v, float lv, float& uo, float& vo)
{
    const float uvv = __fmul_rn(u, __fmul_rn(v, v));
    const float su = __fadd_rn(__fsub_rn(__fmul_rn(p.du, lu), uvv), __fmul_rn(p.f, __fsub_rn(1.f, u)));
    const float sv = __fsub_rn(__fadd_rn(__fmul_rn(p.dv, lv), uvv), __fmul_rn(p.fk, v));
    uo = __fadd_rn(u, __fmul_rn(p.dt, su));
    vo = __fadd_rn(v, __fmul_rn(p.dt, sv));
}

struct REpiReactionDiffusion {
    static constexpr bool kTwoFields = true;
    float* un; float* vn; RdParams p;
    int field, k;                                  // set by the consumer before each call
    float4 cu[RING_G], lu[RING_G];                 // u and laplace(u) of group k, field 0 -> field 1
    __device__ __forceinline__ void set_plane(int, int) {}
    __device__ __forceinline__ void set_acc(const float4&) {}
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid, const float4&, const float4&, const float4&)
    {
        if (field == 0) { cu[k] = c; lu[k] = q; return; }
        float4 a, b;
        rd_cell(p, cu[k].x, lu[k].x, c.x, q.x, a.x, b.x);
        rd_cell(p, cu[k].y, lu[k].y, c.y, q.y, a.y, b.y);
        rd_cell(p, cu[k].z, lu[k].z, c.z, q.z, a.z, b.z);
        rd_cell(p, cu[k].w, lu[k].w, c.w, q.w, a.w, b.w);
        if (nvalid == 4) { *reinterpret_cast<float4*>(un + off) = a; *reinterpret_cast<float4*>(vn + off) = b; }
        else for (int j = 0; j < nvalid; ++j) { un[off + j] = f4_get(a, j); vn[off + j] = f4_get(b, j); }
    }
};

// stage of k_rd_ring: u and v with their halo lines
constexpr int RD_NH = 2, RD_NE = 0;

// All substeps of one call in one cooperative launch.  The state ping-pongs between (u, v) and the scratch (su, sv) so that the last
// substep writes (u, v); an odd count first copies (u, v) into the scratch.
template <int DIM, bool GENERIC>
__global__ void __launch_bounds__(RING_THREADS, 1)
k_rd_ring(DGrid g, DField f, RingCfg cfg, float* u, float* v, float* su, float* sv, RdParams p, int substeps)
{
    extern __shared__ __align__(128) unsigned char smem[];
    Ring rg;
    ring_init(rg, smem, cfg);
    cg::grid_group grid = cg::this_grid();
    ThreadGroups tg;
    groups_init(tg, cfg, g, f);
    float* src[2] = {u, v};
    float* dst[2] = {su, sv};
    if (substeps & 1) {
        step_copy_units<DIM, true>(cfg, g, f, tg, su, u, sv, v);
        step_grid_sync(grid);
        src[0] = su; src[1] = sv; dst[0] = u; dst[1] = v;
    }
    for (int s = 0; s < substeps; ++s) {
        const float* hsrc[2] = {src[0], src[1]};
        const float* esrc[2] = {nullptr, nullptr};
        REpiReactionDiffusion epi;
        epi.un = dst[0]; epi.vn = dst[1]; epi.p = p;
        for (int unit = blockIdx.x; unit < cfg.total_units; unit += gridDim.x)
            ring_process_unit<GENERIC, DIM, RD_NH, RD_NE, false>(rg, cfg, g, f, tg, hsrc, esrc, 0.f, ring_unit<DIM>(cfg, g, unit), epi);
        if (s + 1 < substeps) step_grid_sync(grid);
        float* t0 = src[0]; float* t1 = src[1];
        src[0] = dst[0]; src[1] = dst[1]; dst[0] = t0; dst[1] = t1;
    }
}

// ---- N8 wave step (the Waves notebook) -------------------------------------------------------------------------------------------
// One substep of the notebook's step, per cell, with the disc of substep s stamped on both states first:
//   h_c' = where(disc_s, v_s, h_c);  h_p' = where(disc_s, v_s, h_p)
//   h_n = ((2 h_c') - h_p') + dd ((k_speed laplace(h_c')) - (k_damp (h_c' - h_p'))),   returns (h_n, h_c')
// each operation rounded on its own, as the reference's float32 field arithmetic rounds it.  h_c is the one haloed array of a stage,
// h_p the one element-wise array: it is read only at its own cell, so h_n overwrites h_p in place and the two arrays swap roles every
// substep.  The stamp costs no pass over the grid: the stored h_c of substep s is always already stamped (by the epilogue of substep
// s - 1, which stamps disc s on the h_n it writes, or by a pre-pass over disc 0's box), and h_p is stamped as it is read.
// disc_s = { cells with ((p_x - c_x)^2 + (p_y - c_y)^2) [+ (p_z - c_z)^2] <= r^2 } at the float32 cell centres p (Sphere.lies_inside).
struct WaveCoords { const float* p[3]; };     // cell centres along x, y, z
__device__ __forceinline__ bool wave_in_disc(const WaveDisc& d, const WaveCoords& pc, float r2, int x, int y, int z, int dim)
{
    float t = __fsub_rn(pc.p[0][x], d.c[0]);
    float s = __fmul_rn(t, t);
    t = __fsub_rn(pc.p[1][y], d.c[1]);
    s = __fadd_rn(s, __fmul_rn(t, t));
    if (dim == 3) { t = __fsub_rn(pc.p[2][z], d.c[2]); s = __fadd_rn(s, __fmul_rn(t, t)); }
    return s <= r2;
}

// the unit's lines [y0, y0 + TY) of planes [z0, z1) meet the disc's box
template <int DIM>
__device__ __forceinline__ bool wave_unit_hit(const WaveDisc& d, const RingCfg& cfg, const RingUnit& u)
{
    return d.lo[0] < d.hi[0] && d.lo[1] < u.y0 + cfg.TY && d.hi[1] > u.y0 && (DIM == 2 || (d.lo[2] < u.z1 && d.hi[2] > u.z0));
}

template <int DIM>
struct REpiWave {
    static constexpr bool kRefStencil = true;
    float* hn;                 // h_n (the h_p array, or the scratch in the last substep of an odd count)
    float* hc_out;             // the last substep of an odd count: h_c' goes to the h_p array; nullptr otherwise
    WaveCoords pc; WaveParams p;
    WaveDisc dp, dn;           // disc of this substep (stamped on h_p) and of the next one (stamped on h_n)
    bool hit_p, hit_n;         // per unit: the unit meets dp's / dn's box
    long long bbase, sz; int sy, z;
    __device__ __forceinline__ void set_plane(int zz, int) { z = zz < 0 ? 0 : zz; }
    __device__ __forceinline__ void set_acc(const float4&) {}
    __device__ __forceinline__ void stamp(float4& v, const WaveDisc& d, int x0, int y, int nvalid) const
    {
        if (y < d.lo[1] || y >= d.hi[1] || x0 + 4 <= d.lo[0] || x0 >= d.hi[0] || (DIM == 3 && (z < d.lo[2] || z >= d.hi[2]))) return;
        for (int j = 0; j < nvalid; ++j)
            if (wave_in_disc(d, pc, p.r2, x0 + j, y, z, DIM)) f4_set(v, j, d.value);
    }
    __device__ __forceinline__ float cell(float c, float q, float hp) const
    {
        const float damp = __fmul_rn(p.k_damp, __fsub_rn(c, hp));
        return __fadd_rn(__fsub_rn(__fmul_rn(2.f, c), hp), __fmul_rn(p.dd, __fsub_rn(__fmul_rn(p.k_speed, q), damp)));
    }
    __device__ __forceinline__ void operator()(long long off, const float4& c, const float4& q, int nvalid, const float4& e0, const float4&, const float4&)
    {
        float4 hp = e0;
        int x0 = 0, y = 0;
        if (hit_p || hit_n) {
            const int rel = (int)(off - bbase - z * sz);
            y = rel / sy; x0 = rel - y * sy;
        }
        if (hit_p) stamp(hp, dp, x0, y, nvalid);
        float4 h = make_float4(cell(c.x, q.x, hp.x), cell(c.y, q.y, hp.y), cell(c.z, q.z, hp.z), cell(c.w, q.w, hp.w));
        if (hit_n) stamp(h, dn, x0, y, nvalid);
        if (nvalid == 4) {
            *reinterpret_cast<float4*>(hn + off) = h;
            if (hc_out) *reinterpret_cast<float4*>(hc_out + off) = c;
        } else {
            for (int j = 0; j < nvalid; ++j) { hn[off + j] = f4_get(h, j); if (hc_out) hc_out[off + j] = f4_get(c, j); }
        }
    }
};

// stage of k_wave_ring: h_c with its halo lines, h_p element-wise
constexpr int WAVE_NH = 1, WAVE_NE = 1;

// All substeps of one call in one cooperative launch.  Before the loop, disc 0 is stamped on h_c over its box.  Substep s reads the
// array a (h_c, staged with halo lines) and b (h_p, element-wise) and writes h_n into b; then a and b swap.  After an even count
// the newest state is in hc and the previous (stamped) one in hp.  For an odd count the last substep writes h_n into the scratch and
// h_c' into hp, and a final pass copies the scratch into hc.  12 B/cell per substep (+ 12 B/cell once for an odd count, + the box of
// disc 0).
template <int DIM, bool GENERIC>
__global__ void __launch_bounds__(RING_THREADS, 1)
k_wave_ring(DGrid g, DField f, RingCfg cfg, float* hc, float* hp, float* tmp, const WaveDisc* discs, const float* coords, WaveParams p,
            int substeps)
{
    extern __shared__ __align__(128) unsigned char smem[];
    Ring rg;
    ring_init(rg, smem, cfg);
    cg::grid_group grid = cg::this_grid();
    ThreadGroups tg;
    groups_init(tg, cfg, g, f);
    const bool odd = substeps & 1;
    const WaveCoords pc = {{coords, coords + g.n[0], coords + g.n[0] + g.n[1]}};
    {
        const WaveDisc d = discs[0];
        const int bx = d.hi[0] - d.lo[0], by = d.hi[1] - d.lo[1], bz = DIM == 3 ? d.hi[2] - d.lo[2] : 1;
        if (bx > 0 && by > 0 && bz > 0) {
            const long long cells = (long long)bx * by * bz * g.batch;
            for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < cells; i += (long long)gridDim.x * blockDim.x) {
                long long r = i;
                const int x = d.lo[0] + (int)(r % bx); r /= bx;
                const int y = d.lo[1] + (int)(r % by); r /= by;
                const int z = DIM == 3 ? d.lo[2] + (int)(r % bz) : 0;
                const int b = (int)(r / bz);
                if (wave_in_disc(d, pc, p.r2, x, y, z, DIM))
                    hc[(long long)b * f.sb + (long long)z * f.sz + (long long)y * f.sy + x] = d.value;
            }
            step_grid_sync(grid);
        }
    }
    float* a = hc;
    float* b = hp;
    for (int s = 0; s < substeps; ++s) {
        const bool last_odd = odd && s == substeps - 1;
        REpiWave<DIM> epi;
        epi.hn = last_odd ? tmp : b;
        epi.hc_out = last_odd ? b : nullptr;
        epi.pc = pc; epi.p = p; epi.z = 0; epi.sy = (int)f.sy; epi.sz = f.sz;
        epi.dp = discs[s];
        if (s + 1 < substeps) epi.dn = discs[s + 1];
        const float* hsrc[1] = {a};
        const float* esrc[1] = {b};
        for (int unit = blockIdx.x; unit < cfg.total_units; unit += gridDim.x) {
            const RingUnit u = ring_unit<DIM>(cfg, g, unit);
            epi.hit_p = wave_unit_hit<DIM>(epi.dp, cfg, u);
            epi.hit_n = s + 1 < substeps && wave_unit_hit<DIM>(epi.dn, cfg, u);
            epi.bbase = (long long)u.b * f.sb;
            ring_process_unit<GENERIC, DIM, WAVE_NH, WAVE_NE, false>(rg, cfg, g, f, tg, hsrc, esrc, 0.f, u, epi);
        }
        if (s + 1 < substeps || last_odd) step_grid_sync(grid);
        float* t = a; a = b; b = t;
    }
    if (odd) step_copy_units<DIM, false>(cfg, g, f, tg, hc, tmp);
}

// ---- host side of the persistent steppers -----------------------------------------------------------------------------------------
// The ring of a stepper stages its NH haloed arrays with their halo lines and its NE element-wise arrays: (NH + NE) TY + 2 NH lines per
// stage; the whole shared memory, one CTA per SM (cooperative launch).  kernel: PHI_KERNEL_RD_RING or PHI_KERNEL_WAVE_RING.
static bool step_ring_config(const DGrid& g, int kernel, int target_units, RingCfg* c)
{
    int nh, ne;
    switch (kernel) {
    case PHI_KERNEL_RD_RING: nh = RD_NH; ne = RD_NE; break;
    case PHI_KERNEL_WAVE_RING: nh = WAVE_NH; ne = WAVE_NE; break;
    default: return false;
    }
    return ring_config(g, nh + ne, 2 * nh, 0, g.dim == 3 ? 4 : 2, RING_MAX_STAGES, target_units, c);
}

bool phi_step_ring_fits(const DGrid& g, int kernel)
{
    RingCfg c;
    return g.halo == 0 && step_ring_config(g, kernel, 1, &c);
}

int phi_step_ring_max_width(const DGrid& g, int kernel)
{
    return ring_max_width(g, [&](const DGrid& h) { return phi_step_ring_fits(h, kernel); });
}

// Sets the dynamic shared memory of fn, sizes the grid from its occupancy (at most one CTA per unit) and launches it cooperatively
// with args.  -100: not even one CTA fits on an SM.  name: the stepper, in the error message of a failed launch.
static int launch_step_ring(const void* fn, const RingCfg& cfg, void** args, int kernel, bool generic, const char* name, cudaStream_t s)
{
    const size_t smem = 128 + (size_t)cfg.R * cfg.stage_floats * 4;
    int per_sm = 0;
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, RING_THREADS, smem);
    if (e != cudaSuccess) return (int)e;
    if (per_sm < 1) return -100;
    int grid = phi_sm_count() * per_sm;
    if (grid > cfg.total_units) grid = cfg.total_units;
    e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(RING_THREADS), args, smem, s);
    if (e != cudaSuccess) { phi_set_error("%s: cooperative launch failed: %s", name, cudaGetErrorString(e)); return (int)e; }
    note_ring_launch(kernel, cfg, generic, false, false, grid);
    return 0;
}

int phi_launch_reaction_diffusion(const DGrid& g, const DField& f, float* u, float* v, float* su, float* sv, const RdParams& p,
                                  int substeps, cudaStream_t s)
{
    RingCfg cfg;
    if (!step_ring_config(g, PHI_KERNEL_RD_RING, phi_sm_count(), &cfg)) return -100;
    const bool generic = !ring_all_fast(g, f, cfg);
    const void* fn = g.dim == 3 ? (generic ? (const void*)k_rd_ring<3, true> : (const void*)k_rd_ring<3, false>)
                                : (generic ? (const void*)k_rd_ring<2, true> : (const void*)k_rd_ring<2, false>);
    DGrid ga = g; DField fa = f; RdParams pa = p; int ns = substeps;
    void* args[] = {&ga, &fa, &cfg, &u, &v, &su, &sv, &pa, &ns};
    return launch_step_ring(fn, cfg, args, PHI_KERNEL_RD_RING, generic, "reaction_diffusion", s);
}

int phi_launch_wave(const DGrid& g, const DField& f, float* hc, float* hp, float* tmp, const WaveDisc* discs, const float* coords,
                    const WaveParams& p, int substeps, cudaStream_t s)
{
    RingCfg cfg;
    if (!step_ring_config(g, PHI_KERNEL_WAVE_RING, phi_sm_count(), &cfg)) return -100;
    const bool generic = !ring_all_fast(g, f, cfg);
    const void* fn = g.dim == 3 ? (generic ? (const void*)k_wave_ring<3, true> : (const void*)k_wave_ring<3, false>)
                                : (generic ? (const void*)k_wave_ring<2, true> : (const void*)k_wave_ring<2, false>);
    DGrid ga = g; DField fa = f; WaveParams pa = p; int ns = substeps;
    void* args[] = {&ga, &fa, &cfg, &hc, &hp, &tmp, &discs, &coords, &pa, &ns};
    return launch_step_ring(fn, cfg, args, PHI_KERNEL_WAVE_RING, generic, "wave", s);
}
