// A2 + A12: conjugate gradients on the matrix-free pressure Poisson operator  --  ONE persistent cooperative kernel
// per solve.
//
// Reference algorithm: Shewchuk CG as written in PhiML/phiml/backend/_linalg.py:52-90 with the stopping rule of
// stop_on_l2 (:23-40) and the rank-1 offset of linear() (:784-789), applied by the reference to an explicit CSR matrix
// that it obtains by tracing fluid.masked_laplace (phi/physics/fluid.py:165-202).  Here the operator is applied on the
// fly (SURVEY.md Appendix A: it is the 5/7-point laplace with the PRESSURE boundary), and the iteration is reorganised
// into two grid-wide passes with 32 B/cell of HBM traffic instead of the textbook three passes / 44 B:
//
//   pass A:  d' = r + beta*d          (written)          dq = sum d' * (A d')       S = sum d'
//            -- grid barrier --       alpha = delta / (dq + c*S^2)
//   pass B:  q = A d' + c*S  (recomputed, never stored)  x += alpha*d'   r -= alpha*q    delta' = sum r*r
//            -- grid barrier --       beta = delta'/delta, convergence test per batch entry
//
// d is double-buffered because pass A needs the OLD d in the halo cells of neighbouring tiles.  Dot products are
// accumulated per thread in fp32 over at most a few hundred cells, then in fp64 across warps / CTAs in a fixed order
// (deterministic, independent of scheduling).  Every CTA redundantly reduces the per-CTA partials and therefore
// takes identical control-flow decisions; nothing returns to the host until the solve is over.
#include <cooperative_groups.h>
#include <type_traits>
#include "phi_internal.cuh"
#include "launch.cuh"

namespace cg = cooperative_groups;

#include "cg_common.cuh"

// ---- sources / epilogues ---------------------------------------------------------------------------------

template <class T>
struct SrcDirection {          // d' = r + beta*d
    const T* r; const T* d; T beta;
    __device__ __forceinline__ Vec4<T> load4(long long off) const
    {
        Vec4<T> a = *reinterpret_cast<const Vec4<T>*>(r + off);
        if (beta != T(0)) {
            const Vec4<T> o = *reinterpret_cast<const Vec4<T>*>(d + off);
            a.x += beta * o.x; a.y += beta * o.y; a.z += beta * o.z; a.w += beta * o.w;
        }
        return a;
    }
    __device__ __forceinline__ T load1(long long off) const
    {
        T a = r[off];
        if (beta != T(0)) a += beta * d[off];
        return a;
    }
};

template <class T>
struct EpiResidual0 {          // r = (rhs - mean) - A x0 [- c*sum(x0)];  acc0 = |r|^2, acc1 = |r without offset|^2
    using V = Vec4<T>;
    const T* rhs; T* r; T mean; T offs;
    T acc0, acc1;
    const T* accm;                 // N4: balanced rhs is  div - accessible * mean(div)/mean(accessible)  (fluid.py:205-209)
    __device__ __forceinline__ void operator()(long long off, const V& c, const V& q, int nvalid)
    {
        const V y = *reinterpret_cast<const V*>(rhs + off);
        V mm = f4_splat(mean);
        if (accm) { const V a4 = *reinterpret_cast<const V*>(accm + off); mm = f4_make(mean * a4.x, mean * a4.y, mean * a4.z, mean * a4.w); }
        V rt;                                         // residual without offset (tolerance reference, _linalg.py:61-67)
        rt.x = (y.x - mm.x) - q.x; rt.y = (y.y - mm.y) - q.y; rt.z = (y.z - mm.z) - q.z; rt.w = (y.w - mm.w) - q.w;
        V rr = f4_make(rt.x - offs, rt.y - offs, rt.z - offs, rt.w - offs);
        if (nvalid == 4) {
            *reinterpret_cast<V*>(r + off) = rr;
            acc0 += rr.x * rr.x + rr.y * rr.y + rr.z * rr.z + rr.w * rr.w;
            acc1 += rt.x * rt.x + rt.y * rt.y + rt.z * rt.z + rt.w * rt.w;
        } else {
            for (int j = 0; j < nvalid; ++j) {
                const T a = f4_get(rr, j), t = f4_get(rt, j);
                r[off + j] = a; acc0 += a * a; acc1 += t * t;
            }
        }
    }
};

template <class T>
struct EpiPassA {              // store d', acc0 = d'.(A d'), acc1 = sum d'
    using V = Vec4<T>;
    T* dnew; T acc0, acc1;
    __device__ __forceinline__ void operator()(long long off, const V& c, const V& q, int nvalid)
    {
        if (nvalid == 4) {
            *reinterpret_cast<V*>(dnew + off) = c;
            acc0 += c.x * q.x + c.y * q.y + c.z * q.z + c.w * q.w;
            acc1 += (c.x + c.y) + (c.z + c.w);
        } else {
            for (int j = 0; j < nvalid; ++j) { const T v = f4_get(c, j); dnew[off + j] = v; acc0 += v * f4_get(q, j); acc1 += v; }
        }
    }
};

template <class T>
struct EpiPassB {              // x += alpha d', r -= alpha (A d' + c S), acc0 = |r|^2
    using V = Vec4<T>;
    T* x; T* r; T alpha; T offs; T acc0, acc1;
    __device__ __forceinline__ void operator()(long long off, const V& c, const V& q, int nvalid)
    {
        if (nvalid == 4) {
            V xv = *reinterpret_cast<V*>(x + off);
            V rv = *reinterpret_cast<V*>(r + off);
            xv.x += alpha * c.x; xv.y += alpha * c.y; xv.z += alpha * c.z; xv.w += alpha * c.w;
            rv.x -= alpha * (q.x + offs); rv.y -= alpha * (q.y + offs); rv.z -= alpha * (q.z + offs); rv.w -= alpha * (q.w + offs);
            *reinterpret_cast<V*>(x + off) = xv;
            *reinterpret_cast<V*>(r + off) = rv;
            acc0 += rv.x * rv.x + rv.y * rv.y + rv.z * rv.z + rv.w * rv.w;
        } else {
            for (int j = 0; j < nvalid; ++j) {
                const T xv = x[off + j] + alpha * f4_get(c, j);
                const T rv = r[off + j] - alpha * (f4_get(q, j) + offs);
                x[off + j] = xv; r[off + j] = rv; acc0 += rv * rv;
            }
        }
    }
};

// ---- helpers ------------------------------------------------------------------------------------------------

// Iterate over the cells of a warp unit without a stencil (sums, final mean removal).
template <int DIM, class T, class F>
__device__ __forceinline__ void for_unit_cells(const DGridT<T>& g, const DFieldT<T>& pf, const WarpUnit& w, F&& fn)
{
    const int lane = threadIdx.x & 31;
    const int x0 = w.xt0 + lane * 4;
    if (x0 >= g.n[0]) return;
    const int nvalid = min(4, g.n[0] - x0);
    for (int m = w.m0; m < w.m1; ++m) {
        const long long off = (long long)w.b * pf.sb + (DIM == 3 ? (long long)m * pf.sz + (long long)w.t * pf.sy : (long long)m * pf.sy) + x0;
        fn(off, nvalid);
    }
}

// ---- the solver ---------------------------------------------------------------------------------------------

// T = float: the fp32 solve (per-thread dot products in float); T = double: the fp64 solve (N9), everything in double.
template <int DIM, bool MASK, class T>
__global__ void __launch_bounds__(PHI_WARPS_PER_CTA * 32, 2)
k_cg_poisson(CgArgsT<T> a)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    CgSharedT<T> sh = cg_carve<T>(smem_raw, a.g.batch);
    cg::grid_group grid = cg::this_grid();
    const DGridT<T>& g = a.g;
    const UnitMap& um = a.um;
    const int warp = threadIdx.x >> 5;
    const int batch = g.batch;
    const double cells = (double)g.n[0] * g.n[1] * g.n[2];
    const T coffs = a.prm.matrix_offset;
    int region = 0;

    // Runs `body(w, acc0, acc1)` over the units of this CTA, flushing the accumulators whenever the batch entry changes.
    auto sweep = [&](const unsigned char* active, auto&& body) {
        int cur_b = -1; T acc0 = 0, acc1 = 0;
        for (int unit = blockIdx.x; unit < um.total_units; unit += gridDim.x) {
            const int b = unit / um.units_per_batch;
            if (active && !active[b]) continue;
            if (b != cur_b) {
                if (cur_b >= 0) flush_partials(sh, a.partials, region, batch, cur_b, acc0, acc1);
                cur_b = b; acc0 = 0; acc1 = 0;
            }
            const WarpUnit w = phi_warp_unit<DIM>(g, um, unit, warp);
            if (w.valid) body(w, acc0, acc1);
        }
        if (cur_b >= 0) flush_partials(sh, a.partials, region, batch, cur_b, acc0, acc1);
    };
    auto barrier_and_reduce = [&](const unsigned char* active) {
        grid.sync();
        reduce_partials(sh, a.partials, region, batch, um.units_per_batch, active);
        region ^= 1;
    };

    for (int b = threadIdx.x; b < batch; b += blockDim.x) { sh.mean[b] = 0; sh.offs[b] = 0; }
    __syncthreads();

    // ---- setup: mean(rhs) for the balanced right-hand side, sum(x0) for the offset term -----------------------
    if (a.prm.balance_rhs || coffs != T(0)) {
        sweep(nullptr, [&](const WarpUnit& w, T& acc0, T& acc1) {
            for_unit_cells<DIM>(g, a.pf, w, [&](long long off, int nvalid) {
                for (int j = 0; j < nvalid; ++j) { acc0 += a.rhs[off + j]; acc1 += MASK ? a.acc[off + j] : a.x[off + j]; }
            });
        });
        barrier_and_reduce(nullptr);
        for (int b = threadIdx.x; b < batch; b += blockDim.x) cg_balance<MASK>(sh, a.prm, b, cells);
        __syncthreads();
    }

    // ---- r0 = y - (A + c 11^T) x0,  delta0 -----------------------------------------------------------------------
    sweep(nullptr, [&](const WarpUnit& w, T& acc0, T& acc1) {
        SrcArrayT<T> src{a.x};
        EpiResidual0<T> epi{a.rhs, a.r, sh.mean[w.b], sh.offs[w.b], 0, 0, MASK ? a.acc : nullptr};
        if constexpr (MASK) phi_march_masked<DIM>(g, a.pf, src, a.acc, epi, w.b, w.xt0, w.t, w.m0, w.m1);
        else                phi_march<DIM>(g, a.pf, src, epi, w.b, w.xt0, w.t, w.m0, w.m1);
        acc0 += epi.acc0; acc1 += epi.acc1;
    });
    barrier_and_reduce(nullptr);
    cg_start(sh, a.prm, batch);

    T* dold = a.d0; T* dnew = a.d1;
    while (*sh.any_cont) {
        // ---- pass A ---------------------------------------------------------------------------------------------
        sweep(sh.cont, [&](const WarpUnit& w, T& acc0, T& acc1) {
            SrcDirection<T> src{a.r, dold, sh.beta[w.b]};
            EpiPassA<T> epi{dnew, 0, 0};
            if constexpr (MASK) phi_march_masked<DIM>(g, a.pf, src, a.acc, epi, w.b, w.xt0, w.t, w.m0, w.m1);
            else                phi_march<DIM>(g, a.pf, src, epi, w.b, w.xt0, w.t, w.m0, w.m1);
            acc0 += epi.acc0; acc1 += epi.acc1;
        });
        barrier_and_reduce(sh.cont);
        for (int b = threadIdx.x; b < batch; b += blockDim.x) {
            if (!sh.cont[b]) continue;
            const double S = sh.sum1[b];
            const double dq = sh.sum0[b] + (double)coffs * S * S;
            sh.alpha[b] = (dq != 0.0) ? (T)(sh.delta[b] / dq) : T(0);      // divide_no_nan (_linalg.py:74)
            sh.offs[b] = coffs * (T)S;
        }
        __syncthreads();
        // ---- pass B ---------------------------------------------------------------------------------------------
        sweep(sh.cont, [&](const WarpUnit& w, T& acc0, T& acc1) {
            SrcArrayT<T> src{dnew};
            EpiPassB<T> epi{a.x, a.r, sh.alpha[w.b], sh.offs[w.b], 0, 0};
            if constexpr (MASK) phi_march_masked<DIM>(g, a.pf, src, a.acc, epi, w.b, w.xt0, w.t, w.m0, w.m1);
            else                phi_march<DIM>(g, a.pf, src, epi, w.b, w.xt0, w.t, w.m0, w.m1);
            acc0 += epi.acc0;
        });
        barrier_and_reduce(sh.cont);
        for (int b = threadIdx.x; b < batch; b += blockDim.x) {
            if (!sh.cont[b]) continue;
            const double dn = sh.sum0[b];
            const double dold_ = sh.delta[b];
            sh.beta[b] = (dold_ != 0.0) ? (T)(dn / dold_) : T(0);
            cg_iteration_done(sh, a.prm, b, dn);
        }
        cg_count_running(sh, batch);
        T* t = dold; dold = dnew; dnew = t;
    }

    // ---- zero-mean solution of the rank-deficient system ------------------------------------------------------
    if (a.prm.project_mean) {
        sweep(nullptr, [&](const WarpUnit& w, T& acc0, T& acc1) {
            for_unit_cells<DIM>(g, a.pf, w, [&](long long off, int nvalid) {
                for (int j = 0; j < nvalid; ++j) { if (MASK) { acc0 += a.x[off + j] * a.acc[off + j]; acc1 += a.acc[off + j]; } else acc0 += a.x[off + j]; }
            });
        });
        barrier_and_reduce(nullptr);
        for (int unit = blockIdx.x; unit < um.total_units; unit += gridDim.x) {
            const WarpUnit w = phi_warp_unit<DIM>(g, um, unit, warp);
            if (!w.valid) continue;
            const T m = cg_projection_mean<MASK>(sh, w.b, cells);
            for_unit_cells<DIM>(g, a.pf, w, [&](long long off, int nvalid) {
                for (int j = 0; j < nvalid; ++j) a.x[off + j] -= MASK ? m * a.acc[off + j] : m;
            });
        }
    }

    cg_write_result(sh, a.result, batch, true);
}

// ---- host side --------------------------------------------------------------------------------------------------

template <class T>
static const void* cg_kernel(int dim, bool mask)
{
    if constexpr (std::is_same<T, float>::value) {
        if (dim == 3) return mask ? (const void*)k_cg_poisson<3, true, float> : (const void*)k_cg_poisson<3, false, float>;
        return mask ? (const void*)k_cg_poisson<2, true, float> : (const void*)k_cg_poisson<2, false, float>;
    } else {
        return dim == 3 ? (const void*)k_cg_poisson<3, false, T> : (const void*)k_cg_poisson<2, false, T>;
    }
}

template <class T>
static int cg_grid_size(int dim, int batch, bool mask, int* blocks_per_sm_out)
{
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t smem = cg_smem_bytes<T>(batch);
    cudaFuncSetAttribute(cg_kernel<T>(dim, mask), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cg_kernel<T>(dim, mask), PHI_WARPS_PER_CTA * 32, smem);
    if (blocks_per_sm_out) *blocks_per_sm_out = per_sm;
    return sms * per_sm;
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

CgWorkspace phi_cg_workspace(const DGrid& g, void* base)
{
    const size_t arr = align_up((size_t)g.cext[0] * g.cext[1] * g.cext[2] * g.batch * sizeof(float), 256);
    const size_t pbytes = align_up((size_t)8 * g.batch * CG_MAX_GRID * sizeof(double), 256);
    CgWorkspace w = {};
    w.bytes = 4 * arr + pbytes;
    if (!base) return w;
    unsigned char* ws = (unsigned char*)base;
    const size_t hoff = (size_t)g.halo * g.cext[0] * g.cext[1];
    w.r = (float*)ws + hoff; w.d0 = (float*)(ws + arr) + hoff; w.d1 = (float*)(ws + 2 * arr) + hoff;
    w.partials = (double*)(ws + 3 * arr);
    w.d2 = (float*)(ws + 3 * arr + pbytes) + hoff;
    return w;
}

// The launch of the register-marching kernel once the caller has checked the solve; a.rhs, a.x, a.acc, the work vectors, result and
// prm are set.
template <class T>
static int launch_cg_march(CgArgsT<T> a, bool mask, cudaStream_t s)
{
    const auto& g = a.g;
    int per_sm = 0;
    int grid = cg_grid_size<T>(g.dim, g.batch, mask, &per_sm);
    if (grid <= 0) { phi_set_error("cg: kernel does not fit on the device (occupancy 0)"); return PHI_ERR_INVALID; }
    a.um = phi_make_unit_map(g, grid * 8);
    if (grid > a.um.total_units) grid = a.um.total_units;
    if (grid > CG_MAX_GRID) grid = CG_MAX_GRID;
    if (g.halo != 0) { phi_set_error("cg: z-slab grids need the TMA ring kernel (grid lines too long)"); return PHI_ERR_UNSUPPORTED; }
    void* args[] = {&a};
    const size_t smem = cg_smem_bytes<T>(g.batch);
    cudaError_t err;
    err = cudaLaunchCooperativeKernel(cg_kernel<T>(g.dim, mask), dim3(grid), dim3(PHI_WARPS_PER_CTA * 32), args, smem, s);
    if (err != cudaSuccess) { phi_set_error("cg: cooperative launch failed: %s", cudaGetErrorString(err)); return (int)err; }
    phi_note_cg_passes(2);
    phi_note_cg_operator(PHI_CG_OP_POISSON);
    PhiLaunchInfo li = {}; li.kernel = PHI_KERNEL_CG_MARCH; li.generic = 1; li.masked = mask; li.total_units = a.um.total_units; li.grid_ctas = grid;
    phi_note_launch(li);
    return 0;
}

int phi_launch_cg(const CgLaunch& l, cudaStream_t s)
{
    const DGrid& g = l.g;
    if (g.batch > CG_MAX_BATCH) { phi_set_error("cg: batch %d exceeds %d (split the batch)", g.batch, CG_MAX_BATCH); return PHI_ERR_UNSUPPORTED; }
    const CgWorkspace w = phi_cg_workspace(g, l.workspace);
    if (l.workspace_bytes < w.bytes) { phi_set_error("cg: workspace %zu < %zu bytes", l.workspace_bytes, w.bytes); return PHI_ERR_WORKSPACE; }
    const bool mask = l.op.kind == CgOp::Masked;
    const bool adaptive = l.prm.method == PHI_SOLVER_CG_ADAPTIVE;
    if (l.prm.method != PHI_SOLVER_CG && !adaptive) { phi_set_error("cg: unknown solver method %d", l.prm.method); return PHI_ERR_INVALID; }
    if (adaptive && l.prm.matrix_offset != 0.f) { phi_set_error("cg: CG-adaptive does not take a matrix_offset"); return PHI_ERR_UNSUPPORTED; }
    if (phi_ring_enabled()) {        // obstacles included: the mask is staged as an extra haloed array of the ring
        const int e = phi_launch_cg_ring(l, nullptr, s);
        if (e != -100) return e;
    }
    if (adaptive) {
        if (!phi_ring_enabled()) phi_set_error("cg: CG-adaptive runs on the TMA ring kernel only, which PHICUDA_NO_RING switches off");
        else phi_set_error("cg: CG-adaptive runs on the TMA ring kernel only; grid lines of %d cells do not fit it (%d-D%s, batch %d: at most %d cells)",
                           g.n[0], g.dim, mask ? " with obstacles" : "", g.batch, phi_cg_ring_max_width(g, l.op.kind, true));
        return PHI_ERR_UNSUPPORTED;
    }
    if (mask && l.prm.matrix_offset != 0.f) { phi_set_error("cg: matrix_offset is not supported together with obstacles"); return PHI_ERR_UNSUPPORTED; }
    CgArgs a;
    a.g = g; a.pf = l.pf;
    a.rhs = l.rhs; a.x = l.x; a.acc = l.op.mask;
    a.r = w.r; a.d0 = w.d0; a.d1 = w.d1; a.partials = w.partials;
    a.result = l.result; a.prm = l.prm;
    return launch_cg_march<float>(a, mask, s);
}

// fp64 workspace: r | d0 | d1 | partials[2][2][batch][CG_MAX_GRID] (the register-marching kernel uses partial regions 0 and 1 only)
size_t phi_cg_workspace_bytes_f64(const DGridT<double>& g)
{
    const size_t arr = align_up((size_t)g.cext[0] * g.cext[1] * g.cext[2] * g.batch * sizeof(double), 256);
    return 3 * arr + align_up((size_t)4 * g.batch * CG_MAX_GRID * sizeof(double), 256);
}

int phi_launch_cg(const CgLaunch64& l, cudaStream_t s)
{
    // the entry points check the solve (api.cu cg_setup64: batch, z-slabs, method, workspace size) before the first CUDA call
    const DGridT<double>& g = l.g;
    const size_t arr = align_up((size_t)g.cext[0] * g.cext[1] * g.cext[2] * g.batch * sizeof(double), 256);
    unsigned char* ws = (unsigned char*)l.workspace;
    CgArgsT<double> a;
    a.g = g; a.pf = l.pf;
    a.rhs = l.rhs; a.x = l.x; a.acc = nullptr;
    a.r = (double*)ws; a.d0 = (double*)(ws + arr); a.d1 = (double*)(ws + 2 * arr); a.partials = (double*)(ws + 3 * arr);
    a.result = l.result; a.prm = l.prm;
    return launch_cg_march<double>(a, false, s);
}
