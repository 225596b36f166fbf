// Shared pieces of the two CG implementations (LDG marching kernel in cg_kernels.cu, TMA ring kernel in ring_kernels.cu).
#pragma once
#include "phi_internal.cuh"

#define CG_MAX_BATCH 1024
#define CG_MAX_GRID 2048

// The C-ABI parameter and result records of a solve in each precision.
template <class T> struct CgTypes;
template <> struct CgTypes<float> { using Params = PhiCgParams; using Result = PhiCgResult; };
template <> struct CgTypes<double> { using Params = PhiCgParams64; using Result = PhiCgResult64; };

template <class T>
struct CgArgsT {
    DGridT<T> g; DFieldT<T> pf; UnitMap um;
    const T* rhs; T* x; T* r; T* d0; T* d1;
    const T* acc;                  // N4: accessible mask (1 = fluid, 0 = obstacle) or nullptr
    double* partials;              // [2 regions][2 accumulators][batch][grid]
    typename CgTypes<T>::Result* result;
    typename CgTypes<T>::Params prm;
};
using CgArgs = CgArgsT<float>;

// Per-entry state of a solve: pointers carved from one block of shared memory (the CTA's dynamic block) or of global memory (the
// collocated solve's workspace).  Step sizes, offset, mean and tolerances are T: in fp64 a step size rounded to float would hold
// every update to float precision, and a 1e-12 solve could not rely on converging.
template <class T>
struct CgSharedT {
    double (*warp_acc)[32];   // [2][warps] (up to 32 warps per CTA)
    double* sum0;                  // reduced accumulator 0 per batch entry
    double* sum1;
    double* delta;
    T* alpha;
    T* aprev;                      // alpha of the previous iteration (deferred x update of the ring kernel)
    T* beta;
    T* offs;                       // c * S  (offset part of q)
    T* mean;
    T* tol_sq;
    T* rsq0;
    int* iters;
    int* any_cont;
    unsigned char *cont, *conv, *divg;
    T* bprev;                      // beta of the previous iteration (one-sweep ring CG: r_k = d_k - beta_k d_{k-1})
    T* aprev2;                     // one-sweep ring CG: alpha_{k-2} and beta_{k-1}, which rebuild d_{k-2} for a three-direction
    T* bprev2;                     // x update
    int* owed;                     // one-sweep ring CG: directions whose step x still owes (0 .. 2)
};
using CgShared = CgSharedT<float>;

template <class T = float>
__host__ __device__ inline size_t cg_smem_bytes(int batch)
{
    const size_t b8 = ((size_t)batch + 1) / 2 * 2;      // keep 8-byte alignment of what follows
    return 2 * 32 * sizeof(double) + 3 * b8 * sizeof(double) + 10 * b8 * sizeof(T)
         + (2 * b8 + 2) * sizeof(int) + 3 * (b8 + 16) + (sizeof(T) - sizeof(float));   // fp64: room to realign bprev
}

template <class T = float>
__host__ __device__ __forceinline__ CgSharedT<T> cg_carve(unsigned char* base, int batch)
{
    const size_t b8 = ((size_t)batch + 1) / 2 * 2;
    CgSharedT<T> sh;
    unsigned char* p = base;
    sh.warp_acc = reinterpret_cast<double (*)[32]>(p); p += 2 * 32 * sizeof(double);
    sh.sum0 = (double*)p; p += b8 * sizeof(double);
    sh.sum1 = (double*)p; p += b8 * sizeof(double);
    sh.delta = (double*)p; p += b8 * sizeof(double);
    sh.alpha = (T*)p; p += b8 * sizeof(T);
    sh.aprev = (T*)p; p += b8 * sizeof(T);
    sh.beta = (T*)p; p += b8 * sizeof(T);
    sh.offs = (T*)p; p += b8 * sizeof(T);
    sh.mean = (T*)p; p += b8 * sizeof(T);
    sh.tol_sq = (T*)p; p += b8 * sizeof(T);
    sh.rsq0 = (T*)p; p += b8 * sizeof(T);
    sh.iters = (int*)p; p += b8 * sizeof(int);
    sh.any_cont = (int*)p; p += 2 * sizeof(int);
    sh.cont = p; p += b8 + 16;
    sh.conv = p; p += b8;
    sh.divg = p; p += (b8 + 3) / 4 * 4;            // divg starts 4-byte aligned (b8 is even)
    if constexpr (sizeof(T) == 8) p = base + ((size_t)(p - base) + 7) / 8 * 8;
    sh.bprev = (T*)p; p += b8 * sizeof(T);
    sh.aprev2 = (T*)p; p += b8 * sizeof(T);
    sh.bprev2 = (T*)p; p += b8 * sizeof(T);
    sh.owed = (int*)p;
    return sh;
}


#ifndef CG_BLOCK_WARPS
#define CG_BLOCK_WARPS PHI_WARPS_PER_CTA
#endif

// Block-level flush of the two thread accumulators of the current batch entry into partials[region][k][b][cta].
template <class T>
__device__ __forceinline__ void flush_partials(const CgSharedT<T>& sh, double* partials, int region, int batch, int b, double a0, double a1)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    a0 = warp_sum(a0); a1 = warp_sum(a1);
    if (lane == 0) { sh.warp_acc[0][warp] = a0; sh.warp_acc[1][warp] = a1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s0 = 0, s1 = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { s0 += sh.warp_acc[0][w]; s1 += sh.warp_acc[1][w]; }
        const size_t G = gridDim.x;
        partials[((size_t)(region * 2 + 0) * batch + b) * G + blockIdx.x] = s0;
        partials[((size_t)(region * 2 + 1) * batch + b) * G + blockIdx.x] = s1;
    }
    __syncthreads();
}

// After a grid barrier: every CTA sums, in a fixed order, the partials of the CTAs that own units of batch entry b.
template <class T>
__device__ __forceinline__ void reduce_partials(const CgSharedT<T>& sh, const double* partials, int region, int batch, int units_per_batch,
                                                const unsigned char* active)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int G = gridDim.x;
    const int cnt = min(units_per_batch, G);
    for (int b = warp; b < batch; b += (int)(blockDim.x >> 5)) {
        if (active && !active[b]) continue;
        const int first = (int)(((long long)b * units_per_batch) % G);
        double s0 = 0, s1 = 0;
        for (int i = lane; i < cnt; i += 32) {
            int c = first + i; if (c >= G) c -= G;
            s0 += __ldcg(&partials[((size_t)(region * 2 + 0) * batch + b) * G + c]);
            s1 += __ldcg(&partials[((size_t)(region * 2 + 1) * batch + b) * G + c]);
        }
        s0 = warp_sum(s0); s1 = warp_sum(s1);
        if (lane == 0) { sh.sum0[b] = s0; sh.sum1[b] = s1; }
    }
    __syncthreads();
}

// ---- per-entry bookkeeping of a solve (the caller runs these in its `for (b = threadIdx.x; ...)` loops) -----------------------

// Setup sums sum0 = sum y, sum1 = sum of the accessible mask (MASK) or of x0 -> balanced right-hand side y - mean (* mask,
// fluid.py:205-209) and the offset c * sum x0 of the rank-1 matrix offset.  cells: the global cell count.
template <bool MASK, class T, class P>
__device__ __forceinline__ void cg_balance(const CgSharedT<T>& sh, const P& prm, int b, double cells)
{
    if (MASK) { sh.mean[b] = (prm.balance_rhs && sh.sum1[b] > 0.0) ? (T)(sh.sum0[b] / sh.sum1[b]) : T(0); sh.offs[b] = 0; }
    else { sh.mean[b] = prm.balance_rhs ? (T)(sh.sum0[b] / cells) : T(0); sh.offs[b] = prm.matrix_offset * (T)sh.sum1[b]; }
}

// Sums of the zero-mean projection, sum0 = sum x (* mask), sum1 = sum of the mask (MASK) -> the mean to remove.
template <bool MASK, class T>
__device__ __forceinline__ T cg_projection_mean(const CgSharedT<T>& sh, int b, double cells)
{
    return MASK ? (sh.sum1[b] > 0.0 ? (T)(sh.sum0[b] / sh.sum1[b]) : T(0)) : (T)(sh.sum0[b] / cells);
}

// End of an iteration of entry b with the new |r|^2 (the caller has formed its step sizes): iteration count and the stopping
// rule of stop_on_l2 (_linalg.py:29-36).  Returns whether the entry continues.
template <class T, class P>
__device__ __forceinline__ bool cg_iteration_done(const CgSharedT<T>& sh, const P& prm, int b, double rsq_new)
{
    sh.delta[b] = rsq_new;
    const int it = ++sh.iters[b];
    const T rsq = phi_abs((T)rsq_new);
    const bool conv = rsq <= sh.tol_sq[b];
    const bool divg = !isfinite(rsq) || (rsq / sh.rsq0[b] > T(1e5) && it >= 8);
    const bool cont = !conv && !divg && it < prm.max_iter;
    sh.conv[b] = conv; sh.divg[b] = divg; sh.cont[b] = cont ? 1 : 0;
    return cont;
}

// ---- whole-CTA steps ----------------------------------------------------------------------------------------------------------

// *any_cont = whether any entry still runs.  Every CTA computes it from its own copy of the flags, so all take the same branch.
template <class T>
__device__ __forceinline__ void cg_count_running(const CgSharedT<T>& sh, int batch)
{
    __syncthreads();
    if (threadIdx.x == 0) { int any = 0; for (int b = 0; b < batch; ++b) any |= sh.cont[b]; *sh.any_cont = any; }
    __syncthreads();
}

// Start of the solve from the r0 sums: sum0 = |r0|^2, sum1 = the tolerance reference (|r0| without the matrix offset, or |y|^2
// for CG-adaptive; _linalg.py:61-67).  An entry that already meets the tolerance does not iterate.
template <class T, class P>
__device__ __forceinline__ void cg_start(const CgSharedT<T>& sh, const P& prm, int batch)
{
    for (int b = threadIdx.x; b < batch; b += blockDim.x) {
        const double d0 = sh.sum0[b], d0tol = sh.sum1[b];
        sh.delta[b] = d0;
        const T tol = phi_max(prm.rtol * prm.rtol * (T)d0tol, prm.atol * prm.atol);
        sh.tol_sq[b] = tol; sh.rsq0[b] = (T)d0;
        const bool conv = (T)d0 <= tol;
        const bool divg = !isfinite((T)d0);
        sh.conv[b] = conv; sh.divg[b] = divg; sh.iters[b] = 0;
        sh.cont[b] = (!conv && !divg && prm.max_iter > 0) ? 1 : 0;
        sh.beta[b] = 0; sh.alpha[b] = 0; sh.aprev[b] = 0;
    }
    cg_count_running(sh, batch);
}

// Block 0 writes the PhiCgResult of every entry.  comm_ok false (a multi-GPU all-reduce timed out): diverged = -1.
template <class T>
__device__ __forceinline__ void cg_write_result(const CgSharedT<T>& sh, typename CgTypes<T>::Result* result, int batch, bool comm_ok)
{
    if (blockIdx.x != 0) return;
    for (int b = threadIdx.x; b < batch; b += blockDim.x) {
        typename CgTypes<T>::Result res;
        res.iterations = sh.iters[b]; res.converged = sh.conv[b]; res.diverged = comm_ok ? sh.divg[b] : -1;
        res.residual_sq = phi_abs((T)sh.delta[b]); res.tol_sq = sh.tol_sq[b]; res.initial_residual_sq = sh.rsq0[b];
        result[b] = res;
    }
}

