// CenteredGrid (collocated) velocities: fluid.make_incompressible with wide_stencil = True (phi/physics/fluid.py:154-155, 197-202;
// SURVEY.md Appendix A "CenteredGrid velocity variant"; reference tests tests/commit/physics/test_fluid.py:34-36).
//
//   div     = sum_c (v_c[i+1] - v_c[i-1]) / (2 dx_c)            ghosts of v_c from the velocity boundary   (_field_math.py:627-632)
//   A p     = divergence_centered(gradient_centered(p))           gradient ghosts: pressure boundary; divergence ghosts: velocity
//                                                                 boundary with constants removed               (fluid.py:197-202)
//   v_c    -= (p[i+1] - p[i-1]) / (2 dx_c)                                                                  (fluid.py:158-161)
//
// The wide operator ([1 0 -2 0 1] / 4dx^2 in the interior) is not symmetric at the boundary rows, so the reference's default
// Solve() = 'auto' = CG-adaptive (PhiML/phiml/backend/_linalg.py:93-128) is what converges on it; that is the solver here, with
// the reference's rank-1 matrix_offset for rank-deficient systems (linear(), _linalg.py:784-789).
//
// This is NOT the tuned path (the north-star workloads are staggered): one thread per cell, seven launches per iteration, the
// host reads the per-entry running flags every 8 iterations (the entry point is a `_host` call).  Dot products are summed in double
// in a fixed order - per block (warp butterflies, then the four warps in turn), then per entry over the blocks (k_co_reduce) -
// so the same call gives the same bits every time and a batch entry's result does not depend on its neighbours.
// The per-entry bookkeeping - balanced right-hand side, start, stopping rule (stop_on_l2 with the divergence test) and result
// record - is that of the persistent CG kernels (cg_common.cuh), on a CgShared view of the workspace.
// It exists so that CenteredGrid velocities run on the GPU with the reference's semantics instead of falling through.
#include "phi_internal.cuh"
#include "launch.cuh"
#include "cg_common.cuh"

#include <vector>

struct CoVec { DField f[3]; const float* p[3]; };          // three centred arrays with their own boundaries
struct CoOut { float* p[3]; };
// per batch entry, written by k_co_reduce: dir.q, dir.r, sum(dir) (operator application), |r|^2, r.q (phase 1)
struct CoDots { double *dq, *dr, *sd, *rr, *rq; };

template <int DIM>
__device__ __forceinline__ bool co_index(const DGrid& g, int& b, int& x, int& y, int& z)
{
    x = blockIdx.x * blockDim.x + threadIdx.x;
    y = blockIdx.y;
    const int zb = blockIdx.z;
    if (DIM == 3) { z = zb % g.n[2]; b = zb / g.n[2]; } else { z = 0; b = zb; }
    return x < g.n[0] && y < g.n[1];
}

// Blocks of one batch entry: ceil(n_x / 128) x n_y x n_z (co_grid); this block's index among them.
__device__ __forceinline__ int co_block_of_entry(const DGrid& g)
{
    const int z = g.dim == 3 ? blockIdx.z % g.n[2] : 0;
    return (z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
}

// Block sums of N values in a fixed order (butterfly per warp, then warps 0..3 in turn), stored as this block's partials
// part[k * slot + entry * nblk + block], k < N.  Every thread of the block must call it.
template <int N>
__device__ __forceinline__ void co_block_partials(const double (&v)[N], double* __restrict__ part, const DGrid& g, int bb, size_t slot)
{
    __shared__ double w[N][4];
    double s[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
        s[k] = v[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
        if ((threadIdx.x & 31) == 0) w[k][threadIdx.x >> 5] = s[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nblk = gridDim.x * gridDim.y * (g.dim == 3 ? g.n[2] : 1);
        const size_t at = (size_t)bb * nblk + co_block_of_entry(g);
#pragma unroll
        for (int k = 0; k < N; ++k) part[k * slot + at] = ((w[k][0] + w[k][1]) + w[k][2]) + w[k][3];
    }
}

// g_c = (p[i + e_c] - p[i - e_c]) / (2 dx_c), ghosts from pf.   SUB: v_c -= g_c (final correction) instead of storing g_c.
template <int DIM, bool SUB>
__global__ void __launch_bounds__(128)
k_co_gradient(const __grid_constant__ DGrid g, const __grid_constant__ DField pf, const float* __restrict__ p, const __grid_constant__ CoOut out,
              const unsigned char* __restrict__ cont)
{
    int b, x, y, z;
    const bool in = co_index<DIM>(g, b, x, y, z);
    if (!in || (cont && !cont[b])) return;
    const long long off = (long long)b * pf.sb + (long long)z * pf.sz + (long long)y * pf.sy + x;
#pragma unroll
    for (int c = 0; c < DIM; ++c) {
        const float up = phi_fetch<DIM>(p, g, pf, b, x + (c == 0), y + (c == 1), z + (c == 2));
        const float lw = phi_fetch<DIM>(p, g, pf, b, x - (c == 0), y - (c == 1), z - (c == 2));
        const float grad = phi_div(up - lw, g.dx[c] * 2.f, g.inv_dx[c] * 0.5f);
        if (SUB) out.p[c][off] = out.p[c][off] - grad; else out.p[c][off] = grad;
    }
}

// out = sum_c (v_c[i + e_c] - v_c[i - e_c]) / (2 dx_c), ghosts from v.f[c].
// MODE 0: plain (right-hand side).  MODE 1: out = A dir; accumulates dir.out, dir.r and sum(dir) (operator application in the loop).
template <int DIM, int MODE>
__global__ void __launch_bounds__(128)
k_co_divergence(const __grid_constant__ DGrid g, const __grid_constant__ CoVec v, const __grid_constant__ DField cf, float* __restrict__ out,
                const float* __restrict__ dir, const float* __restrict__ r, const unsigned char* __restrict__ cont, double* __restrict__ part,
                size_t slot)
{
    int b, x, y, z;
    const bool in = co_index<DIM>(g, b, x, y, z);
    double a[3] = {0, 0, 0};
    const bool live = in && (MODE == 0 || cont[b]);
    if (live) {
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < DIM; ++c) {
            const float up = phi_fetch<DIM>(v.p[c], g, v.f[c], b, x + (c == 0), y + (c == 1), z + (c == 2));
            const float lw = phi_fetch<DIM>(v.p[c], g, v.f[c], b, x - (c == 0), y - (c == 1), z - (c == 2));
            const float term = phi_div(up - lw, g.dx[c] * 2.f, g.inv_dx[c] * 0.5f);
            acc = (c == 0) ? term : acc + term;
        }
        const long long off = (long long)b * cf.sb + (long long)z * cf.sz + (long long)y * cf.sy + x;
        out[off] = acc;
        if (MODE == 1) { const float d = dir[off]; a[0] = (double)d * acc; a[1] = (double)d * r[off]; a[2] = d; }
    }
    if (MODE == 1) {
        // all threads of a block share b (one grid line per block row)
        const int bb = (DIM == 3) ? blockIdx.z / g.n[2] : blockIdx.z;
        co_block_partials<3>(a, part, g, bb, slot);
    }
}

// Element-wise pieces of the CG-adaptive iteration (_linalg.py:109-122); q = A dir + c * sum(dir) with c = matrix_offset.
//   PHASE 0 (initial residual): r = y - mean - q(x0) with sh.sum1 = sum(x0); dir = r; block partials of |r|^2 and |y|^2
//   PHASE 1: step = (dir.r) / (dir.q); x += step dir; r -= step q; block partials of |r|^2 and r.q
//   PHASE 2: dir = r - ((r.q) / (dir.q)) dir  (k_co_control then advances the iteration count and the stopping rule)
// The offset terms are formed here from the double sums, not taken from cg_balance's rounded sh.offs: nvcc contracts
// q + c * (float)sum into one FFMA, and the bits of the solve depend on it.
template <int DIM, int PHASE>
__global__ void __launch_bounds__(128)
k_co_update(const __grid_constant__ DGrid g, const __grid_constant__ DField cf, float* __restrict__ x, float* __restrict__ r, float* __restrict__ dir,
            const float* __restrict__ q, const float* __restrict__ y, float offset, const CgShared sh, const CoDots d,
            double* __restrict__ part, size_t slot)
{
    int b, xx, yy, zz;
    const bool in = co_index<DIM>(g, b, xx, yy, zz);
    const int bb = (DIM == 3) ? blockIdx.z / g.n[2] : blockIdx.z;
    const long long off = (long long)bb * cf.sb + (long long)zz * cf.sz + (long long)yy * cf.sy + xx;
    double a[2] = {0, 0};
    if (PHASE == 0) {
        if (in) {
            const float yv = y[off] - sh.mean[bb];
            const float rv = yv - (q[off] + offset * (float)sh.sum1[bb]);
            r[off] = rv; dir[off] = rv;
            a[0] = (double)rv * rv; a[1] = (double)yv * yv;
        }
        co_block_partials<2>(a, part, g, bb, slot);
        return;
    }
    if (!sh.cont[bb]) return;
    const double S = d.sd[bb];
    const double dxdy = d.dq[bb] + (double)offset * S * S;              // dir . (A dir + c sum(dir))
    if (PHASE == 1) {
        const float step = dxdy != 0.0 ? (float)(d.dr[bb] / dxdy) : 0.f;  // divide_no_nan
        if (in) {
            const float qv = q[off] + offset * (float)S;
            x[off] = x[off] + step * dir[off];
            const float rv = r[off] - step * qv;
            r[off] = rv;
            a[0] = (double)rv * rv; a[1] = (double)rv * qv;
        }
        co_block_partials<2>(a, part, g, bb, slot);
        return;
    }
    // PHASE 2
    const float coef = dxdy != 0.0 ? (float)(d.rq[bb] / dxdy) : 0.f;
    if (in) dir[off] = r[off] - coef * dir[off];
}

// Per-entry bookkeeping between the phases (cg_common.cuh).  k_co_balance and k_co_control run one thread per batch entry,
// k_co_start and k_co_result one block.
// sum0 = sum(y), sum1 = sum(x0) -> the balanced right-hand side (sh.mean)
__global__ void k_co_balance(const CgShared sh, const PhiCgParams prm, int batch, double cells)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) cg_balance<false>(sh, prm, b, cells);
}

// sum0 = |r0|^2, sum1 = |y|^2 -> tolerance, flags and rsq0 (CG-adaptive's tolerance is relative to |y|^2, _linalg.py:109)
__global__ void k_co_start(const CgShared sh, const PhiCgParams prm, int batch) { cg_start(sh, prm, batch); }

// rr = |r|^2 after the direction update -> iteration count and stopping rule of the running entries
__global__ void k_co_control(const CgShared sh, const PhiCgParams prm, int batch, const double* __restrict__ rr)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch && sh.cont[b]) cg_iteration_done(sh, prm, b, rr[b]);
}

__global__ void k_co_result(const CgShared sh, PhiCgResult* result, int batch) { cg_write_result(sh, result, batch, true); }

// One block per batch entry: sums the block partials of each of up to three values in a fixed order (a strided pass per thread,
// then a tree over the threads) into out0[b], out1[b], out2[b] (nullptr: fewer values).  cont: skip entries that have stopped -
// their partials were not written.
__global__ void __launch_bounds__(256) k_co_reduce(const double* __restrict__ part, size_t slot, int nblk, const unsigned char* __restrict__ cont,
                                                   double* out0, double* out1, double* out2)
{
    const int b = blockIdx.x;
    if (cont && !cont[b]) return;
    const int nq = out2 ? 3 : (out1 ? 2 : 1);
    __shared__ double red[3][256];
    for (int k = 0; k < nq; ++k) {
        const double* p = part + k * slot + (size_t)b * nblk;
        double s = 0;
        for (int j = threadIdx.x; j < nblk; j += blockDim.x) s += p[j];
        red[k][threadIdx.x] = s;
    }
    __syncthreads();
    for (int h = blockDim.x / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) for (int k = 0; k < nq; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    out0[b] = red[0][0];
    if (nq > 1) out1[b] = red[1][0];
    if (nq > 2) out2[b] = red[2][0];
}

// block partials of sum(y) and sum(x0) per batch entry (x0 == nullptr: 0)
__global__ void __launch_bounds__(128)
k_co_sum(const __grid_constant__ DGrid g, const __grid_constant__ DField cf, const float* __restrict__ y, const float* __restrict__ x0,
         double* __restrict__ part, size_t slot)
{
    int b, x, yy, z;
    const bool in = g.dim == 3 ? co_index<3>(g, b, x, yy, z) : co_index<2>(g, b, x, yy, z);
    const int bb = (g.dim == 3) ? blockIdx.z / g.n[2] : blockIdx.z;
    double v[2] = {0, 0};
    if (in) {
        const long long off = (long long)bb * cf.sb + (long long)z * cf.sz + (long long)yy * cf.sy + x;
        v[0] = y[off];
        if (x0) v[1] = x0[off];
    }
    co_block_partials<2>(v, part, g, bb, slot);
}

static dim3 co_grid(const DGrid& g) { return dim3((g.n[0] + 127) / 128, g.n[1], g.n[2] * g.batch); }
static int co_blocks_per_entry(const DGrid& g) { return (g.n[0] + 127) / 128 * g.n[1] * g.n[2]; }
static size_t co_round(size_t bytes) { return (bytes + 255) / 256 * 256; }
static size_t co_array_bytes(const DGrid& g) { return co_round((size_t)g.cext[0] * g.cext[1] * g.cext[2] * g.batch * sizeof(float)); }
static size_t co_state_bytes(int batch) { return co_round(cg_smem_bytes(batch)); }
static size_t co_dots_bytes(int batch) { return co_round(5 * (size_t)batch * sizeof(double)); }

// r, dir, q, div, 3 gradient components | per-entry state (CgShared) | the CoDots | block partials of up to 3 values per entry,
// each part 256-byte aligned (k_co_reduce reads the partials warp-wide: an unaligned base costs it a sector more per load)
size_t phi_collocated_workspace_bytes(const DGrid& g)
{
    return 7 * co_array_bytes(g) + co_state_bytes(g.batch) + co_dots_bytes(g.batch) + 3 * (size_t)g.batch * co_blocks_per_entry(g) * sizeof(double);
}

// Host-synchronising: reads the per-entry running flags every 8 iterations.
int phi_make_incompressible_collocated(const DGrid& g, const DField vfields[3], const DField vfields0[3], const DField& pf, const DField& cf,
                                       float* const v[3], float* p, const PhiCgParams& prm, PhiCgResult* result,
                                       void* workspace, size_t ws_bytes, cudaStream_t s)
{
    if (ws_bytes < phi_collocated_workspace_bytes(g)) { phi_set_error("collocated: workspace %zu < %zu bytes", ws_bytes, phi_collocated_workspace_bytes(g)); return PHI_ERR_WORKSPACE; }
    const int B = g.batch, tb = (B + 63) / 64;
    const size_t arr = co_array_bytes(g);
    unsigned char* ws = (unsigned char*)workspace;
    float* r = (float*)ws; float* dir = (float*)(ws + arr); float* q = (float*)(ws + 2 * arr); float* div = (float*)(ws + 3 * arr);
    CoOut grad; for (int c = 0; c < 3; ++c) grad.p[c] = (float*)(ws + (4 + c) * arr);
    unsigned char* state = ws + 7 * arr;
    const CgShared sh = cg_carve(state, B);
    double* dots = (double*)(state + co_state_bytes(B));
    const CoDots d = {dots, dots + B, dots + 2 * B, dots + 3 * B, dots + 4 * B};
    const int nblk = co_blocks_per_entry(g);
    const size_t slot = (size_t)B * nblk;
    double* part = (double*)((unsigned char*)dots + co_dots_bytes(B));
    const dim3 grid = co_grid(g), block(128);
    const double cells = (double)g.n[0] * g.n[1] * g.n[2];
    cudaError_t e = cudaMemsetAsync(state, 0, co_state_bytes(B), s);
    if (e) return (int)e;
    CoVec vin, gvec;
    for (int c = 0; c < 3; ++c) { vin.f[c] = vfields[c]; vin.p[c] = v[c]; gvec.f[c] = vfields0[c]; gvec.p[c] = grad.p[c]; }
    const bool d3 = g.dim == 3;
#define CO_LAUNCH(K2, K3, ...) do { if (d3) K3<<<grid, block, 0, s>>>(__VA_ARGS__); else K2<<<grid, block, 0, s>>>(__VA_ARGS__); } while (0)
    // right-hand side: divergence of the input velocity, balanced when the system is rank deficient (fluid.py:145-148, 205-209),
    // and sum(x0) for the offset c 11^T x0 of r0.  sum(x0) is taken only with c != 0: with c = 0 the term c * (float)sum(x0) must
    // be exactly +0, which a negative or non-finite sum would break.
    CO_LAUNCH((k_co_divergence<2, 0>), (k_co_divergence<3, 0>), g, vin, cf, div, nullptr, nullptr, nullptr, part, slot);
    if (prm.balance_rhs || prm.matrix_offset != 0.f) {
        k_co_sum<<<grid, block, 0, s>>>(g, cf, div, prm.matrix_offset != 0.f ? p : nullptr, part, slot);
        k_co_reduce<<<B, 256, 0, s>>>(part, slot, nblk, nullptr, sh.sum0, sh.sum1, nullptr);
        k_co_balance<<<tb, 64, 0, s>>>(sh, prm, B, cells);
    }
    auto apply = [&](const float* vec, bool loop) {          // q = A vec (and, inside the loop, the dot products)
        CO_LAUNCH((k_co_gradient<2, false>), (k_co_gradient<3, false>), g, pf, vec, grad, loop ? sh.cont : nullptr);
        if (loop) {
            CO_LAUNCH((k_co_divergence<2, 1>), (k_co_divergence<3, 1>), g, gvec, cf, q, vec, r, sh.cont, part, slot);
            k_co_reduce<<<B, 256, 0, s>>>(part, slot, nblk, sh.cont, d.dq, d.dr, d.sd);
        } else {
            CO_LAUNCH((k_co_divergence<2, 0>), (k_co_divergence<3, 0>), g, gvec, cf, q, nullptr, nullptr, nullptr, part, slot);
        }
    };
    // r0 = y - (A + c 11^T) x0
    apply(p, false);
    CO_LAUNCH((k_co_update<2, 0>), (k_co_update<3, 0>), g, cf, p, r, dir, q, div, prm.matrix_offset, sh, d, part, slot);
    k_co_reduce<<<B, 256, 0, s>>>(part, slot, nblk, nullptr, sh.sum0, sh.sum1, nullptr);
    k_co_start<<<1, 64, 0, s>>>(sh, prm, B);
    apply(dir, true);
    int h_cont = 1;
    std::vector<unsigned char> hcont(B);
    for (int it = 0; it < prm.max_iter && h_cont; ++it) {
        CO_LAUNCH((k_co_update<2, 1>), (k_co_update<3, 1>), g, cf, p, r, dir, q, div, prm.matrix_offset, sh, d, part, slot);
        k_co_reduce<<<B, 256, 0, s>>>(part, slot, nblk, sh.cont, d.rr, d.rq, nullptr);
        CO_LAUNCH((k_co_update<2, 2>), (k_co_update<3, 2>), g, cf, p, r, dir, q, div, prm.matrix_offset, sh, d, part, slot);
        k_co_control<<<tb, 64, 0, s>>>(sh, prm, B, d.rr);
        apply(dir, true);
        if ((it & 7) == 7 || it + 1 == prm.max_iter) {
            e = cudaMemcpyAsync(hcont.data(), sh.cont, B, cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s);
            if (e) return (int)e;
            h_cont = 0;
            for (unsigned char c : hcont) h_cont |= c;
        }
    }
    k_co_result<<<1, 64, 0, s>>>(sh, result, B);
    // v -= grad p
    CoOut vout; for (int c = 0; c < 3; ++c) vout.p[c] = v[c];
    CO_LAUNCH((k_co_gradient<2, true>), (k_co_gradient<3, true>), g, pf, p, vout, nullptr);
#undef CO_LAUNCH
    return (int)cudaGetLastError();
}

// y = divergence_centered(gradient_centered(x)): fluid.masked_laplace(wide_stencil=True) on its own (matrix_offset estimate, tests)
int phi_wide_laplace(const DGrid& g, const DField vfields0[3], const DField& pf, const DField& cf, const float* x, float* y,
                     void* workspace, size_t ws_bytes, cudaStream_t s)
{
    const size_t arr = co_array_bytes(g);
    if (ws_bytes < 3 * arr) { phi_set_error("wide_laplace: workspace %zu < %zu bytes", ws_bytes, 3 * arr); return PHI_ERR_WORKSPACE; }
    CoOut grad; CoVec gvec;
    for (int c = 0; c < 3; ++c) { grad.p[c] = (float*)((unsigned char*)workspace + c * arr); gvec.f[c] = vfields0[c]; gvec.p[c] = grad.p[c]; }
    const dim3 grid = co_grid(g), block(128);
    if (g.dim == 3) {
        k_co_gradient<3, false><<<grid, block, 0, s>>>(g, pf, x, grad, nullptr);
        k_co_divergence<3, 0><<<grid, block, 0, s>>>(g, gvec, cf, y, nullptr, nullptr, nullptr, nullptr, 0);
    } else {
        k_co_gradient<2, false><<<grid, block, 0, s>>>(g, pf, x, grad, nullptr);
        k_co_divergence<2, 0><<<grid, block, 0, s>>>(g, gvec, cf, y, nullptr, nullptr, nullptr, nullptr, 0);
    }
    return (int)cudaGetLastError();
}
