// N12 SPH (the SPH notebook's dam break, phi/physics/sph.py): every substep of a call in one cooperative persistent launch.
//
// One substep is apply_bounds(sph_step(v)) of the notebook with the poly6 kernel and a hash-grid neighbour search
// (PhiML's find_neighbors_sparse / build_hash_grid).  Its phases, separated by grid barriers:
//   A  bin: cell of every particle (trunc((x - lower) / cell), clamped into [0, res - 1]); count per cell, rank inside the cell
//   B1 sum of the counts over each CTA's chunk of cells;  B2 exclusive scan of the counts into start[], counts reset to 0
//   C  scatter: order[start[cell] + rank] = particle;     D  sort every occupied cell's list by particle index (insertion sort) and
//      copy x and v into that slot order
//   E  density rho_i = (sum_j W_ij) m over the 3^DIM neighbour cells
//   F  force, kick, drift and bounds; the new state goes to the other buffer, so every force reads the old state.  F also runs
//      the next substep's A on the new position, so a substep costs six grid barriers.
// E and F take the particles in slot order and read x, v and rho in slot order: the threads of a warp walk the same neighbour cells,
// and a row of three neighbour cells is one contiguous range of slots.
// Summation order: each particle walks the neighbour cells in the order of PhiML's neighbour offsets (meshgrid(-1, 0, 1) with
// indexing 'ij': x outermost) and each cell's particles by ascending index.  That order is a property of the particles alone, so
// the result depends neither on the atomics of phase A nor on the launch geometry.  PhiML walks the same cells in the same order,
// but orders a cell's particles by NumPy's unstable argsort; tests/oracle_sph.py states the sums this kernel forms.
// Every operation is an explicitly rounded intrinsic: nothing is contracted into an FMA.
#include <algorithm>
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include "launch.cuh"
#include "persistent.cuh"

namespace cg = cooperative_groups;

#define SPH_THREADS 256

namespace {

struct SphBufs {
    int* count;     // [ncells]: particles per cell (zero between substeps)
    int* start;     // [ncells + 1]: first slot of every cell in `order`
    int* bsum;      // [SPH_MAX_CTAS]: counts per CTA chunk
    int* cell;      // [n]: linear cell of every particle
    int* rank;      // [n]: slot of the particle inside its cell, as phase A's atomic handed it out
    int* order;     // [n]: particles in cell order, ascending index inside a cell
    float* x2;      // [n * DIM], [n * DIM]: the second state buffer
    float* v2;
    float* xc;      // [n * DIM], [n * DIM], [n]: x, v and rho in the slot order of `order`
    float* vc;
    float* rhoc;
    float* rho;     // [n]: rho by particle
};

template <int DIM>
__device__ __forceinline__ int sph_cell(const SphParams& p, const float* x, int* c)
{
    int id = 0;
#pragma unroll
    for (int a = 0; a < DIM; ++a) {
        // cvt.rzi: NaN -> 0, beyond the int range -> INT_MIN / INT_MAX; the clamp keeps every cell in range
        const int k = __float2int_rz(__fdiv_rn(__fsub_rn(x[a], p.lower[a]), p.cell[a]));
        c[a] = k < 0 ? 0 : (k > p.res[a] - 1 ? p.res[a] - 1 : k);
        id = id * p.res[a] + c[a];
    }
    return id;
}

// Calls f(slot) for every slot of `order` in the 3^DIM cells around cell c (those inside the grid), in summation order.  The three
// cells along the last axis are consecutive in `order`, so each row of them is one range of slots: 9 ranges in 3-D, 3 in 2-D.
template <int DIM, class Fn>
__device__ __forceinline__ void sph_visit(const SphParams& p, const SphBufs& b, const int* c, Fn&& f)
{
    constexpr int L = DIM - 1;
    const int lo = max(c[L] - 1, 0), hi = min(c[L] + 1, p.res[L] - 1);
    for (int o = 0; o < (DIM == 3 ? 9 : 3); ++o) {
        int id = 0;
        bool inside = true;
#pragma unroll
        for (int a = 0; a < L; ++a) {
            const int k = c[a] + (DIM == 3 && a == 0 ? o / 3 : o % 3) - 1;
            inside = inside && k >= 0 && k < p.res[a];
            id = id * p.res[a] + k;
        }
        if (!inside) continue;
        id *= p.res[L];
        const int end = b.start[id + hi + 1];
        for (int s = b.start[id + lo]; s < end; ++s) f(s);
    }
}

// delta = x_j - x_i, r2 = sum(delta ** 2) in axis order; the pair is stored when sqrt(r2) < s
template <int DIM>
__device__ __forceinline__ bool sph_pair(const SphParams& p, const float* xi, const float* xj, float* d, float& r2)
{
    r2 = 0.f;
#pragma unroll
    for (int a = 0; a < DIM; ++a) {
        d[a] = __fsub_rn(xj[a], xi[a]);
        r2 = a == 0 ? __fmul_rn(d[0], d[0]) : __fadd_rn(r2, __fmul_rn(d[a], d[a]));
    }
    return __fsqrt_rn(r2) < p.s;
}

// Phase A for particle i at x: its cell, and its slot in the cell's count
template <int DIM>
__device__ __forceinline__ void sph_bin(const SphParams& p, const SphBufs& b, int i, const float* x)
{
    int c[DIM];
    const int id = sph_cell<DIM>(p, x, c);
    b.cell[i] = id;
    b.rank[i] = atomicAdd(b.count + id, 1);
}

template <int DIM>
__global__ void __launch_bounds__(SPH_THREADS, 4)      // 64 registers: without the hint ptxas caps the 2-D kernel at 48 and spills
k_sph(SphParams p, SphBufs b, const float* x, const float* v, float* xo, float* vo, int substeps)
{
    using Reduce = cub::BlockReduce<int, SPH_THREADS>;
    using Scan = cub::BlockScan<int, SPH_THREADS>;
    __shared__ union { typename Reduce::TempStorage r; typename Scan::TempStorage s; } tmp;
    __shared__ int s_off;
    cg::grid_group grid = cg::this_grid();
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    const float s2 = __fmul_rn(p.s, p.s);
    const float* xs = x;
    const float* vs = v;
    // A of the first substep; every later substep's A runs in the previous substep's phase F
    for (int i = tid; i < p.n; i += stride) sph_bin<DIM>(p, b, i, xs + (long long)i * DIM);
    for (int step = 0; step < substeps; ++step) {
        float* xd = ((substeps - 1 - step) & 1) ? b.x2 : xo;
        float* vd = ((substeps - 1 - step) & 1) ? b.v2 : vo;
        step_grid_sync(grid);
        // B1.  CTA b scans the cells [c0, c1), thread t the run [r0, r1) of them
        const int chunk = (p.ncells + gridDim.x - 1) / gridDim.x;
        const int c0 = min(blockIdx.x * chunk, p.ncells), c1 = min(c0 + chunk, p.ncells);
        const int run = (c1 - c0 + blockDim.x - 1) / blockDim.x;
        const int r0 = min(c0 + (int)threadIdx.x * run, c1), r1 = min(r0 + run, c1);
        int sum = 0;
        for (int c = r0; c < r1; ++c) sum += b.count[c];
        const int csum = Reduce(tmp.r).Sum(sum);
        if (threadIdx.x == 0) b.bsum[blockIdx.x] = csum;
        step_grid_sync(grid);
        // B2: starts of this CTA's cells; the counts go back to 0 for the next substep's A
        int off = 0;
        for (int k = threadIdx.x; k < (int)blockIdx.x; k += blockDim.x) off += b.bsum[k];
        off = Reduce(tmp.r).Sum(off);
        if (threadIdx.x == 0) s_off = off;
        __syncthreads();
        int ex;
        Scan(tmp.s).ExclusiveSum(sum, ex);
        int at = s_off + ex;
        for (int c = r0; c < r1; ++c) { const int k = b.count[c]; b.start[c] = at; b.count[c] = 0; at += k; }
        if (tid == 0) b.start[p.ncells] = p.n;
        step_grid_sync(grid);
        // C
        for (int i = tid; i < p.n; i += stride) b.order[b.start[b.cell[i]] + b.rank[i]] = i;
        step_grid_sync(grid);
        // D: the particle of rank 0 of every occupied cell sorts it and copies its particles' x and v into slot order
        for (int i = tid; i < p.n; i += stride) {
            if (b.rank[i] != 0) continue;
            const int c = b.cell[i], lo = b.start[c], hi = b.start[c + 1];
            for (int k = lo + 1; k < hi; ++k) {
                const int e = b.order[k];
                int m = k;
                for (; m > lo && b.order[m - 1] > e; --m) b.order[m] = b.order[m - 1];
                b.order[m] = e;
            }
            for (int k = lo; k < hi; ++k) {
                const int j = b.order[k];
#pragma unroll
                for (int a = 0; a < DIM; ++a) { b.xc[(long long)k * DIM + a] = xs[(long long)j * DIM + a]; b.vc[(long long)k * DIM + a] = vs[(long long)j * DIM + a]; }
            }
        }
        step_grid_sync(grid);
        // E, in slot order: neighbouring threads walk the same cells
        for (int k = tid; k < p.n; k += stride) {
            float xi[DIM];
            int c[DIM];
#pragma unroll
            for (int a = 0; a < DIM; ++a) xi[a] = b.xc[(long long)k * DIM + a];
            sph_cell<DIM>(p, xi, c);
            float acc = 0.f;
            sph_visit<DIM>(p, b, c, [&](int s) {
                float d[DIM], r2;
                if (!sph_pair<DIM>(p, xi, b.xc + (long long)s * DIM, d, r2)) return;
                const float diff = __fsub_rn(s2, r2);
                acc = __fadd_rn(acc, __fmul_rn(p.norm, __fmul_rn(__fmul_rn(diff, diff), diff)));
            });
            const float rho = __fmul_rn(acc, p.m);
            b.rhoc[k] = rho;
            b.rho[b.order[k]] = rho;
        }
        step_grid_sync(grid);
        // F, in slot order; A of the next substep on the new position
        const bool bin = step + 1 < substeps;
        for (int k = tid; k < p.n; k += stride) {
            float xi[DIM], vi[DIM], f[DIM];
            int c[DIM];
#pragma unroll
            for (int a = 0; a < DIM; ++a) { xi[a] = b.xc[(long long)k * DIM + a]; vi[a] = b.vc[(long long)k * DIM + a]; f[a] = 0.f; }
            sph_cell<DIM>(p, xi, c);
            const float rho_i = b.rhoc[k];
            const float p_i = __fmul_rn(p.iso, __fsub_rn(rho_i, p.base));
            sph_visit<DIM>(p, b, c, [&](int s) {
                float d[DIM], r2;
                if (!sph_pair<DIM>(p, xi, b.xc + (long long)s * DIM, d, r2)) return;
                const float rho_j = b.rhoc[s];
                const float p_j = __fmul_rn(p.iso, __fsub_rn(rho_j, p.base));
                const float dist = __fsqrt_rn(fmaxf(r2, 1e-5f));
                const float gap = __fsub_rn(p.h, dist), gap2 = __fmul_rn(gap, gap);
                const float avg = __fdiv_rn(__fadd_rn(p_i, p_j), __fmul_rn(2.f, rho_j));
#pragma unroll
                for (int a = 0; a < DIM; ++a) {
                    const float pf = __fmul_rn(__fmul_rn(-__fdiv_rn(d[a], dist), avg), gap2);
                    const float vf = __fmul_rn(__fdiv_rn(__fsub_rn(b.vc[(long long)s * DIM + a], vi[a]), rho_j), gap);
                    f[a] = __fadd_rn(f[a], __fadd_rn(__fmul_rn(p.P, pf), __fmul_rn(p.V, vf)));
                }
            });
            const int i = b.order[k];
#pragma unroll
            for (int a = 0; a < DIM; ++a) {
                const float acc = __fadd_rn(__fdiv_rn(f[a], rho_i), p.gravity[a]);
                float vn = __fadd_rn(vi[a], __fmul_rn(acc, p.dt));
                const float xa = __fadd_rn(xi[a], __fmul_rn(p.dt, vn));
                // np.clip: NaN stays NaN (and compares unequal, so its velocity is damped as in the reference)
                xi[a] = xa < p.lower[a] ? p.lower[a] : (xa > p.upper[a] ? p.upper[a] : xa);
                if (!(xi[a] == xa)) vn = __fmul_rn(vn, p.damping);
                xd[(long long)i * DIM + a] = xi[a];
                vd[(long long)i * DIM + a] = vn;
            }
            if (bin) sph_bin<DIM>(p, b, i, xi);
        }
        xs = xd;
        vs = vd;
    }
}

// Carves the scratch into SphBufs (256-byte aligned pieces); returns the bytes used.  base may be 0 to size the scratch.
size_t sph_layout(const SphParams& p, void* base, SphBufs* b)
{
    size_t off = 0;
    auto carve = [&](size_t bytes) {
        void* r = reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(base) + off);
        off += (bytes + 255) / 256 * 256;
        return r;
    };
    b->count = static_cast<int*>(carve((size_t)p.ncells * sizeof(int)));
    b->start = static_cast<int*>(carve(((size_t)p.ncells + 1) * sizeof(int)));
    b->bsum = static_cast<int*>(carve(SPH_MAX_CTAS * sizeof(int)));
    b->cell = static_cast<int*>(carve((size_t)p.n * sizeof(int)));
    b->rank = static_cast<int*>(carve((size_t)p.n * sizeof(int)));
    b->order = static_cast<int*>(carve((size_t)p.n * sizeof(int)));
    b->x2 = static_cast<float*>(carve((size_t)p.n * p.dim * sizeof(float)));
    b->v2 = static_cast<float*>(carve((size_t)p.n * p.dim * sizeof(float)));
    b->xc = static_cast<float*>(carve((size_t)p.n * p.dim * sizeof(float)));
    b->vc = static_cast<float*>(carve((size_t)p.n * p.dim * sizeof(float)));
    b->rhoc = static_cast<float*>(carve((size_t)p.n * sizeof(float)));
    b->rho = static_cast<float*>(carve((size_t)p.n * sizeof(float)));
    return off;
}

}  // namespace

size_t phi_sph_scratch_bytes(const SphParams& p)
{
    SphBufs b;
    return sph_layout(p, nullptr, &b);
}

int phi_launch_sph(const SphParams& p, const float* x, const float* v, float* xo, float* vo, float* rho, void* scratch, int substeps,
                   int max_ctas, cudaStream_t s)
{
    SphBufs b;
    sph_layout(p, scratch, &b);
    cudaError_t e = cudaMemsetAsync(b.count, 0, (size_t)p.ncells * sizeof(int), s);
    if (e != cudaSuccess) return (int)e;
    const void* fn = p.dim == 3 ? (const void*)k_sph<3> : (const void*)k_sph<2>;
    SphParams pa = p; int ns = substeps;
    void* args[] = {&pa, &b, &x, &v, &xo, &vo, &ns};
    // enough CTAs for the particles and for the cells (a thread scans at most 16 cells per substep)
    long long cap = (std::max((long long)p.n, ((long long)p.ncells + 15) / 16) + SPH_THREADS - 1) / SPH_THREADS;
    if (cap < 1) cap = 1;
    if (cap > max_ctas) cap = max_ctas;
    int grid = 0;
    const int r = phi_launch_cooperative(fn, SPH_THREADS, 0, cap, args, "sph", s, &grid);
    if (r != 0) return r;
    PhiLaunchInfo li = {}; li.kernel = PHI_KERNEL_SPH; li.grid_ctas = grid;
    phi_note_launch(li);
    if (rho) {
        e = cudaMemcpyAsync(rho, b.rho, (size_t)p.n * sizeof(float), cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}
