// N10  Julia sets: the Julia_Set notebook's escape counts (examples/grids/Julia_Set.ipynb), one thread per (batch entry, cell).
//
//   z_0 = x_i + i y_j;   for t < iterations:  count += abs(z_t) < 2;  z_{t+1} = z_t ** 2 + c_b
//
// rounded as PhiML's NumPy backend rounds complex64 on an AVX-512 CPU (tests/oracle_julia.py, tests/golden/phiml_julia.npz):
//   z ** 2 + c:  re' = fl(fl(fl(a a) - fl(b b)) + c_re),  im' = fl(fl(fl(a b) + fl(a b)) + c_im)     (np.power, no fma)
//   abs(z):      fl(big * fl(sqrt(fma(r, r, 1)))),  r = fl(small / big),  big / small = max / min(|a|, |b|)
// Every operation is an explicitly rounded intrinsic, so nvcc can neither contract nor reassociate it.
//
// The band.  The exact abs costs a divide and a square root; the loop tests s = fma(a, a, fl(b b)) instead (fl(b b) is needed for
// re' too) and takes the exact formula only for s in [JULIA_LO, JULIA_HI] = 4 (1 -+ 2^-20).  With u = 2^-24 and |z|^2 = a^2 + b^2:
//   s = (a^2 + b^2 (1 + d1)) (1 + d2), |d| <= u, so  |s / |z|^2 - 1| <= 2u + u^2 < 2.01u;
//   abs = |z| (1 + e) with |e| < 3.01u: r^2 is off by at most 2.01u relative, which moves 1 + r^2 by at most half of that (r <= 1);
//   the fma, the square root (halving its input's error) and the product add u each.
//   s < 4 (1 - 16u)  =>  |z|^2 < 4 (1 - 16u) / (1 - 2.01u) < 4 (1 - 13.9u)  =>  abs < 2 (1 - 6.9u)(1 + 3.01u) < 2: inside.
//   s > 4 (1 + 16u)  =>  |z|^2 > 4 (1 + 13.9u)  =>  abs > 2 (1 + 6.9u)(1 - 3.01u) > 2: outside.
// A NaN s (NaN in z) fails both tests and counts as outside, as abs(z) < 2 is False for NumPy's NaN or inf abs; the exact formula
// therefore only ever sees finite z with |z| near 2.  tests/test_julia_host.py checks the shortcut against the formula at the band's
// edges.
//
// Early exit.  For |c_re|, |c_im| <= 4 (|c| < 5.66) a thread stops at the first s > 16: no later abs is below 2.  Proof: s > 16
// gives |z| > 4 (1 - 1.01u) =: R.  One step: fl(z^2) is z^2 with an error below 2.25u |z|^2 (the re part is off by at most
// u (a^2 + b^2 + |a^2 - b^2|)(1 + u) <= 2.01u |z|^2, the im part by u |2ab| <= u |z|^2), adding c and rounding loses at most 5.66 and a factor
// (1 - u), so |z'| >= (R^2 (1 - 2.25u) - 5.66)(1 - u) > 10 > R.  By induction every later finite z has |z| > R and abs > 3.9; a z
// that overflows to inf or NaN stays non-finite (fma(inf, inf, x) is inf or NaN, NaN propagates) and never counts.  Above the bound
// the thread runs every iteration, and inf / NaN decide as in NumPy.
#include "phi_internal.cuh"
#include "launch.cuh"

#define JULIA_THREADS 128
#define JULIA_LO (4.0f - 0x1p-18f)       // 4 (1 - 2^-20)
#define JULIA_HI (4.0f + 0x1p-18f)       // 4 (1 + 2^-20)
#define JULIA_ESCAPE 16.0f               // |z| > ~4: escaped for good when |c_re|, |c_im| <= JULIA_CMAX
#define JULIA_CMAX 4.0f

// NumPy's abs of a complex64 with finite components, not both 0
__device__ __forceinline__ float julia_abs(float a, float b)
{
    const float x = fabsf(a), y = fabsf(b);
    const float big = fmaxf(x, y), small = fminf(x, y);
    const float r = __fdiv_rn(small, big);
    return __fmul_rn(big, __fsqrt_rn(__fmaf_rn(r, r, 1.0f)));
}

// grid (ceil(nx / JULIA_THREADS), ny, batch); counts[b][y][x] at b * sb + y * sy + x (the centred-array layout, 64-bit offsets)
__global__ void __launch_bounds__(JULIA_THREADS)
k_julia(const float2* __restrict__ c, const float* __restrict__ xc, const float* __restrict__ yc, int nx, long long sy, long long sb,
        int iterations, int32_t* __restrict__ counts)
{
    const int x = blockIdx.x * JULIA_THREADS + threadIdx.x;
    if (x >= nx) return;
    const int y = blockIdx.y, b = blockIdx.z;
    const float2 cb = c[b];
    const bool may_exit = fabsf(cb.x) <= JULIA_CMAX && fabsf(cb.y) <= JULIA_CMAX;     // false for inf / NaN
    float re = xc[x], im = yc[y];
    int count = 0;
    for (int t = 0; t < iterations; ++t) {
        const float b2 = __fmul_rn(im, im);
        const float s = __fmaf_rn(re, re, b2);
        if (s < JULIA_LO) ++count;
        else if (s <= JULIA_HI) count += julia_abs(re, im) < 2.0f;
        else if (may_exit && s > JULIA_ESCAPE) break;
        const float ab = __fmul_rn(re, im);
        re = __fadd_rn(__fsub_rn(__fmul_rn(re, re), b2), cb.x);
        im = __fadd_rn(__fadd_rn(ab, ab), cb.y);
    }
    counts[(long long)b * sb + (long long)y * sy + x] = count;
}

int phi_launch_julia(const DGrid& g, const float* c, const float* xc, const float* yc, int iterations, int32_t* counts, cudaStream_t s)
{
    const dim3 grid((g.n[0] + JULIA_THREADS - 1) / JULIA_THREADS, g.n[1], g.batch);
    const long long sy = g.cext[0], sb = (long long)g.cext[0] * g.cext[1];
    k_julia<<<grid, JULIA_THREADS, 0, s>>>(reinterpret_cast<const float2*>(c), xc, yc, g.n[0], sy, sb, iterations, counts);
    PhiLaunchInfo li = {}; li.kernel = PHI_KERNEL_JULIA;
    phi_note_launch(li);
    return (int)cudaGetLastError();
}
