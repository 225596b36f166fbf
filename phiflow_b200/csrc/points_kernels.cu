// N11  advect.points: world-space points moved through a StaggeredGrid velocity (phi/physics/advect.py:20-35, 136-153), Euler or
// RK4, every step of a trajectory in one launch.  One thread per (batch entry, point); the position stays in registers.
//
// One velocity sample at p (sample_staggered_grid, phi/field/_resample.py:276-284), for every component c:
//   idx_a = fl(fl(fl(fl(p_a - lower'_ca) / size'_ca) * res'_ca) - 0.5)          (Box.global_to_local, _resample.py:257)
// with the component grid's bounds and resolution (UniformGrid.stagger, phi/geom/_grid.py:204-209) as the caller computes them, then
// math.grid_sample of component c at idx with its own boundary (_closest_grid_values, PhiML/phiml/math/_ops.py:902-933, and the
// fallback of _grid_sample, :1010-1014):
//   frac_a = fl(idx_a - floor(idx_a))                                            (idx % 1; NaN for a non-finite idx)
//   k_a    = int32(floor(fl(idx_a + s_a)))   s_a = 1 where the lower side is a constant (the grid is padded there by one ghost
//                                            layer and the coordinate shifted in float32), else 0
//   neighbours k_a, k_a + 1 of the padded axis: PERIODIC mod n, otherwise clamped to the padded range
// int32(x) is NumPy's float32 -> int32 cast on x86 (recorded in the fixture): the truncated value for |x| < 2^31, INT_MIN for NaN,
// +-inf and |x| >= 2^31.  Any index then stays safe:
//   * non-periodic axes: every k <= -2 and every k >= N (N = stored count + constant ghosts) select the same clamped pair as
//     k = -2 and k = N, so k is clamped to [-2, N] first; the stored index k - s + lo then lies in [lo - 3, hi + 2] and phi_resolve
//     maps it (and k + 1) onto the clamped stored index or the side's constant, the same value the padded array holds there.
//   * periodic axes: k mod n is taken in int (INT_MIN % n is defined for n >= 1), which equals PhiML's (k mod n) and gives
//     (k + 1) mod n through phi_resolve's wrap of lo + n.
// No index arithmetic overflows, and only stored values are read; a non-finite coordinate yields NaN through frac, as in PhiML.
//
// Integrators (Python scalars times float32 tensors round as f32(c) * x; h = 0.5 dt is exact):
//   Euler:  p + fl(v0 * dt)
//   RK4:    vh = v(p + fl(h vh0)), vh2 = v(p + fl(h vh)), v1 = v(p + fl(dt vh2)),
//           p + fl(dt * fl(f32(1/6) * fl(fl(v0 + fl(2 fl(vh + vh2))) + v1)))
// Every operation is an explicitly rounded intrinsic (no contraction); the division is __fdiv_rn.
#include <climits>
#include "phi_internal.cuh"
#include "launch.cuh"
#include "fk_interp.cuh"

#define PTS_THREADS 128

// NumPy's float32 -> int32 cast on x86 of an integral value
__device__ __forceinline__ int pts_to_int32(float x)
{
    return (x >= -2147483648.f && x < 2147483648.f) ? __float2int_rz(x) : INT_MIN;
}

// velocity at p: v[c] sampled from component c
template <int DIM>
__device__ __forceinline__ void pts_sample(const DGrid& g, const DVec& vel, const PhiPointMap& m, int b, const float p[3], float v[3])
{
#pragma unroll
    for (int c = 0; c < DIM; ++c) {
        const DField& f = vel.f[c];
        FkLookup L; L.i[2] = 0; L.t[2] = 0.f;
#pragma unroll
        for (int a = 0; a < DIM; ++a) {
            const float idx = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(p[a], m.lower[c][a]), m.size[c][a]), m.res[c][a]), 0.5f);
            L.t[a] = __fsub_rn(idx, floorf(idx));
            const int n = f.hi[a] - f.lo[a] + 1;
            if (f.klo[a] == PHI_BC_PERIODIC) {
                int r = pts_to_int32(floorf(idx)) % n;
                if (r < 0) r += n;
                L.i[a] = f.lo[a] + r;
            } else {
                const int s = f.klo[a] == PHI_BC_CONST, N = n + s + (f.khi[a] == PHI_BC_CONST);
                const int k = min(max(pts_to_int32(floorf(__fadd_rn(idx, (float)s))), -2), N);
                L.i[a] = k - s + f.lo[a];
            }
        }
        v[c] = fk_interp<DIM, true>(vel.p[c], g, f, b, L);
    }
}

// grid-stride over B * npoints threads; point j of batch entry b at (b * npoints + j) * DIM, read from batch entry b * pbs,
// sampled in batch entry b * gbs of the velocity; trajectory entry s at ((s * B + b) * npoints + j) * DIM (64-bit offsets)
template <int DIM, int INTEGRATOR>
__global__ void __launch_bounds__(PTS_THREADS)
k_advect_points(const __grid_constant__ DGrid g, const __grid_constant__ DVec vel, const __grid_constant__ PhiPointMap map,
                const float* points, long long npoints, int B, int pbs, int gbs, float dt, int steps, float* out, float* traj)
{
    const long long total = (long long)B * npoints;
    const float half = __fmul_rn(0.5f, dt), sixth = 1.f / 6.f;
    for (long long t = (long long)blockIdx.x * PTS_THREADS + threadIdx.x; t < total; t += (long long)gridDim.x * PTS_THREADS) {
        const int b = (int)(t / npoints);
        const long long j = t - (long long)b * npoints;
        const int gb = b * gbs;
        float p[3] = {0.f, 0.f, 0.f};
        const float* src = points + ((long long)b * pbs * npoints + j) * DIM;
#pragma unroll
        for (int a = 0; a < DIM; ++a) p[a] = src[a];
        if (traj) {
#pragma unroll
            for (int a = 0; a < DIM; ++a) traj[t * DIM + a] = p[a];
        }
        for (int s = 1; s <= steps; ++s) {
            float v0[3], q[3];
            pts_sample<DIM>(g, vel, map, gb, p, v0);
            if (INTEGRATOR == PHI_INTEGRATOR_EULER) {
#pragma unroll
                for (int a = 0; a < DIM; ++a) p[a] = __fadd_rn(p[a], __fmul_rn(v0[a], dt));
            } else {
                // v0 + 2 (vh + vh2) is formed as soon as vh2 is known, so that only p and it stay live across the last sample
                float vh[3], vh2[3], v1[3];
#pragma unroll
                for (int a = 0; a < DIM; ++a) q[a] = __fadd_rn(p[a], __fmul_rn(half, v0[a]));
                pts_sample<DIM>(g, vel, map, gb, q, vh);
#pragma unroll
                for (int a = 0; a < DIM; ++a) q[a] = __fadd_rn(p[a], __fmul_rn(half, vh[a]));
                pts_sample<DIM>(g, vel, map, gb, q, vh2);
#pragma unroll
                for (int a = 0; a < DIM; ++a) {
                    q[a] = __fadd_rn(p[a], __fmul_rn(dt, vh2[a]));
                    v0[a] = __fadd_rn(v0[a], __fmul_rn(2.f, __fadd_rn(vh[a], vh2[a])));
                }
                pts_sample<DIM>(g, vel, map, gb, q, v1);
#pragma unroll
                for (int a = 0; a < DIM; ++a) p[a] = __fadd_rn(p[a], __fmul_rn(dt, __fmul_rn(sixth, __fadd_rn(v0[a], v1[a]))));
            }
            if (traj) {
#pragma unroll
                for (int a = 0; a < DIM; ++a) traj[((long long)s * total + t) * DIM + a] = p[a];
            }
        }
#pragma unroll
        for (int a = 0; a < DIM; ++a) out[t * DIM + a] = p[a];
    }
}

int phi_launch_advect_points(const DGrid& g, const DVec& vel, const PhiPointMap& map, const float* points, long long npoints,
                             int points_batch, float dt, int integrator, int steps, float* out, float* traj, cudaStream_t s)
{
    const int B = max(g.batch, points_batch);
    const int pbs = points_batch == 1 ? 0 : 1, gbs = g.batch == 1 ? 0 : 1;
    const long long total = (long long)B * npoints;
    const int blocks = (int)min((total + PTS_THREADS - 1) / PTS_THREADS, (long long)phi_sm_count() * 64);
    auto launch = [&](auto kernel) { kernel<<<blocks, PTS_THREADS, 0, s>>>(g, vel, map, points, npoints, B, pbs, gbs, dt, steps, out, traj); };
    if (g.dim == 3) { if (integrator == PHI_INTEGRATOR_RK4) launch(k_advect_points<3, PHI_INTEGRATOR_RK4>); else launch(k_advect_points<3, PHI_INTEGRATOR_EULER>); }
    else            { if (integrator == PHI_INTEGRATOR_RK4) launch(k_advect_points<2, PHI_INTEGRATOR_RK4>); else launch(k_advect_points<2, PHI_INTEGRATOR_EULER>); }
    PhiLaunchInfo li = {}; li.kernel = PHI_KERNEL_POINTS;
    phi_note_launch(li);
    return (int)cudaGetLastError();
}
