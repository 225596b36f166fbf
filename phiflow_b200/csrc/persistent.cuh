// Persistent cooperative kernels: the grid barrier between the phases of one launch and the host-side fit query and launch
// (ring_kernels.cu: the reaction-diffusion and wave steppers; sph_kernels.cu: the SPH stepper).
#pragma once
#include <cooperative_groups.h>
#include "phi_internal.cuh"

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }

// Between two phases: the generic-proxy stores of one phase must be visible to the TMA (async proxy) loads of the next one, whose
// halo lines other CTAs wrote - the sequence k_cg_ring uses between passes.
__device__ __forceinline__ void step_grid_sync(cooperative_groups::grid_group& grid)
{
    fence_proxy_async();
    grid.sync();
    fence_proxy_async();
}

// Sets the dynamic shared memory of fn, sizes the grid from its occupancy (at most max_ctas CTAs) and launches it cooperatively with
// args; *grid = the CTAs launched.  -100: not even one CTA fits on an SM.  name: the caller, in the error message of a failed launch.
int phi_launch_cooperative(const void* fn, int threads, size_t smem, long long max_ctas, void** args, const char* name, cudaStream_t s,
                           int* grid);
