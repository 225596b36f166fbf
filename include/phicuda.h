/*
 * phicuda.h  --  C ABI of libphicuda.so: the H100 (sm_90a) incompressible-fluid hot path of PhiFlow.
 *
 * Every entry point replaces one piece of the reference's Python hot path (file:line relative to the PhiFlow tree,
 * PhiML = its vendored arithmetic layer); see DESIGN.md for the data layout and INTEGRATION.md for the ctypes binding.
 *
 * Conventions (SURVEY.md §8b):
 *   - plain C types only; all array arguments are DEVICE pointers unless the name ends in `_host`;
 *   - functions enqueue work on `stream` (a cudaStream_t passed as void*) and return immediately;
 *     they never allocate, free or synchronise.  Exceptions, each saying so at its declaration: the `*_host` calls
 *     (synchronise the stream) and the SET-UP calls of the multi-GPU communicator (phicuda_comm_create / _connect / _destroy:
 *     cudaMalloc + cudaMemset + device synchronisation / CUDA-IPC open / cudaFree - once per run, never inside a step);
 *   - return 0 on success, a negative PHI_ERR_* or a positive cudaError_t otherwise; the message is kept per thread
 *     and read with phicuda_last_error();
 *   - fp32 (`_f32`) throughout (phicuda_julia_f32 computes in float32 and writes int32 counts); fp64 (`_f64`, math.set_global_precision(64)) for the stencils, semi-Lagrangian advection and the
 *     CG pressure projection (see "fp64" below).  Other precisions are not part of this path (the reference falls through to its
 *     stock backends).
 *
 * Device layout (one PhiGrid describes every array that lives on a domain):
 *   element (b, z, y, x)  at  ((b*E[2] + z)*E[1] + y)*E[0] + x               (x contiguous, z-slabs contiguous)
 *   with E = cext for centred arrays (smoke, pressure, divergence) and E = fext for every component of a staggered
 *   array.  Component d of a staggered array stores the value of the face at the LOWER side of cell i at index i along
 *   axis d, so index n[d] is the upper boundary face; it exists only where the boundary stores it (ZERO_GRADIENT),
 *   which requires fext[d] > n[d].  cext[0] and fext[0] are multiples of 4 so every row is 16-byte aligned; for
 *   periodic or closed domains cext == fext == n (rounded up along x).  2-D grids have n[2] = cext[2] = fext[2] = 1.
 */
#ifndef PHICUDA_H
#define PHICUDA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PHICUDA_ABI_VERSION 2

/* boundary kinds per side  (PhiML/phiml/math/extrapolation.py:247 ConstantExtrapolation incl. ZERO/ONE,
 * :544 _ZeroGradient == BOUNDARY, :648 _PeriodicExtrapolation; per-side mixes: combine_sides :1209) */
#define PHI_BC_CONST         0
#define PHI_BC_ZERO_GRADIENT 1
#define PHI_BC_PERIODIC      2
/* Multi-GPU z-slabs only: the side borders another rank's slab.  Neighbour values are read from the `halo` planes that
 * the caller allocated around the owned range and keeps up to date (halo exchange); faces are stored as for PERIODIC. */
#define PHI_BC_HALO          3

#define PHI_ERR_INVALID   (-1)   /* bad argument (message says which) */
#define PHI_ERR_UNSUPPORTED (-2) /* valid in the reference but outside this fast path: caller must fall through */
#define PHI_ERR_WORKSPACE (-3)   /* workspace too small */

typedef struct PhiGrid {
    int32_t dim;        /* 2 or 3 */
    int32_t batch;      /* independent systems (PhiML batch dims, _linalg.py:72-87) */
    int32_t n[3];       /* cells per axis, x first */
    int32_t cext[3];    /* allocated extent of centred arrays   (see layout above) */
    int32_t fext[3];    /* allocated extent of staggered components */
    float   dx[3];      /* cell size = bounds.size / resolution  (phi/geom/_grid.py:117-119) */
    int32_t halo;       /* 3-D z-slabs: planes allocated below AND above the owned range n[2]; array pointers address the
                           first OWNED plane, cext[2] = fext[2] = n[2] + 2*halo.  0 on a single GPU. */
} PhiGrid;

/* Boundary of one scalar array (a centred field or ONE component of a staggered field). */
typedef struct PhiBC {
    uint8_t lo[3], hi[3];      /* PHI_BC_* per axis side */
    float   clo[3], chi[3];    /* constant value where kind == PHI_BC_CONST */
} PhiBC;

/* Boundary of a vector field: one PhiBC per component.  The KINDS must agree between components (they decide which
 * faces are stored, extrapolation.py:57-62 valid_outer_faces); the constants may differ. */
typedef struct PhiVBC {
    PhiBC comp[3];
} PhiVBC;

/* Solver parameters: phiml.math.Solve (PhiML/phiml/math/_optimize.py:25-41) + stop_on_l2 (_linalg.py:23-40). */
typedef struct PhiCgParams {
    float   rtol;            /* relative to the INITIAL residual |y - A x0| (_linalg.py:61-67) */
    float   atol;
    int32_t max_iter;        /* Solve.max_iterations, default 1000 */
    int32_t balance_rhs;     /* 1: subtract mean(rhs) per batch entry (fluid._balance_divergence, fluid.py:205-209) */
    int32_t project_mean;    /* 1: remove mean(x) at the end (the rank-1 matrix_offset of _optimize.py:705-714 selects
                                the zero-mean solution of the singular system) */
    float   matrix_offset;   /* c of (A + c 1 1^T); 0 = plain CG on the range space */
    int32_t method;          /* PHI_SOLVER_CG: Shewchuk CG (_linalg.py:52-90);  PHI_SOLVER_CG_ADAPTIVE: the Hestenes-Stiefel
                                variant behind Solve('CG-adaptive') and, in PhiML 1.7, Solve('auto') (_linalg.py:93-128,
                                _backend.py:1446): step (d.r)/(d.Ad), direction r - ((r.Ad)/(d.Ad)) d, tolerance relative
                                to |y|^2 (with balance_rhs: the balanced y').  Requires matrix_offset == 0 and the TMA ring
                                kernel, with or without obstacles (single GPU); elsewhere PHI_ERR_UNSUPPORTED. */
} PhiCgParams;
#define PHI_SOLVER_CG 0
#define PHI_SOLVER_CG_ADAPTIVE 1

/* Per batch entry, mirrors SolveResult (PhiML/phiml/backend/_backend.py:24-32). */
typedef struct PhiCgResult {
    int32_t iterations;
    int32_t converged;
    int32_t diverged;
    float   residual_sq;     /* |r|^2 at exit */
    float   tol_sq;          /* max(rtol^2 |r0|^2, atol^2) */
    float   initial_residual_sq;
} PhiCgResult;

/* ---- library ------------------------------------------------------------------------------------------------- */
int         phicuda_abi_version(void);
/* Copies the calling thread's last error message (NUL terminated) into buf; returns its length. */
size_t      phicuda_last_error(char* buf, size_t buf_len);
/* Name, SM count and compute capability of the current device; returns 0 or a cudaError_t. */
int         phicuda_device_info(char* name, size_t name_len, int* sm_count, int* cc_major, int* cc_minor);

/* Diagnostics: which kernel variant the calling thread's most recent laplace / CG launch selected.  The parity tests use
 * it to assert that a case really ran on the instantiation it was written for (e.g. the branch-free TMA-ring variant that
 * bench.py times) instead of silently taking another path. */
#define PHI_KERNEL_NONE          0
#define PHI_KERNEL_LAPLACE_RING  1   /* k_laplace_ring  (TMA ring) */
#define PHI_KERNEL_LAPLACE_MARCH 2   /* k_laplace       (register marching) */
#define PHI_KERNEL_CG_RING       3   /* k_cg_ring       (persistent, TMA ring) */
#define PHI_KERNEL_CG_MARCH      4   /* k_cg_poisson    (persistent, register marching) */
#define PHI_KERNEL_STENCIL_RING  5   /* k_div_ring / k_gradsub_ring / k_advect_ring: see `stencil` */
#define PHI_KERNEL_RD_RING       6   /* k_rd_ring       (persistent, TMA ring): phicuda_reaction_diffusion_f32 */
#define PHI_KERNEL_WAVE_RING     7   /* k_wave_ring     (persistent, TMA ring): phicuda_wave_f32 */
#define PHI_KERNEL_JULIA         8   /* k_julia         (one thread per batch entry and cell): phicuda_julia_f32 */
#define PHI_KERNEL_POINTS        9   /* k_advect_points (one thread per batch entry and point): phicuda_advect_points_f32 */
#define PHI_KERNEL_SPH          10   /* k_sph           (persistent, cooperative; grid_ctas set): phicuda_sph_f32 */
typedef struct PhiLaunchInfo {
    int32_t kernel;        /* PHI_KERNEL_* */
    int32_t generic;       /* 1: variant with per-tile boundary handling, 0: branch-free variant (every tile qualifies) */
    int32_t dist;          /* 1: multi-GPU instantiation (peer halo stores + in-kernel all-reduce) */
    int32_t adaptive;      /* 1: CG-adaptive */
    int32_t masked;        /* 1: obstacle mask variant */
    int32_t TY, stages;    /* tile height (grid lines), ring depth */
    int32_t ZC, nzc;       /* planes per unit, z chunks */
    int32_t groups;        /* float4 groups per consumer thread and plane */
    int32_t total_units;   /* units of the whole launch */
    int32_t grid_ctas;     /* CTAs launched (units per CTA = ceil(total_units / grid_ctas)) */
    int32_t split;         /* CG ring: 1 = tail-split decomposition (CTA c < tiles marches planes [0, ZC), the rest share the tails) */
} PhiLaunchInfo;
int phicuda_last_launch_info(PhiLaunchInfo* out);
/* Sweeps over the grid per iteration of this thread's most recent CG launch: 1 = one-sweep ring CG (3-D, periodic y and z,
 * one GPU, plain CG), 2 = two-sweep kernels (every other case, or PHICUDA_CG_PASSES=2); 0 before the first CG launch. */
int phicuda_last_cg_passes(void);
/* Operator of this thread's most recent CG launch (0 before the first one). */
#define PHI_CG_OP_POISSON           1   /* laplace / masked laplace (pressure solves, cg_poisson) */
#define PHI_CG_OP_HELMHOLTZ         2   /* I - a L0 (diffuse.implicit, plain-number diffusivity) */
#define PHI_CG_OP_HELMHOLTZ_VARYING 3   /* I + D0 with face coefficients min(-dt k) (diffuse.implicit, varying diffusivity) */
int phicuda_last_cg_operator(void);

/* ---- A7  field.laplace order 2 (phi/field/_field_math.py:118-145 -> PhiML/phiml/math/_nd.py:825-861) ------------- */
/* y = sum_d (x[i-1] + x[i+1] - 2 x[i]) / dx_d^2, ghost cells from `bc`.  8 B/cell. */
int phicuda_laplace_f32(const PhiGrid* g, const PhiBC* bc, const float* x, float* y, void* stream);
/* y = x + coeff * laplace(x):  diffuse.explicit single sub-step (phi/physics/diffuse.py:13-60). */
int phicuda_laplace_axpy_f32(const PhiGrid* g, const PhiBC* bc, const float* x, float coeff, float* y, void* stream);

/* ---- A5  field.divergence, staggered order 2 (phi/field/_field_math.py:617-626, bake_extrapolation :20-39) ---- */
int phicuda_divergence_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const v[3], float* div, void* stream);

/* ---- A6  v -= spatial_gradient(p, at='face')  (phi/physics/fluid.py:158-161, _field_math.py:229-236, 535-581) -----
 * The pressure boundary is derived from vbc as fluid._pressure_extrapolation does (fluid.py:264-274). */
int phicuda_grad_sub_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], const float* p, void* stream);

/* ---- A9-A11  advect.semi_lagrangian with the euler integrator (phi/physics/advect.py:156-179, 20-24) ------------
 * Back-trace from every sample point of the advected field with the velocity sampled there (shift resampling,
 * phi/field/_resample.py:341-364) and interpolate n-linearly (PhiML/phiml/math/_ops.py:936-1015).
 * centred:   src/dst one array with boundary fbc[0];   staggered: `dim` component arrays with boundaries fbc->comp[c]
 * (the advected staggered field must store the same faces as one with boundary kinds fbc).  dst must not alias src. */
int phicuda_advect_centered_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const vel[3],
                                const PhiBC* fbc, const float* src, float* dst, float dt, void* stream);
int phicuda_advect_staggered_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const vel[3],
                                 const PhiVBC* fbc, const float* const src[3], float* const dst[3], float dt, void* stream);
/* A11 alone: math.grid_sample (PhiML/phiml/math/_ops.py:936-1015) = Backend.grid_sample of the reference-side plugin
 * (PhiML/phiml/backend/_backend.py:1578-1593).  out[b][i] = n-linear interpolation of the centred array grid[b] at
 * coords[b][i][0..dim) (index space: 0 = first cell centre, x first), neighbours outside follow `bc`. */
int phicuda_grid_sample_f32(const PhiGrid* g, const PhiBC* bc, const float* grid, const float* coords, int64_t npoints,
                            float* out, void* stream);
/* N1  advect.mac_cormack for a centred field (phi/physics/advect.py:182-215); tmp = one scratch array. */
int phicuda_mac_cormack_centered_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const vel[3],
                                     const PhiBC* fbc, const float* src, float* dst, float* tmp,
                                     float dt, float correction_strength, void* stream);

/* ---- N2  small per-step helpers of the notebook step (examples/grids/Smoke_Plume.ipynb:58-68) --------------------
 * y += a * x over the cells of a centred array (inflow: s += rate * mask). */
int phicuda_axpy_centered_f32(const PhiGrid* g, float a, const float* x, float* y, void* stream);
/* v_c += dt * resample(s * b_c, to=faces of c)  (sample_grid_at_faces, phi/field/_resample.py:272-276). */
int phicuda_add_buoyancy_f32(const PhiGrid* g, const PhiVBC* vbc, const PhiBC* sbc, const float* s,
                             const float b[3], float dt, float* const v[3], void* stream);

/* out[c] = max |v_c| over the stored faces of the owned planes, c < dim (out: 3 floats on the device).  The semi-Lagrangian
 * back-trace is unbounded in the reference (phi/physics/advect.py:20-24); z-slab runs size the advection halo
 * h = ceil(max|v_z| dt / dz) + 1 from it before every step (SURVEY.md section 8e).  NaN is reported as +inf. */
int phicuda_max_abs_velocity_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const v[3], float* out, void* stream);

/* ---- A2 + A12  pressure solve: CG on the matrix-free Poisson operator ------------------------------------------
 * Replaces math.solve_linear(masked_laplace, div, Solve('CG', ...)) (phi/physics/fluid.py:156,
 * PhiML/phiml/math/_optimize.py:511-745, PhiML/phiml/backend/_linalg.py:52-90).
 * x: in = initial guess x0, out = solution.  result: device array of `batch` PhiCgResult.
 * One persistent cooperative kernel runs the whole solve; no host involvement until the caller reads `result`. */
size_t phicuda_cg_workspace_bytes(const PhiGrid* g);
int phicuda_cg_poisson_f32(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x,
                           const PhiCgParams* prm, PhiCgResult* result, void* workspace, size_t workspace_bytes,
                           void* stream);

/* ---- multi-GPU (one process per GPU, z-slab decomposition; SURVEY.md section 8e) ------------------------------------------
 * The distributed solve is the SAME persistent kernel as phicuda_cg_poisson_f32; in addition every rank
 *   - stores the first / last owned plane of the vectors it updates straight into the neighbour's halo planes through
 *     NVLink peer pointers (the halo exchange is fused into the pass epilogues), and
 *   - closes each dot product by writing its partial sums into every peer's mailbox and summing the mailboxes in rank
 *     order (an all-reduce without leaving the kernel; identical results on all ranks).
 * PhiComm owns one cudaMalloc'd buffer per rank that holds the mailboxes and the CG work vectors; the buffers are
 * exchanged as CUDA IPC handles (64 bytes each) by the caller (e.g. with torch.distributed.all_gather). */
typedef struct PhiComm PhiComm;
#define PHI_IPC_HANDLE_BYTES 64
/* SET-UP calls (allocate / synchronise / free; see the conventions at the top): create allocates this rank's buffer and returns its
 * IPC handle, connect opens the peers' handles, destroy closes them and frees the buffer.  The grid fixes the buffer layout: a
 * communicator serves solves on exactly that PhiGrid (dist.SlabPlume rebuilds it when the halo is re-allocated). */
int phicuda_comm_create(int rank, int nranks, const PhiGrid* g, PhiComm** comm, void* ipc_handle_out);
int phicuda_comm_connect(PhiComm* comm, const void* all_handles /* nranks * 64 bytes, rank order */);
int phicuda_comm_destroy(PhiComm* comm);
/* g describes the LOCAL slab (boundary kind PHI_BC_HALO on interior slab faces); x must carry valid halo planes. */
int phicuda_cg_poisson_dist_f32(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x,
                                const PhiCgParams* prm, PhiCgResult* result, PhiComm* comm, void* stream);
/* N4 on z-slabs: the same with static obstacles; `accessible` carries valid halo planes (exchanged once, the mask is static). */
int phicuda_cg_poisson_dist_masked_f32(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x, const float* accessible,
                                       const PhiCgParams* prm, PhiCgResult* result, PhiComm* comm, void* stream);

/* ---- N5  diffuse.implicit (phi/physics/diffuse.py:63-95) ---------------------------------------------------------------
 * Solves sharpen(x) = x - amount * laplace_bc(x) = y with CG, amount = diffusivity * dt, as the reference's solve_linear does:
 * M x = y - bias, M = I - amount * L0 (L0: laplace with every constant ghost 0), bias = sharpen(0)
 * (PhiML/phiml/math/_optimize.py:616-645).  Same persistent TMA-ring CG as the pressure solve (two sweeps per iteration,
 * phicuda_last_cg_passes() reports 2), single GPU, no z-slabs.
 * components = C in {1, 2, 3}: batch entry b is component b % C of a vector field (a CenteredGrid with a vector channel, or the
 * components of a periodic StaggeredGrid) and uses bc->comp[b % C] (kinds must agree, constants may differ).  Every entry is its
 * own system with its own stopping rule: the reference's tracer keeps the uncoupled vector dim out of the matrix and solves the
 * components as a batch.  x: in = x0, out = solution; x == y is allowed (the reference's default x0 is the field itself).
 * prm: method PHI_SOLVER_CG, balance_rhs = project_mean = 0, matrix_offset = 0.  result: `batch` records.
 * workspace: phicuda_cg_workspace_bytes(g).  Grids whose lines do not fit the ring return PHI_ERR_UNSUPPORTED. */
int phicuda_diffuse_implicit_f32(const PhiGrid* g, const PhiVBC* bc, int32_t components, float amount,
                                 const float* y, float* x, const PhiCgParams* prm, PhiCgResult* result,
                                 void* workspace, size_t workspace_bytes, void* stream);

/* ---- N6  diffuse.implicit with a spatially varying diffusivity (phi/physics/diffuse.py:48-59, 90-95, 129-141) ---------------
 * Solves sharpen(x) = explicit(x, k, -dt) = y for a scalar centred field: w = fl(-dt * k) per cell, every face takes
 * f = min(w_lo, w_hi) and sharpen(x) = x + sum_d [f_{i+1/2} (x_{i+1} - x_i) - f_{i-1/2} (x_i - x_{i-1})] / dx_d^2.  The coefficient
 * ghosts follow the field's boundary `bc`, not k's own (amount.at(u), phi/field/_resample.py:56-63): PERIODIC wraps,
 * ZERO_GRADIENT copies the edge, a constant side with value c gives f_b = min(w_edge, c).  For dt > 0 the faces therefore take the
 * MAXIMUM of k.  Solved as M x = y - bias with CG (x0 = x on entry, x == y allowed), M = I + D0 (value ghosts of constant sides
 * 0), bias = sum over constant sides of f_b c / dx^2.  Every batch entry is its own system.
 * diffusivity: centred array(s) in the grid's layout, diffusivity_batch = 1 (one k for every entry) or g->batch.
 * prm: method PHI_SOLVER_CG, balance_rhs = project_mean = 0, matrix_offset = 0.  Same persistent TMA-ring CG as N5 (two sweeps,
 * about 38 B/cell per iteration), phicuda_last_cg_operator() reports PHI_CG_OP_HELMHOLTZ_VARYING.  Single GPU, no z-slabs;
 * grids that do not fit the ring return PHI_ERR_UNSUPPORTED.  workspace: phicuda_cg_workspace_bytes(g). */
int phicuda_diffuse_implicit_varying_f32(const PhiGrid* g, const PhiBC* bc, const float* diffusivity, int32_t diffusivity_batch,
                                         float dt, const float* y, float* x, const PhiCgParams* prm, PhiCgResult* result,
                                         void* workspace, size_t workspace_bytes, void* stream);

/* ---- A1  fluid.make_incompressible (phi/physics/fluid.py:94-162), no obstacles, order 2, staggered ------------------
 * div scratch: one centred array.  Equivalent to divergence + cg_poisson + grad_sub on the same stream. */
int phicuda_make_incompressible_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], float* p, float* div,
                                    const PhiCgParams* prm, PhiCgResult* result, void* workspace,
                                    size_t workspace_bytes, void* stream);

/* ---- A1 for CenteredGrid velocities: wide stencil (phi/physics/fluid.py:154-155, 197-202; SURVEY.md Appendix A) ---------------
 * v: `dim` CENTRED arrays (component c with boundary vbc->comp[c]); div and grad are central differences
 * (phi/field/_field_math.py:230-233, 627-632), the operator divergence(gradient(p)) is not symmetric at the boundary rows, so the
 * solver is CG-adaptive (prm->method must be PHI_SOLVER_CG_ADAPTIVE = what Solve('auto') runs, PhiML backend/_linalg.py:93-128) with
 * prm->matrix_offset = the reference's rank-1 offset for rank-deficient systems (_optimize.py:705-714; estimate it with
 * phicuda_wide_laplace_f32 on a random vector).  p: in = x0, out = pressure.  Not the tuned path: simple kernels, and the call
 * SYNCHRONISES the stream every few iterations to read the stopping flags (hence `_host`). */
size_t phicuda_collocated_workspace_bytes(const PhiGrid* g);
int phicuda_wide_laplace_f32(const PhiGrid* g, const PhiVBC* vbc, const float* x, float* y, void* workspace, size_t workspace_bytes, void* stream);
int phicuda_make_incompressible_centered_host_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], float* p, const PhiCgParams* prm,
                                                  PhiCgResult* result, void* workspace, size_t workspace_bytes, void* stream);

/* ---- N4  static obstacles (phi/physics/fluid.py:121-137, 165-202, 212-240) ---------------------------------------------
 * accessible: centred mask, 1 in fluid cells, 0 inside obstacles (`~union(obstacle geometries)` sampled at cell centres).
 * make_incompressible_masked = divergence * active, CG on masked_laplace (faces touching an obstacle carry no flux,
 * obstacle cells are identity rows), v -= hard_bcs * grad p.  The caller applies apply_boundary_conditions first
 * (v *= 1 - obstacle mask at faces: phicuda_mul_faces_f32).  The solve runs on the TMA-ring kernel with the mask staged as an
 * extra haloed array (k_cg_ring<..., CgOp::Masked>; 5 lines per tile line and stage instead of 4); grids whose lines do not fit the
 * ring fall back to the register-marching kernel with PHI_SOLVER_CG, and return PHI_ERR_UNSUPPORTED with PHI_SOLVER_CG_ADAPTIVE
 * (CG-adaptive runs on the ring only; the z-slab entry phicuda_cg_poisson_dist_masked_f32 takes PHI_SOLVER_CG only). */
int phicuda_mul_faces_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], const float* const mask[3], void* stream);
/* the two stencil pieces of the masked projection on their own (z-slab runs exchange halo planes between them):
 * div = divergence(v) * accessible;   v -= hard_bcs * grad p, hard_bcs = min of the two adjacent cells' accessibility */
int phicuda_divergence_masked_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const v[3], const float* accessible, float* div, void* stream);
int phicuda_grad_sub_masked_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], const float* p, const float* accessible, void* stream);
int phicuda_cg_poisson_masked_f32(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x, const float* accessible,
                                  const PhiCgParams* prm, PhiCgResult* result, void* workspace, size_t workspace_bytes,
                                  void* stream);
int phicuda_make_incompressible_masked_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], float* p, float* div,
                                           const float* accessible, const PhiCgParams* prm, PhiCgResult* result,
                                           void* workspace, size_t workspace_bytes, void* stream);

/* ---- incompressible_step: the notebook step as ONE call (SURVEY.md §3.3) -------------------------------------------
 * s' = advect(s, v, dt) + inflow_rate * inflow ; v* = semi_lagrangian(v, v, dt) + dt * buoyancy(s') ;
 * v', p' = make_incompressible(v*, Solve('CG', x0 = p)).   mac_cormack != 0 selects advect.mac_cormack for s.
 * Five kernel launches + one device copy: inflow and buoyancy are epilogues of the two advection kernels (all staggered
 * components advected in one launch), the projected velocity is written straight into v.
 * All state is updated in place; scratch = 2 centred + dim staggered arrays (phicuda_plume_scratch_bytes). */
typedef struct PhiPlumeParams {
    float   dt;
    float   inflow_rate;
    float   buoyancy[3];
    int32_t mac_cormack;
    int32_t static_scalar;   /* 1: `s` is a stationary source (body force / forcing field, e.g. the Kolmogorov sin(4y) forcing): it is
                                not advected and gets no inflow; the step is v* = semi_lagrangian(v, v, dt) + dt * resample(s * b, to=v),
                                then the projection */
    void*   cg_start_event;  /* optional cudaEvent_t handles recorded on `stream` right before / after the pressure solve, */
    void*   cg_stop_event;   /* so a caller can time the CG kernel inside the single fused call (bench.py roofline); or NULL */
} PhiPlumeParams;
size_t phicuda_plume_scratch_bytes(const PhiGrid* g);
int phicuda_plume_step_f32(const PhiGrid* g, const PhiVBC* vbc, const PhiBC* sbc, float* const v[3], float* s, float* p,
                           const float* inflow, const PhiPlumeParams* sp, const PhiCgParams* prm, PhiCgResult* result,
                           float* scratch, void* workspace, size_t workspace_bytes, void* stream);
/* The same step with static obstacles (N4; Batched_Smoke, Fluid_Logo): the smoke is advected as above, then
 * v* = (semi_lagrangian(v, v, dt) + dt * buoyancy(s')) * face_factors   (apply_boundary_conditions, one advection launch) and
 * v', p' = make_incompressible(v*, obstacles, Solve(x0 = p)) as phicuda_make_incompressible_masked_f32 computes it.
 * accessible: centred mask (1 fluid, 0 obstacle); face_factors[c]: 1 - resample(geometry, v, soft=True, balance=1) on the stored
 * faces of component c (fext layout).  Both carry the full batch: every batch entry may have its own obstacle.  The result is bit for
 * bit that of phicuda_plume_step_f32's advection, phicuda_mul_faces_f32 and phicuda_make_incompressible_masked_f32 in sequence.
 * prm->method: PHI_SOLVER_CG or PHI_SOLVER_CG_ADAPTIVE (ring-only, as phicuda_cg_poisson_masked_f32), matrix_offset 0.
 * Single GPU: z-slab grids (halo > 0) return PHI_ERR_UNSUPPORTED.  Every argument check runs before the first CUDA call. */
int phicuda_plume_step_masked_f32(const PhiGrid* g, const PhiVBC* vbc, const PhiBC* sbc, float* const v[3], float* s, float* p,
                                  const float* inflow, const float* accessible, const float* const face_factors[3],
                                  const PhiPlumeParams* sp, const PhiCgParams* prm, PhiCgResult* result,
                                  float* scratch, void* workspace, size_t workspace_bytes, void* stream);

/* ---- N7  reaction-diffusion: the Reaction_Diffusion notebook's Gray-Scott step --------------------------------------------
 * `substeps` times, on centred arrays u and v of the grid (every batch entry with the same parameters):
 *   uvv = u * v**2;  su = du * laplace(u) - uvv + f * (1 - u);  sv = dv * laplace(v) + uvv - (f + k) * v;
 *   u = u + dt * su;  v = v + dt * sv
 * laplace as phicuda_laplace_f32, ghost cells of u from bc->comp[0] and of v from bc->comp[1].  Every operation is rounded as the
 * reference's float32 field arithmetic rounds it.  Boundaries: PERIODIC, ZERO_GRADIENT and constant 0 per side, the same kinds for u
 * and v - the extrapolations that the reference's step maps to themselves; a non-zero constant becomes 2c - c^2 after one step
 * and returns PHI_ERR_UNSUPPORTED.  The update is in place and the call never allocates: all substeps run in one persistent
 * kernel (PHI_KERNEL_RD_RING), 16 B/cell per substep (+ 16 B/cell once for an odd count), state ping-ponging through `scratch`
 * (phicuda_reaction_diffusion_scratch_bytes).  substeps == 0 leaves u and v untouched.  Single GPU, no z-slabs; grid lines that do
 * not fit the ring return PHI_ERR_UNSUPPORTED with the widest line that does.  Every argument check runs before the first CUDA
 * call: a refused call leaves u and v untouched. */
size_t phicuda_reaction_diffusion_scratch_bytes(const PhiGrid* g);
int phicuda_reaction_diffusion_f32(const PhiGrid* g, const PhiVBC* bc, float* u, float* v, float du, float dv, float f, float k,
                                   float dt, int32_t substeps, float* scratch, size_t scratch_bytes, void* stream);

/* ---- N8  wave step: the Waves notebook's explicit wave equation with a moving source disc ------------------------------------
 * `substeps` times, on centred arrays h_c (current) and h_p (previous) of the grid, with disc s of `discs` in substep s:
 *   h_c = where(disc_s, value_s, h_c);  h_p = where(disc_s, value_s, h_p);
 *   h_n = 2 * h_c - h_p + dd * (k_speed * laplace(h_c) - k_damp * (h_c - h_p));  (h_c, h_p) = (h_n, h_c)
 * laplace as phicuda_laplace_f32 with ghost cells from `bc`.  Boundaries: PERIODIC, ZERO_GRADIENT and constant 0 per side - the
 * extrapolations that the reference's step maps to themselves; a non-zero constant c becomes c - c = 0 after one step (2.0 * h_c
 * keeps h_c's extrapolation) and returns PHI_ERR_UNSUPPORTED.  Every operation is rounded as the reference's float32 field arithmetic rounds it.  disc_s holds the cells whose
 * centre p satisfies ((p_x - c_x)^2 + (p_y - c_y)^2) [+ (p_z - c_z)^2] <= radius_sq in float32 (Sphere.lies_inside), with the
 * cell centres taken from `centers`: n[0] x coordinates, then n[1] y, then n[2] z (host memory), as the caller's grid computes
 * them.  One disc per substep for every batch entry; `present == 0` stamps nothing.  `discs` and `centers` are host arrays,
 * copied into `scratch` (phicuda_wave_scratch_bytes) on `stream` - a copy from pageable memory, which waits for the stream's
 * earlier work.  The update is in place and the call never allocates: on return h_c holds the newest state and h_p the
 * previous, stamped one, for either parity of `substeps`.  All substeps run in one persistent kernel (PHI_KERNEL_WAVE_RING),
 * 12 B/cell per substep (+ 12 B/cell once for an odd count).  substeps == 0 returns before any CUDA call.  Single GPU, no
 * z-slabs; grid lines that do not fit the ring return PHI_ERR_UNSUPPORTED with the widest line that does.  Every argument check
 * runs before the first CUDA call: a refused call leaves h_c and h_p untouched. */
typedef struct PhiWaveDisc {
    float   center[3];     /* x, y[, z] */
    float   value;         /* stamped value */
    int32_t present;       /* 0: no disc in this substep */
} PhiWaveDisc;
size_t phicuda_wave_scratch_bytes(const PhiGrid* g, int32_t substeps);
int phicuda_wave_f32(const PhiGrid* g, const PhiBC* bc, float* h_c, float* h_p, float dd, float k_speed, float k_damp,
                     const PhiWaveDisc* discs, float radius_sq, const float* centers, int32_t substeps, void* scratch,
                     size_t scratch_bytes, void* stream);

/* ---- N10  Julia sets: the Julia_Set notebook's escape counts ---------------------------------------------------------------------
 * For batch entry b with constant c_b = c[2b] + i c[2b+1] and every cell (i, j) of a 2-D grid, with z_0 = x_i + i y_j:
 *   counts[b][j][i] = #{ t < iterations : abs(z_t) < 2 },   z_{t+1} = z_t ** 2 + c_b
 * rounded as PhiML's NumPy backend rounds complex64 on an AVX-512 CPU: z ** 2 = (a*a - b*b, a*b + b*a) without fma (np.power),
 * then + c per component; abs(z) = big * sqrt(fma(r, r, 1)), r = small / big over |a|, |b|.  Counts are int32 in the centred-array layout of `g`
 * (element size 4); only the owned cells are written, iterations == 0 writes zeros.  `centers`: n[0] x coordinates, then n[1] y
 * (host memory, finite), as the caller's grid computes them; `c`: 2 * batch floats (host memory), any values - non-finite constants
 * count as NumPy's inf / NaN arithmetic does.  Both are copied into `scratch` (phicuda_julia_scratch_bytes) on `stream`, a copy from
 * pageable memory that waits for the stream's earlier work.  One kernel launch (PHI_KERNEL_JULIA), compute-bound: 4 B/cell written.
 * 2-D only (3-D returns PHI_ERR_UNSUPPORTED), one GPU.  Every argument check runs before the first CUDA call: a refused call leaves
 * counts untouched. */
size_t phicuda_julia_scratch_bytes(const PhiGrid* g);
int phicuda_julia_f32(const PhiGrid* g, const float* centers, const float* c, int32_t iterations, int32_t* counts, void* scratch,
                      size_t scratch_bytes, void* stream);

/* ---- N12  SPH: the SPH notebook's dam break (examples/particles/SPH.ipynb, phi/physics/sph.py) ------------------------------------
 * `substeps` times apply_bounds(sph_step(v)) of the notebook, all in one cooperative launch (PHI_KERNEL_SPH), for n particles in `dim`
 * = 2 or 3 dimensions with the poly6 kernel.  One substep, per particle i, over the pairs j with sqrt(r2) < support (self included),
 * delta = x_j - x_i, r2 = sum(delta^2):
 *   rho_i = (sum_j kernel_norm (support^2 - r2)^3) mass,  p_i = isotropic_exp (rho_i - base_density)
 *   d = sqrt(max(r2, 1e-5)), gap = smoothing_length - d
 *   F_i = sum_j pressure_norm ((-delta / d) (p_i + p_j) / (2 rho_j)) gap^2 + viscous_norm ((v_j - v_i) / rho_j) gap
 *   v' = v + (F_i / rho_i + gravity) dt,  x' = x + dt v';  every component of x' outside [lower, upper] is clipped and its v' scaled
 *   by damping.
 * Neighbours are found on PhiML's hash grid: res = max(1, ceil(max(upper - lower, support) / support)) cells per axis of edge
 * (support res) / res, cell = trunc((x - lower) / edge) clamped into [0, res - 1] (the reference only clamps above; a particle
 * more than a cell below `lower`, or with a NaN or infinite coordinate, lands in the first or last cell here instead of indexing out
 * of range).  Sums run over the 3^dim neighbour cells in PhiML's offset order (x outermost), each cell's particles by ascending
 * index, with one float32 rounding per operation: the result is independent of the launch and equals tests/oracle_sph.py bit for bit.
 * x, v: device arrays (n, dim); x_out, v_out: (n, dim), rho_out: NULL or (n,), the density of the last substep.  Outputs must not
 * overlap each other, the inputs or the scratch.  scratch: device memory of phicuda_sph_scratch_bytes (0 for invalid parameters).
 * n == 0 returns 0 without a CUDA call; every argument check runs before the first CUDA call, and a refused call leaves the outputs
 * untouched. */
typedef struct PhiSphParams {
    float lower[3], upper[3];      /* domain corners (the first `dim` entries) */
    float support;                 /* s: the neighbour cutoff and minimum hash cell edge */
    float smoothing_length;        /* h: the gap h - d */
    float kernel_norm;             /* poly6 normalisation: (315 / 64 / pi) / s^9 in 3-D, (4 / pi) / s^8 in 2-D, rounded by the caller */
    float mass, pressure_norm, viscous_norm;
    float isotropic_exp, base_density;
    float dt, damping;
    float gravity[3];
} PhiSphParams;
size_t phicuda_sph_scratch_bytes(int64_t n, int32_t dim, const PhiSphParams* prm);
int phicuda_sph_f32(const float* x, const float* v, int64_t n, int32_t dim, const PhiSphParams* prm, int32_t substeps, float* x_out,
                    float* v_out, float* rho_out, void* scratch, size_t scratch_bytes, void* stream);

/* ---- N11  advect.points: points moved through a StaggeredGrid velocity (Euler, RK4) -----------------------------------------------
 * advect.points(points, velocity, dt, integrator) (phi/physics/advect.py:20-35, 136-153) applied `steps` times, every step in one
 * launch (PHI_KERNEL_POINTS).  One velocity sample at p: for every component c, idx_a = ((p_a - lower[c][a]) / size[c][a]) * res[c][a]
 * - 0.5, then math.grid_sample of component c at idx with its own boundary (vbc->comp[c], per-component constants included).
 *   Euler: p + v0 dt.   RK4: vh = v(p + (dt/2) v0), vh2 = v(p + (dt/2) vh), v1 = v(p + dt vh2), p + dt ((1/6) ((v0 + 2 (vh + vh2)) + v1)).
 * Every operation is rounded as PhiML's NumPy backend rounds float32 (DESIGN.md row N11): the results equal PhiML's bit for bit.
 * `map`: the component grids' bounds and resolution [component][axis] in float32, as UniformGrid.stagger computes them
 * (phi/geom/_grid.py:204-209): size = upper' - lower', res[c][a] = the number of faces of component c stored along axis a.
 * `points`, `out`: device arrays (batch, npoints, dim), batch = points_batch for `points` and B = max(points_batch, g->batch) for `out`;
 * points_batch is 1 or g->batch, or g->batch is 1 (the batch broadcasts as in PhiML).  `out` may be `points` when points_batch == B.
 * `trajectory`: NULL or (steps + 1, B, npoints, dim), entry 0 = the input positions.  Any point is taken, NaN and +-inf included.
 * One GPU (z-slabs return PHI_ERR_UNSUPPORTED).  npoints == 0 returns 0 without a CUDA call; every argument check runs before the
 * first CUDA call, and a refused call leaves out and trajectory untouched. */
#define PHI_INTEGRATOR_EULER 0
#define PHI_INTEGRATOR_RK4   1
typedef struct PhiPointMap { float lower[3][3], size[3][3], res[3][3]; } PhiPointMap;   /* [component][axis] */
int phicuda_advect_points_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const vel[3], const PhiPointMap* map,
                              const float* points, int64_t npoints, int32_t points_batch, float dt, int32_t integrator,
                              int32_t steps, float* out, float* trajectory, void* stream);

/* ---- N9  fp64: the Taylor-Green step of math.set_global_precision(64) -----------------------------------------------------
 * The same operations as their _f32 counterparts on float64 arrays (same layout, element size 8; x-rows stay padded to multiples of
 * 4 elements).  PhiGrid and PhiBC / PhiVBC keep describing the layout and the boundary kinds; their float fields hold the exact
 * values rounded to float, and PhiValues64 carries the exact values: every _f64 call returns PHI_ERR_INVALID unless
 * (float) values->dx[a] == g->dx[a] and (float) values->clo / chi[c][a] == the boundary's clo / chi[a] on every axis a < dim of
 * every component c < dim (a PhiBC argument: row c = 0).  The kernels compute in double throughout: 1 / dx is RN(1 / dx) in double,
 * and CG step sizes, offsets, means, tolerances and |r|^2 are double.
 * Single GPU: z-slab grids (halo != 0) return PHI_ERR_UNSUPPORTED.  The stencils and advection run one thread per sample; the
 * solve is the register-marching persistent CG (phicuda_last_launch_info reports PHI_KERNEL_CG_MARCH), two sweeps and 64 B/cell per
 * iteration.  PHICUDA_NO_RING and PHICUDA_SCALAR_KERNELS do not change this path.  Not offered in fp64: CG-adaptive (ring kernel
 * only), obstacles, MacCormack, diffuse.implicit, the fused steps and CenteredGrid velocities. */
typedef struct PhiValues64 {
    double dx[3];           /* cell size per axis */
    double clo[3][3];       /* [component][axis] constant of the lower side (unused, but still checked, where the kind is not PHI_BC_CONST) */
    double chi[3][3];
} PhiValues64;

typedef struct PhiCgParams64 {
    double  rtol;
    double  atol;
    int32_t max_iter;
    int32_t balance_rhs;
    int32_t project_mean;
    double  matrix_offset;
    int32_t method;          /* PHI_SOLVER_CG only */
} PhiCgParams64;

typedef struct PhiCgResult64 {
    int32_t iterations;
    int32_t converged;
    int32_t diverged;
    double  residual_sq;
    double  tol_sq;
    double  initial_residual_sq;
} PhiCgResult64;

int phicuda_laplace_f64(const PhiGrid* g, const PhiBC* bc, const PhiValues64* values, const double* x, double* y, void* stream);
int phicuda_laplace_axpy_f64(const PhiGrid* g, const PhiBC* bc, const PhiValues64* values, const double* x, double coeff, double* y,
                             void* stream);
int phicuda_divergence_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* values, const double* const v[3], double* div,
                           void* stream);
int phicuda_grad_sub_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* values, double* const v[3], const double* p,
                         void* stream);
/* vvalues: the velocity's exact values (vbc), fvalues: the advected field's (fbc) */
int phicuda_advect_centered_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* vvalues, const double* const vel[3],
                                const PhiBC* fbc, const PhiValues64* fvalues, const double* src, double* dst, double dt, void* stream);
int phicuda_advect_staggered_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* vvalues, const double* const vel[3],
                                 const PhiVBC* fbc, const PhiValues64* fvalues, const double* const src[3], double* const dst[3],
                                 double dt, void* stream);
size_t phicuda_cg_workspace_bytes_f64(const PhiGrid* g);
/* result: device array of `batch` PhiCgResult64 */
int phicuda_cg_poisson_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* values, const double* rhs, double* x,
                           const PhiCgParams64* prm, PhiCgResult64* result, void* workspace, size_t workspace_bytes, void* stream);
int phicuda_make_incompressible_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* values, double* const v[3], double* p,
                                    double* div, const PhiCgParams64* prm, PhiCgResult64* result, void* workspace,
                                    size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PHICUDA_H */
