// Host-side launchers implemented in the kernel translation units, called from api.cu.
#pragma once
#include "phi_internal.cuh"

int phi_launch_laplace(const DGrid& g, const DField& f, const float* x, float* y, float coeff, bool axpy, cudaStream_t s);
int phi_launch_divergence(const DGrid& g, const DVec& v, const DField& cf, float* div, const float* acc, cudaStream_t s);
int phi_launch_grad_sub(const DGrid& g, const DVec& vin, const DVecOut& v, const DField& pf, const float* p,
                        const DField* af, const float* acc, cudaStream_t s);
int phi_launch_mul_faces(const DGrid& g, const DVec& vin, const DVecOut& v, const float* const mask[3], cudaStream_t s);
int phi_launch_buoyancy(const DGrid& g, const DVec& vin, const DVecOut& v, const DField& sf, const float* sarr,
                        const float b[3], float dt, cudaStream_t s);
int phi_launch_absmax(const DGrid& g, const DVec& v, float* out, cudaStream_t s);
int phi_launch_axpy(const DGrid& g, const DField& cf, float a, const float* x, float* y, cudaStream_t s);

// target_comp < 0: centred field
int phi_launch_advect(const DGrid& g, const DVec& vel, const DField& ff, int target_comp, const float* src, float* dst,
                      float dt, cudaStream_t s);
int phi_launch_mac_cormack(const DGrid& g, const DVec& vel, const DField& ff, const float* src, float* dst, float* tmp,
                           float dt, float strength, cudaStream_t s);

// vectorised / fused variants (fused_kernels.cu); acc / af / faces: static obstacle masks (N4), nullptr = none
int phi_launch_divergence_vec(const DGrid& g, const DVec& v, const DField& cf, float* div, const float* acc, cudaStream_t s);
int phi_launch_grad_sub_vec(const DGrid& g, const DVec& vin, const DVecOut& vout, const DField& pf, const float* p,
                            const DField* af, const float* acc, cudaStream_t s);
int phi_launch_advect_centered_vec(const DGrid& g, const DVec& vel, const DField& ff, const float* src, float* dst, float dt,
                                   const float* add, float add_scale, cudaStream_t s);
int phi_launch_advect_staggered_vec(const DGrid& g, const DVec& vel, const DVec& fld, const DVecOut& dst, float dt,
                                    const DField* sf, const float* sarr, const float bu[3], const float* const* faces, cudaStream_t s);
int phi_launch_grid_sample(const DGrid& g, const DField& f, const float* grid, const float* coords, long long npoints, float* out, cudaStream_t s);
// CenteredGrid (collocated) velocities, wide stencil (collocated_kernels.cu)
size_t phi_collocated_workspace_bytes(const DGrid& g);
int phi_make_incompressible_collocated(const DGrid& g, const DField vfields[3], const DField vfields0[3], const DField& pf, const DField& cf,
                                       float* const v[3], float* p, const PhiCgParams& prm, PhiCgResult* result,
                                       void* workspace, size_t ws_bytes, cudaStream_t s);
int phi_wide_laplace(const DGrid& g, const DField vfields0[3], const DField& pf, const DField& cf, const float* x, float* y,
                     void* workspace, size_t ws_bytes, cudaStream_t s);
bool phi_scalar_kernels();      // PHICUDA_SCALAR_KERNELS=1: diagnostics, forces the one-thread-per-sample kernels of round 1

// The operator A of a CG solve A x = y.
enum class CgOp {
    Poisson,            // L (pf: the pressure boundary)
    Masked,             // N4: L with static obstacles, face coefficients min(mask_c, mask_nb); obstacle cells keep their value
    Helmholtz,          // N5 diffuse.implicit: I - amount * L0 (pf carries L0: constants zeroed)
    HelmholtzVarying,   // N6 diffuse.implicit with a varying diffusivity k: I + D0, face coefficients min(fl(ndt k))
};
// the operator stages one more haloed array after the CG vectors: the obstacle mask, or the diffusivity
__host__ __device__ constexpr bool cg_op_xslot(CgOp op) { return op == CgOp::Masked || op == CgOp::HelmholtzVarying; }

// The operator and its data (host side: CgLaunch; device side: the ring CG's kernel parameters, where the mask travels in CgArgs.acc).
struct CgOperator {
    float amount = 0.f;                  // Helmholtz
    CgOp kind = CgOp::Poisson;
    const float* k = nullptr;            // HelmholtzVarying: k per batch entry, or (kbcast) entry 0 for every entry
    int kbcast = 0;
    float ndt = 0.f;                     // -dt
    float kclo[3] = {0.f, 0.f, 0.f}, kchi[3] = {0.f, 0.f, 0.f};   // the real boundary constants of the constant sides: coefficient
                                                                  // ghosts and bias (pf has them zeroed for the value ghosts)
    const float* mask = nullptr;         // Masked: accessible mask (1 = fluid, 0 = obstacle)
};

struct CgLaunch {
    DGrid g; DField pf;
    const float* rhs; float* x;
    PhiCgParams prm; PhiCgResult* result;
    void* workspace; size_t workspace_bytes;
    CgOperator op;
};

// CG workspace: r | d0 | d1 | partials[4][2][batch][CG_MAX_GRID] | d2.  d2 and partial slots 4..7 belong to the one-sweep ring CG.
// The Helmholtz solves never run the one-sweep CG, so implicit diffusion keeps its right-hand side y' = y - bias in d2.  The vectors
// address the first owned plane (z-slabs: after the halo planes).  base == nullptr: only `bytes` is set.
struct CgWorkspace { float *r, *d0, *d1, *d2; double* partials; size_t bytes; };
CgWorkspace phi_cg_workspace(const DGrid& g, void* base);
// TMA ring fast paths (ring_kernels.cu); return -100 when the shape does not fit and the caller must fall back
int phi_launch_laplace_ring(const DGrid& g, const DField& f, const float* x, float* y, float coeff, bool axpy, cudaStream_t s);
#define PHI_MAX_RANKS 8
struct CommDev {                      // device view of the multi-GPU communicator (comm.cu)
    int rank, n;
    int lower, upper;                 // z neighbours (-1: physical boundary)
    double* mbox[PHI_MAX_RANKS];      // mailbox of every rank ([rank] = local), [2 parity][PHI_MAX_RANKS][2*CG_MAX_BATCH]
    unsigned long long* flag[PHI_MAX_RANKS];   // [2 parity][PHI_MAX_RANKS] event numbers
    unsigned long long* seq;          // local persistent event counter
    float *lo_r, *lo_d0, *lo_d1;      // lower neighbour's CG vectors (first owned plane)
    float *hi_r, *hi_d0, *hi_d1;      // upper neighbour's
};
int phi_launch_cg_ring(const CgLaunch& a, const CommDev* cm, cudaStream_t s);
bool phi_ring_enabled();
int phi_launch_cg(const CgLaunch& a, cudaStream_t s);
// diffuse.implicit on the ring CG (ring_kernels.cu): host-only fit test, and the solve (bias pre-pass + k_cg_ring with the
// Helmholtz operator l.op); cf[0 .. C-1] = boundary with constants of component c (batch entry b is component b % C; C = 1 for a varying
// diffusivity).  -100: the grid does not fit the ring.
bool phi_cg_ring_fits(const DGrid& g, CgOp op);
// widest grid line the ring CG takes for g's other extents and batch (host-only; error messages of refused solves)
int phi_cg_ring_max_width(const DGrid& g, CgOp op, bool adapt);
int phi_launch_diffuse_implicit(const CgLaunch& l, int C, const DField* cf, cudaStream_t s);
// N7 / N8 persistent steppers on the TMA ring (ring_kernels.cu), kernel = PHI_KERNEL_RD_RING or PHI_KERNEL_WAVE_RING; host-only, no CUDA call
bool phi_step_ring_fits(const DGrid& g, int kernel);
int phi_step_ring_max_width(const DGrid& g, int kernel);   // widest line (cells) the stepper's ring takes for g's other extents
// N7 reaction-diffusion on the TMA ring (ring_kernels.cu).  fk = f + k, rounded to float once.  -100: the grid does not fit the ring.
struct RdParams { float du, dv, f, fk, dt; };
int phi_launch_reaction_diffusion(const DGrid& g, const DField& f, float* u, float* v, float* su, float* sv, const RdParams& p,
                                  int substeps, cudaStream_t s);
// N8 the Waves notebook's wave step on the TMA ring (ring_kernels.cu).  -100: the grid does not fit the ring.
// WaveDisc: the disc stamped in one substep; lo / hi: per axis the index range of cells whose own axis term (p - c)^2 is <= r^2, a
// box that holds every cell of the disc (empty, lo = hi = 0, when the substep has no disc).
struct WaveDisc { float c[3]; float value; int lo[3], hi[3]; };
struct WaveParams { float dd, k_speed, k_damp, r2; };
// discs: `substeps` entries in device memory; coords: per-axis cell centres (n[0] x, then n[1] y, then n[2] z) in device memory;
// tmp: one centred array, written only for an odd substep count
int phi_launch_wave(const DGrid& g, const DField& f, float* hc, float* hp, float* tmp, const WaveDisc* discs, const float* coords,
                    const WaveParams& p, int substeps, cudaStream_t s);
