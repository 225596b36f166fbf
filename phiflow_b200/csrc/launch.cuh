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

// vectorised / fused variants (fused_kernels.cu); no obstacle masks
int phi_launch_divergence_vec(const DGrid& g, const DVec& v, const DField& cf, float* div, cudaStream_t s);
int phi_launch_grad_sub_vec(const DGrid& g, const DVec& vin, const DVecOut& vout, const DField& pf, const float* p, cudaStream_t s);
int phi_launch_advect_centered_vec(const DGrid& g, const DVec& vel, const DField& ff, const float* src, float* dst, float dt,
                                   const float* add, float add_scale, cudaStream_t s);
int phi_launch_advect_staggered_vec(const DGrid& g, const DVec& vel, const DVec& fld, const DVecOut& dst, float dt,
                                    const DField* sf, const float* sarr, const float bu[3], cudaStream_t s);
int phi_launch_grid_sample(const DGrid& g, const DField& f, const float* grid, const float* coords, long long npoints, float* out, cudaStream_t s);
// CenteredGrid (collocated) velocities, wide stencil (collocated_kernels.cu)
size_t phi_collocated_workspace_bytes(const DGrid& g);
int phi_make_incompressible_collocated(const DGrid& g, const DField vfields[3], const DField vfields0[3], const DField& pf, const DField& cf,
                                       float* const v[3], float* p, const PhiCgParams& prm, int balance, PhiCgResult* result,
                                       void* workspace, size_t ws_bytes, cudaStream_t s);
int phi_wide_laplace(const DGrid& g, const DField vfields0[3], const DField& pf, const DField& cf, const float* x, float* y,
                     void* workspace, size_t ws_bytes, cudaStream_t s);
bool phi_scalar_kernels();      // PHICUDA_SCALAR_KERNELS=1: diagnostics, forces the one-thread-per-sample kernels of round 1

struct CgLaunch {
    DGrid g; DField pf;
    const float* rhs; float* x;
    PhiCgParams prm; PhiCgResult* result;
    void* workspace; size_t workspace_bytes;
    const float* acc = nullptr;    // N4: accessible mask
    bool helm = false;             // N5 diffuse.implicit: operator I - helm_amount * L instead of L (pf carries L0: constants zeroed)
    float helm_amount = 0.f;
    // N6 (with helm): varying diffusivity k, operator I + D0 with face coefficients min(fl(helm_ndt k)); helm_kclo / helm_kchi are
    // the real boundary constants (coefficient ghosts; pf has them zeroed for the value ghosts)
    const float* helm_k = nullptr;
    bool helm_k_bcast = false;     // one k (entry 0) for every batch entry
    float helm_ndt = 0.f;          // -dt
    float helm_kclo[3] = {0.f, 0.f, 0.f}, helm_kchi[3] = {0.f, 0.f, 0.f};
};
size_t phi_cg_workspace_bytes(const DGrid& g);
// TMA ring fast paths (ring_kernels.cu); return -100 when the shape does not fit and the caller must fall back
int phi_launch_laplace_ring(const DGrid& g, const DField& f, const float* x, float* y, float coeff, bool axpy, cudaStream_t s);
#define PHI_MAX_RANKS 8
struct CommDev {                      // device view of the multi-GPU communicator (comm.cu)
    int rank, n;
    int lower, upper;                 // z neighbours (-1: physical boundary)
    double* mbox[PHI_MAX_RANKS];      // mailbox of every rank ([rank] = local), [2 parity][PHI_MAX_RANKS][2*CG_MAX_BATCH]
    unsigned long long* flag[PHI_MAX_RANKS];   // [2 parity][PHI_MAX_RANKS] event numbers
    unsigned long long* seq;          // local persistent event counter
    unsigned* arrive;                 // local arrival counter of the merged barrier (zeroed by the launcher)
    float *lo_r, *lo_d0, *lo_d1;      // lower neighbour's CG vectors (first owned plane)
    float *hi_r, *hi_d0, *hi_d1;      // upper neighbour's
};
int phi_launch_cg_ring(const CgLaunch& a, const CommDev* cm, cudaStream_t s);
bool phi_ring_enabled();
int phi_launch_cg(const CgLaunch& a, cudaStream_t s);
// N5 diffuse.implicit on the ring CG (ring_kernels.cu): host-only fit test, and the solve (bias pre-pass + k_cg_ring<..., HELM>);
// cf[c] = boundary with constants of component c (batch entry b is component b % C).  -100: the grid does not fit the ring.
// xslot: the launch stages one more haloed array (N6: the diffusivity).
bool phi_cg_ring_fits(const DGrid& g, bool xslot = false);
int phi_launch_diffuse_implicit(const CgLaunch& l, int C, const DField cf[3], cudaStream_t s);
// N6 diffuse.implicit with a varying diffusivity (ring_kernels.cu): bias pre-pass + k_cg_ring<..., HELM, VARK>.  -100: no fit.
int phi_launch_diffuse_implicit_varying(const CgLaunch& l, cudaStream_t s);
