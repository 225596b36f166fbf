// Multi-GPU communicator for the distributed pressure solve (SURVEY.md section 8e).
//
// One process per GPU.  Every rank cudaMalloc's one buffer that holds (a) the mailboxes and event flags of the
// in-kernel all-reduce and (b) the CG work vectors r, d0, d1 (+ per-CTA partial sums).  The buffers are exported as CUDA
// IPC handles, exchanged by the caller (torch.distributed all_gather of 64 bytes per rank) and opened with peer access,
// so that the persistent CG kernel can store halo planes and mailbox entries straight into its neighbours' memory over
// NVLink / NVSwitch.  No NCCL call and no host round trip happens inside a solve.
#include <cstdio>
#include <cstring>
#include "cg_common.cuh"
#include "launch.cuh"

struct PhiComm {
    int rank, n;
    unsigned char* local;
    size_t bytes;
    unsigned char* peer[PHI_MAX_RANKS];
    size_t off_flags, off_seq, off_mbox, off_ws, ws_bytes;
    PhiGrid grid;
};

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

extern "C" {

int phicuda_comm_create(int rank, int nranks, const PhiGrid* g, PhiComm** comm, void* ipc_handle_out)
{
    if (!g || !comm || !ipc_handle_out) { phi_set_error("comm_create: NULL argument"); return PHI_ERR_INVALID; }
    if (nranks < 1 || nranks > PHI_MAX_RANKS || rank < 0 || rank >= nranks) { phi_set_error("comm_create: rank %d of %d out of range (max %d ranks)", rank, nranks, PHI_MAX_RANKS); return PHI_ERR_INVALID; }
    static_assert(sizeof(cudaIpcMemHandle_t) == PHI_IPC_HANDLE_BYTES, "IPC handle size");
    DGrid dg;
    int e = phi_make_dgrid(g, &dg); if (e) return e;
    PhiComm* c = new PhiComm();
    memset(c, 0, sizeof(*c));
    c->rank = rank; c->n = nranks; c->grid = *g;
    c->off_flags = 0;
    c->off_seq = 256;
    c->off_mbox = 512;
    c->off_ws = align_up(c->off_mbox + (size_t)2 * PHI_MAX_RANKS * 2 * CG_MAX_BATCH * sizeof(double), 256);
    c->ws_bytes = phi_cg_workspace(dg, nullptr).bytes;
    c->bytes = c->off_ws + c->ws_bytes;
    cudaError_t ce = cudaMalloc((void**)&c->local, c->bytes);
    if (ce != cudaSuccess) { phi_set_error("comm_create: cudaMalloc(%zu) failed: %s", c->bytes, cudaGetErrorString(ce)); delete c; return (int)ce; }
    cudaMemset(c->local, 0, c->bytes);
    cudaDeviceSynchronize();
    cudaIpcMemHandle_t h;
    ce = cudaIpcGetMemHandle(&h, c->local);
    if (ce != cudaSuccess) { phi_set_error("comm_create: cudaIpcGetMemHandle failed: %s", cudaGetErrorString(ce)); cudaFree(c->local); delete c; return (int)ce; }
    memcpy(ipc_handle_out, &h, sizeof(h));
    c->peer[rank] = c->local;
    *comm = c;
    return 0;
}

int phicuda_comm_connect(PhiComm* c, const void* all_handles)
{
    if (!c || !all_handles) { phi_set_error("comm_connect: NULL argument"); return PHI_ERR_INVALID; }
    for (int q = 0; q < c->n; ++q) {
        if (q == c->rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, (const unsigned char*)all_handles + (size_t)q * PHI_IPC_HANDLE_BYTES, sizeof(h));
        void* p = nullptr;
        cudaError_t ce = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (ce != cudaSuccess) { phi_set_error("comm_connect: cudaIpcOpenMemHandle(rank %d) failed: %s", q, cudaGetErrorString(ce)); return (int)ce; }
        c->peer[q] = (unsigned char*)p;
    }
    return 0;
}

int phicuda_comm_destroy(PhiComm* c)
{
    if (!c) return 0;
    for (int q = 0; q < c->n; ++q)
        if (q != c->rank && c->peer[q]) cudaIpcCloseMemHandle(c->peer[q]);
    if (c->local) cudaFree(c->local);
    delete c;
    return 0;
}

static int cg_dist(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x, const float* accessible,
                   const PhiCgParams* prm, PhiCgResult* result, PhiComm* c, void* stream);

int phicuda_cg_poisson_dist_f32(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x,
                                const PhiCgParams* prm, PhiCgResult* result, PhiComm* c, void* stream)
{
    return cg_dist(g, vbc, rhs, x, nullptr, prm, result, c, stream);
}

int phicuda_cg_poisson_dist_masked_f32(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x, const float* accessible,
                                       const PhiCgParams* prm, PhiCgResult* result, PhiComm* c, void* stream)
{
    if (!accessible) { phi_set_error("cg_dist_masked: accessible is NULL"); return PHI_ERR_INVALID; }
    if (prm && prm->method == PHI_SOLVER_CG_ADAPTIVE) { phi_set_error("cg_dist_masked: CG-adaptive with obstacles runs on one GPU only"); return PHI_ERR_UNSUPPORTED; }
    return cg_dist(g, vbc, rhs, x, accessible, prm, result, c, stream);
}

}  // extern "C"

static int cg_dist(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x, const float* accessible,
                   const PhiCgParams* prm, PhiCgResult* result, PhiComm* c, void* stream)
{
    if (!c || !g || !vbc || !rhs || !x || !prm || !result) { phi_set_error("cg_dist: NULL argument"); return PHI_ERR_INVALID; }
    if (memcmp(g, &c->grid, sizeof(PhiGrid)) != 0) { phi_set_error("cg_dist: grid differs from the one the communicator was created for"); return PHI_ERR_INVALID; }
    CgLaunch l; PhiBC pbc;
    int e = phi_make_dgrid(g, &l.g); if (e) return e;
    e = phi_pressure_bc(vbc, g->dim, &pbc); if (e) return e;
    e = phi_make_centered(g, &pbc, &l.pf); if (e) return e;
    l.rhs = rhs; l.x = x; l.prm = *prm; l.result = result;
    if (accessible) { l.op.kind = CgOp::Masked; l.op.mask = accessible; }
    l.workspace = c->local + c->off_ws; l.workspace_bytes = c->ws_bytes;
    CommDev cm;
    memset(&cm, 0, sizeof(cm));
    cm.rank = c->rank; cm.n = c->n;
    const int last = g->dim - 1;
    cm.lower = (pbc.lo[last] == PHI_BC_HALO) ? (c->rank + c->n - 1) % c->n : -1;
    cm.upper = (pbc.hi[last] == PHI_BC_HALO) ? (c->rank + 1) % c->n : -1;
    for (int q = 0; q < c->n; ++q) {
        cm.mbox[q] = (double*)(c->peer[q] + c->off_mbox);
        cm.flag[q] = (unsigned long long*)(c->peer[q] + c->off_flags);
    }
    cm.seq = (unsigned long long*)(c->local + c->off_seq);
    if (cm.lower >= 0) { const CgWorkspace w = phi_cg_workspace(l.g, c->peer[cm.lower] + c->off_ws); cm.lo_r = w.r; cm.lo_d0 = w.d0; cm.lo_d1 = w.d1; }
    if (cm.upper >= 0) { const CgWorkspace w = phi_cg_workspace(l.g, c->peer[cm.upper] + c->off_ws); cm.hi_r = w.r; cm.hi_d0 = w.d0; cm.hi_d1 = w.d1; }
    if (c->n > 1 && (cm.lower < 0 && cm.upper < 0)) { phi_set_error("cg_dist: %d ranks but no PHI_BC_HALO side on the z axis", c->n); return PHI_ERR_INVALID; }
    e = phi_launch_cg_ring(l, &cm, (cudaStream_t)stream);
    if (e == -100) { phi_set_error("cg_dist: the grid does not fit the TMA ring kernel"); return PHI_ERR_UNSUPPORTED; }
    return e;
}
