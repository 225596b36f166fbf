// C ABI of libphicuda.so (declared in include/phicuda.h): argument validation, descriptor construction, launch order.
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "phi_internal.cuh"
#include "cg_common.cuh"
#include "launch.cuh"

// ---- error state -----------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

void phi_set_error(const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

static thread_local PhiLaunchInfo g_last_launch = {};
void phi_note_launch(const PhiLaunchInfo& info) { g_last_launch = info; }
static thread_local int g_last_cg_passes = 0;
void phi_note_cg_passes(int passes) { g_last_cg_passes = passes; }
static thread_local int g_last_cg_operator = 0;
void phi_note_cg_operator(int op) { g_last_cg_operator = op; }

bool phi_ring_enabled()
{
    const char* v = getenv("PHICUDA_NO_RING");       // diagnostics: force the register-marching kernels
    return !(v && v[0] == '1');
}

bool phi_scalar_kernels()
{
    const char* v = getenv("PHICUDA_SCALAR_KERNELS");    // diagnostics / A-B parity: the round-1 one-thread-per-sample kernels
    return v && v[0] == '1';
}

int phi_sm_count()
{
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms > 0 ? sms : 1;
}

static int cuda_fail(int err, const char* what)
{
    if (err > 0) phi_set_error("%s: %s", what, cudaGetErrorString((cudaError_t)err));
    return err;
}

// ---- descriptor construction ---------------------------------------------------------------------------------------
int phi_make_dgrid(const PhiGrid* g, DGrid* o)
{
    if (!g) { phi_set_error("grid is NULL"); return PHI_ERR_INVALID; }
    if (g->dim != 2 && g->dim != 3) { phi_set_error("grid.dim must be 2 or 3, got %d", g->dim); return PHI_ERR_INVALID; }
    if (g->batch < 1) { phi_set_error("grid.batch must be >= 1"); return PHI_ERR_INVALID; }
    if (g->halo < 0 || (g->halo > 0 && g->dim != 3)) { phi_set_error("grid.halo must be 0 for 2-D grids"); return PHI_ERR_INVALID; }
    o->dim = g->dim; o->batch = g->batch; o->halo = g->halo;
    for (int a = 0; a < 3; ++a) {
        const bool used = a < g->dim;
        o->n[a] = used ? g->n[a] : 1;
        o->cext[a] = used ? g->cext[a] : 1;
        o->fext[a] = used ? g->fext[a] : 1;
        const int pad = (a == 2 && g->dim == 3) ? 2 * g->halo : 0;
        if (used && (g->n[a] < 1 || g->cext[a] < g->n[a] + pad || g->fext[a] < g->n[a] + pad)) {
            phi_set_error("grid: n[%d]=%d cext=%d fext=%d invalid", a, g->n[a], g->cext[a], g->fext[a]); return PHI_ERR_INVALID;
        }
        if (used && !(g->dx[a] > 0.f)) { phi_set_error("grid: dx[%d] must be positive", a); return PHI_ERR_INVALID; }
        o->dx[a] = used ? g->dx[a] : 1.f;
        o->inv_dx[a] = used ? 1.f / g->dx[a] : 0.f;
        o->inv_dx2[a] = used ? 1.f / (g->dx[a] * g->dx[a]) : 0.f;
    }
    if (o->cext[0] % 4 != 0 || o->fext[0] % 4 != 0) { phi_set_error("grid: cext[0]=%d and fext[0]=%d must be multiples of 4 (16-byte rows)", o->cext[0], o->fext[0]); return PHI_ERR_INVALID; }
    if (o->fext[1] > 65535 || (long long)o->fext[2] * o->batch > 65535) { phi_set_error("grid: fext[1] and fext[2]*batch must be <= 65535"); return PHI_ERR_UNSUPPORTED; }
    return 0;
}

static void set_strides(DField* o, const int32_t ext[3], int dim)
{
    o->sy = ext[0];
    o->sz = (long long)ext[0] * ext[1];
    o->sb = o->sz * (dim == 3 ? ext[2] : 1);
}

static int check_bc(const PhiBC* bc, int dim)
{
    if (!bc) { phi_set_error("boundary is NULL"); return PHI_ERR_INVALID; }
    for (int a = 0; a < dim; ++a) {
        if (bc->lo[a] > 3 || bc->hi[a] > 3) { phi_set_error("boundary kind out of range on axis %d", a); return PHI_ERR_INVALID; }
        if ((bc->lo[a] == PHI_BC_HALO || bc->hi[a] == PHI_BC_HALO) && !(dim == 3 && a == 2)) { phi_set_error("PHI_BC_HALO is only valid on the z axis of 3-D grids"); return PHI_ERR_INVALID; }
        if ((bc->lo[a] == PHI_BC_PERIODIC) != (bc->hi[a] == PHI_BC_PERIODIC)) { phi_set_error("axis %d: PERIODIC must be set on both sides", a); return PHI_ERR_INVALID; }
    }
    return 0;
}

int phi_make_centered(const PhiGrid* g, const PhiBC* bc, DField* o)
{
    int e = check_bc(bc, g->dim); if (e) return e;
    for (int a = 0; a < 3; ++a) {
        const bool used = a < g->dim;
        o->lo[a] = 0; o->hi[a] = used ? g->n[a] - 1 : 0;
        o->klo[a] = used ? bc->lo[a] : PHI_BC_ZERO_GRADIENT; o->khi[a] = used ? bc->hi[a] : PHI_BC_ZERO_GRADIENT;
        o->clo[a] = used ? bc->clo[a] : 0.f; o->chi[a] = used ? bc->chi[a] : 0.f;
    }
    set_strides(o, g->cext, g->dim);
    o->halo = g->halo;
    if ((bc->lo[g->dim - 1] == PHI_BC_HALO || bc->hi[g->dim - 1] == PHI_BC_HALO) && g->halo < 1) { phi_set_error("PHI_BC_HALO needs grid.halo >= 1"); return PHI_ERR_INVALID; }
    return 0;
}

int phi_make_component(const PhiGrid* g, const PhiBC* bc, int c, DField* o)
{
    int e = phi_make_centered(g, bc, o); if (e) return e;
    // stored faces along the component's own axis (extrapolation.py:57-62): lower stored unless the boundary fixes the
    // value there (constant), upper stored only for ZERO_GRADIENT (PERIODIC: upper == lower face of cell 0)
    const bool lo_stored = bc->lo[c] != PHI_BC_CONST;
    const bool hi_stored = bc->hi[c] == PHI_BC_ZERO_GRADIENT;
    o->lo[c] = lo_stored ? 0 : 1;
    o->hi[c] = g->n[c] - 1 + (hi_stored ? 1 : 0);
    set_strides(o, g->fext, g->dim);
    if (o->hi[c] >= g->fext[c]) { phi_set_error("component %d stores face %d but fext[%d] = %d", c, o->hi[c], c, g->fext[c]); return PHI_ERR_INVALID; }
    if (o->hi[c] < o->lo[c]) { phi_set_error("component %d has no stored faces (n=%d)", c, g->n[c]); return PHI_ERR_UNSUPPORTED; }
    return 0;
}

int phi_pressure_bc(const PhiVBC* vbc, int dim, PhiBC* o)
{
    // fluid._pressure_extrapolation (phi/physics/fluid.py:264-274), per side: the NORMAL component's boundary decides
    memset(o, 0, sizeof(*o));
    for (int a = 0; a < dim; ++a) {
        const uint8_t kl = vbc->comp[a].lo[a], kh = vbc->comp[a].hi[a];
        o->lo[a] = (kl == PHI_BC_PERIODIC || kl == PHI_BC_HALO) ? kl : (kl == PHI_BC_ZERO_GRADIENT ? PHI_BC_CONST : PHI_BC_ZERO_GRADIENT);
        o->hi[a] = (kh == PHI_BC_PERIODIC || kh == PHI_BC_HALO) ? kh : (kh == PHI_BC_ZERO_GRADIENT ? PHI_BC_CONST : PHI_BC_ZERO_GRADIENT);
    }
    return 0;
}

template <class T>
UnitMap phi_make_unit_map(const DGridT<T>& g, int target_units)
{
    UnitMap um;
    um.nxt = (g.n[0] + PHI_TILE_X - 1) / PHI_TILE_X;
    const int nm = g.n[g.dim - 1];
    int mc = nm < 32 ? nm : 32;
    for (;;) {
        um.mc = mc;
        um.nmc = (nm + mc - 1) / mc;
        if (g.dim == 3) {
            um.nyt = (g.n[1] + PHI_WARPS_PER_CTA - 1) / PHI_WARPS_PER_CTA;
            um.wu_per_batch = 0;
            um.units_per_batch = um.nxt * um.nyt * um.nmc;
        } else {
            um.nyt = 1;
            um.wu_per_batch = um.nxt * um.nmc;
            um.units_per_batch = (um.wu_per_batch + PHI_WARPS_PER_CTA - 1) / PHI_WARPS_PER_CTA;
        }
        um.total_units = um.units_per_batch * g.batch;
        if (um.total_units >= target_units || mc <= 8) break;
        mc /= 2;
    }
    return um;
}

template UnitMap phi_make_unit_map<float>(const DGrid& g, int target_units);
template UnitMap phi_make_unit_map<double>(const DGridT<double>& g, int target_units);

static int make_vec(const PhiGrid* g, const PhiVBC* vbc, const float* const v[3], DVec* o)
{
    if (!vbc || !v) { phi_set_error("vector field / boundary is NULL"); return PHI_ERR_INVALID; }
    for (int c = 0; c < 3; ++c) {
        o->p[c] = nullptr;
        if (c >= g->dim) { memset(&o->f[c], 0, sizeof(DField)); continue; }
        if (!v[c]) { phi_set_error("component %d pointer is NULL", c); return PHI_ERR_INVALID; }
        for (int a = 0; a < g->dim; ++a) {
            if (vbc->comp[c].lo[a] != vbc->comp[0].lo[a] || vbc->comp[c].hi[a] != vbc->comp[0].hi[a]) {
                phi_set_error("boundary kinds must agree between components (axis %d)", a); return PHI_ERR_UNSUPPORTED;
            }
        }
        int e = phi_make_component(g, &vbc->comp[c], c, &o->f[c]); if (e) return e;
        o->p[c] = v[c];
    }
    return 0;
}

#define CHECK(expr) do { int _e = (expr); if (_e) return _e; } while (0)

// ---- exported functions ---------------------------------------------------------------------------------------------
extern "C" {

int phicuda_abi_version(void) { return PHICUDA_ABI_VERSION; }

size_t phicuda_last_error(char* buf, size_t buf_len)
{
    const size_t n = strlen(g_err);
    if (buf && buf_len) { strncpy(buf, g_err, buf_len - 1); buf[buf_len - 1] = 0; }
    return n;
}

int phicuda_last_launch_info(PhiLaunchInfo* out)
{
    if (!out) { phi_set_error("last_launch_info: out is NULL"); return PHI_ERR_INVALID; }
    *out = g_last_launch;
    return 0;
}

int phicuda_last_cg_passes(void) { return g_last_cg_passes; }
int phicuda_last_cg_operator(void) { return g_last_cg_operator; }

int phicuda_device_info(char* name, size_t name_len, int* sm_count, int* cc_major, int* cc_minor)
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e) return cuda_fail(e, "cudaGetDevice");
    cudaDeviceProp p;
    e = cudaGetDeviceProperties(&p, dev);
    if (e) return cuda_fail(e, "cudaGetDeviceProperties");
    if (name && name_len) { strncpy(name, p.name, name_len - 1); name[name_len - 1] = 0; }
    if (sm_count) *sm_count = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    return 0;
}

int phicuda_laplace_f32(const PhiGrid* g, const PhiBC* bc, const float* x, float* y, void* stream)
{
    DGrid dg; DField f;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(phi_make_centered(g, bc, &f));
    if (!x || !y || x == y) { phi_set_error("laplace: x and y must be distinct non-NULL arrays"); return PHI_ERR_INVALID; }
    return cuda_fail(phi_launch_laplace(dg, f, x, y, 0.f, false, (cudaStream_t)stream), "laplace");
}

int phicuda_laplace_axpy_f32(const PhiGrid* g, const PhiBC* bc, const float* x, float coeff, float* y, void* stream)
{
    DGrid dg; DField f;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(phi_make_centered(g, bc, &f));
    if (!x || !y || x == y) { phi_set_error("laplace_axpy: x and y must be distinct non-NULL arrays"); return PHI_ERR_INVALID; }
    return cuda_fail(phi_launch_laplace(dg, f, x, y, coeff, true, (cudaStream_t)stream), "laplace_axpy");
}

int phicuda_divergence_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const v[3], float* div, void* stream)
{
    DGrid dg; DVec dv; DField cf; PhiBC none; memset(&none, 0, sizeof(none));
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, v, &dv)); CHECK(phi_make_centered(g, &none, &cf));
    if (!div) { phi_set_error("divergence: div is NULL"); return PHI_ERR_INVALID; }
    if (!phi_scalar_kernels()) return cuda_fail(phi_launch_divergence_vec(dg, dv, cf, div, nullptr, (cudaStream_t)stream), "divergence");
    return cuda_fail(phi_launch_divergence(dg, dv, cf, div, nullptr, (cudaStream_t)stream), "divergence");
}

int phicuda_grad_sub_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], const float* p, void* stream)
{
    DGrid dg; DVec dv; DVecOut out; PhiBC pbc; DField pf;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, v, &dv));
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, &pf));
    if (!p) { phi_set_error("grad_sub: p is NULL"); return PHI_ERR_INVALID; }
    for (int c = 0; c < 3; ++c) out.p[c] = c < g->dim ? v[c] : nullptr;
    if (!phi_scalar_kernels()) return cuda_fail(phi_launch_grad_sub_vec(dg, dv, out, pf, p, nullptr, nullptr, (cudaStream_t)stream), "grad_sub");
    return cuda_fail(phi_launch_grad_sub(dg, dv, out, pf, p, nullptr, nullptr, (cudaStream_t)stream), "grad_sub");
}

int phicuda_advect_centered_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const vel[3],
                                const PhiBC* fbc, const float* src, float* dst, float dt, void* stream)
{
    DGrid dg; DVec dv; DField ff;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, vel, &dv)); CHECK(phi_make_centered(g, fbc, &ff));
    if (!src || !dst || src == dst) { phi_set_error("advect: src and dst must be distinct non-NULL arrays"); return PHI_ERR_INVALID; }
    if (!phi_scalar_kernels()) {
        const int e = phi_launch_advect_centered_vec(dg, dv, ff, src, dst, dt, nullptr, 0.f, (cudaStream_t)stream);
        if (e != -100) return cuda_fail(e, "advect_centered");          // -100: arrays beyond 2^31 elements -> 64-bit scalar kernel
    }
    return cuda_fail(phi_launch_advect(dg, dv, ff, -1, src, dst, dt, (cudaStream_t)stream), "advect_centered");
}

int phicuda_advect_staggered_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const vel[3],
                                 const PhiVBC* fbc, const float* const src[3], float* const dst[3], float dt, void* stream)
{
    DGrid dg; DVec dv; DVec df;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, vel, &dv)); CHECK(make_vec(g, fbc, src, &df));
    for (int c = 0; c < g->dim; ++c) {
        if (!dst[c]) { phi_set_error("advect: dst[%d] is NULL", c); return PHI_ERR_INVALID; }
        for (int k = 0; k < g->dim; ++k) if (dst[c] == src[k] || dst[c] == vel[k]) { phi_set_error("advect: dst must not alias src or vel"); return PHI_ERR_INVALID; }
    }
    if (!phi_scalar_kernels()) {      // all components in one launch: the velocity lines are loaded once and shared
        DVecOut out; for (int c = 0; c < 3; ++c) out.p[c] = c < g->dim ? dst[c] : nullptr;
        const int e = phi_launch_advect_staggered_vec(dg, dv, df, out, dt, nullptr, nullptr, nullptr, nullptr, (cudaStream_t)stream);
        if (e != -100) return cuda_fail(e, "advect_staggered");
    }
    for (int c = 0; c < g->dim; ++c)
        CHECK(cuda_fail(phi_launch_advect(dg, dv, df.f[c], c, src[c], dst[c], dt, (cudaStream_t)stream), "advect_staggered"));
    return 0;
}

int phicuda_grid_sample_f32(const PhiGrid* g, const PhiBC* bc, const float* grid, const float* coords, int64_t npoints, float* out, void* stream)
{
    DGrid dg; DField f;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(phi_make_centered(g, bc, &f));
    if (npoints < 0 || (npoints > 0 && (!grid || !coords || !out))) { phi_set_error("grid_sample: NULL argument"); return PHI_ERR_INVALID; }
    return cuda_fail(phi_launch_grid_sample(dg, f, grid, coords, (long long)npoints, out, (cudaStream_t)stream), "grid_sample");
}

int phicuda_mac_cormack_centered_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const vel[3],
                                     const PhiBC* fbc, const float* src, float* dst, float* tmp,
                                     float dt, float correction_strength, void* stream)
{
    DGrid dg; DVec dv; DField ff;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, vel, &dv)); CHECK(phi_make_centered(g, fbc, &ff));
    if (!src || !dst || !tmp || src == dst || tmp == dst || tmp == src) { phi_set_error("mac_cormack: src, dst, tmp must be distinct non-NULL arrays"); return PHI_ERR_INVALID; }
    return cuda_fail(phi_launch_mac_cormack(dg, dv, ff, src, dst, tmp, dt, correction_strength, (cudaStream_t)stream), "mac_cormack");
}

int phicuda_axpy_centered_f32(const PhiGrid* g, float a, const float* x, float* y, void* stream)
{
    DGrid dg; DField cf; PhiBC none; memset(&none, 0, sizeof(none));
    CHECK(phi_make_dgrid(g, &dg)); CHECK(phi_make_centered(g, &none, &cf));
    if (!x || !y) { phi_set_error("axpy: NULL array"); return PHI_ERR_INVALID; }
    return cuda_fail(phi_launch_axpy(dg, cf, a, x, y, (cudaStream_t)stream), "axpy");
}

int phicuda_add_buoyancy_f32(const PhiGrid* g, const PhiVBC* vbc, const PhiBC* sbc, const float* s,
                             const float b[3], float dt, float* const v[3], void* stream)
{
    DGrid dg; DVec dv; DVecOut out; DField sf;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, v, &dv)); CHECK(phi_make_centered(g, sbc, &sf));
    if (!s || !b) { phi_set_error("add_buoyancy: NULL argument"); return PHI_ERR_INVALID; }
    for (int c = 0; c < 3; ++c) out.p[c] = c < g->dim ? v[c] : nullptr;
    return cuda_fail(phi_launch_buoyancy(dg, dv, out, sf, s, b, dt, (cudaStream_t)stream), "add_buoyancy");
}

int phicuda_max_abs_velocity_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const v[3], float* out, void* stream)
{
    DGrid dg; DVec dv;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, v, &dv));
    if (!out) { phi_set_error("max_abs_velocity: out is NULL"); return PHI_ERR_INVALID; }
    return cuda_fail(phi_launch_absmax(dg, dv, out, (cudaStream_t)stream), "max_abs_velocity");
}

// ---- N4: static obstacles ------------------------------------------------------------------------------------------------
static int accessible_field(const PhiGrid* g, const PhiVBC* vbc, DField* af)
{
    // fluid._accessible_extrapolation (phi/physics/fluid.py:277-288): PERIODIC -> PERIODIC, BOUNDARY -> ONE, constant -> ZERO
    PhiBC abc; memset(&abc, 0, sizeof(abc));
    for (int a = 0; a < g->dim; ++a) {
        const uint8_t kl = vbc->comp[a].lo[a], kh = vbc->comp[a].hi[a];
        // z-slab sides: the mask of the neighbouring slab sits in the halo planes (static: exchanged once by the caller)
        abc.lo[a] = (kl == PHI_BC_PERIODIC || kl == PHI_BC_HALO) ? kl : PHI_BC_CONST; abc.clo[a] = kl == PHI_BC_ZERO_GRADIENT ? 1.f : 0.f;
        abc.hi[a] = (kh == PHI_BC_PERIODIC || kh == PHI_BC_HALO) ? kh : PHI_BC_CONST; abc.chi[a] = kh == PHI_BC_ZERO_GRADIENT ? 1.f : 0.f;
    }
    return phi_make_centered(g, &abc, af);
}

int phicuda_divergence_masked_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const v[3], const float* accessible, float* div, void* stream)
{
    DGrid dg; DVec dv; DField cf; PhiBC none; memset(&none, 0, sizeof(none));
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, v, &dv)); CHECK(phi_make_centered(g, &none, &cf));
    if (!div || !accessible) { phi_set_error("divergence_masked: NULL argument"); return PHI_ERR_INVALID; }
    if (!phi_scalar_kernels()) return cuda_fail(phi_launch_divergence_vec(dg, dv, cf, div, accessible, (cudaStream_t)stream), "divergence_masked");
    return cuda_fail(phi_launch_divergence(dg, dv, cf, div, accessible, (cudaStream_t)stream), "divergence_masked");
}

int phicuda_grad_sub_masked_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], const float* p, const float* accessible, void* stream)
{
    DGrid dg; DVec dv; DVecOut out; PhiBC pbc; DField pf, af;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, v, &dv));
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, &pf)); CHECK(accessible_field(g, vbc, &af));
    if (!p || !accessible) { phi_set_error("grad_sub_masked: NULL argument"); return PHI_ERR_INVALID; }
    for (int c = 0; c < 3; ++c) out.p[c] = c < g->dim ? v[c] : nullptr;
    if (!phi_scalar_kernels()) return cuda_fail(phi_launch_grad_sub_vec(dg, dv, out, pf, p, &af, accessible, (cudaStream_t)stream), "grad_sub_masked");
    return cuda_fail(phi_launch_grad_sub(dg, dv, out, pf, p, &af, accessible, (cudaStream_t)stream), "grad_sub_masked");
}

int phicuda_mul_faces_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], const float* const mask[3], void* stream)
{
    DGrid dg; DVec dv; DVecOut out;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, v, &dv));
    for (int c = 0; c < 3; ++c) { out.p[c] = c < g->dim ? v[c] : nullptr; if (c < g->dim && !mask[c]) { phi_set_error("mul_faces: mask[%d] is NULL", c); return PHI_ERR_INVALID; } }
    return cuda_fail(phi_launch_mul_faces(dg, dv, out, mask, (cudaStream_t)stream), "mul_faces");
}

int phicuda_cg_poisson_masked_f32(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x, const float* accessible,
                                  const PhiCgParams* prm, PhiCgResult* result, void* workspace, size_t workspace_bytes, void* stream)
{
    CgLaunch l; PhiBC pbc; DField af;
    CHECK(phi_make_dgrid(g, &l.g));
    if (!vbc || !rhs || !x || !prm || !result || !workspace || !accessible) { phi_set_error("cg_masked: NULL argument"); return PHI_ERR_INVALID; }
    CHECK(accessible_field(g, vbc, &af));
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, &l.pf));
    l.rhs = rhs; l.x = x; l.prm = *prm; l.result = result; l.workspace = workspace; l.workspace_bytes = workspace_bytes;
    l.op.kind = CgOp::Masked; l.op.mask = accessible;
    return phi_launch_cg(l, (cudaStream_t)stream);
}

static int project(const PhiGrid* g, const PhiVBC* vbc, const float* const vin[3], float* const vout[3], float* p, float* div,
                   const float* accessible, const PhiCgParams* prm, PhiCgResult* result, void* workspace, size_t workspace_bytes,
                   void* ev0, void* ev1, void* stream);

int phicuda_make_incompressible_masked_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], float* p, float* div,
                                           const float* accessible, const PhiCgParams* prm, PhiCgResult* result,
                                           void* workspace, size_t workspace_bytes, void* stream)
{
    if (!accessible || !p || !div) { phi_set_error("make_incompressible_masked: NULL argument"); return PHI_ERR_INVALID; }
    return project(g, vbc, v, v, p, div, accessible, prm, result, workspace, workspace_bytes, nullptr, nullptr, stream);
}

size_t phicuda_cg_workspace_bytes(const PhiGrid* g)
{
    DGrid dg;
    if (phi_make_dgrid(g, &dg)) return 0;
    return phi_cg_workspace(dg, nullptr).bytes;
}

int phicuda_cg_poisson_f32(const PhiGrid* g, const PhiVBC* vbc, const float* rhs, float* x,
                           const PhiCgParams* prm, PhiCgResult* result, void* workspace, size_t workspace_bytes,
                           void* stream)
{
    CgLaunch l; PhiBC pbc;
    CHECK(phi_make_dgrid(g, &l.g));
    if (!vbc || !rhs || !x || !prm || !result || !workspace) { phi_set_error("cg: NULL argument"); return PHI_ERR_INVALID; }
    for (int a = 0; a < g->dim; ++a) CHECK(check_bc(&vbc->comp[a], g->dim));
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, &l.pf));
    l.rhs = rhs; l.x = x; l.prm = *prm; l.result = result; l.workspace = workspace; l.workspace_bytes = workspace_bytes;
    return phi_launch_cg(l, (cudaStream_t)stream);
}

int phicuda_diffuse_implicit_f32(const PhiGrid* g, const PhiVBC* bc, int32_t components, float amount, const float* y, float* x,
                                 const PhiCgParams* prm, PhiCgResult* result, void* workspace, size_t workspace_bytes, void* stream)
{
    // every check runs before the first CUDA call
    CgLaunch l; DField cf[3];
    CHECK(phi_make_dgrid(g, &l.g));
    if (!bc || !y || !x || !prm || !result || !workspace) { phi_set_error("diffuse_implicit: NULL argument"); return PHI_ERR_INVALID; }
    if (components < 1 || components > 3) { phi_set_error("diffuse_implicit: components must be 1, 2 or 3, got %d", components); return PHI_ERR_INVALID; }
    if (g->batch % components != 0) { phi_set_error("diffuse_implicit: batch %d is not a multiple of components %d", g->batch, components); return PHI_ERR_INVALID; }
    if (!std::isfinite(amount)) { phi_set_error("diffuse_implicit: amount is not finite"); return PHI_ERR_INVALID; }
    if (prm->method != PHI_SOLVER_CG) { phi_set_error("diffuse_implicit: only PHI_SOLVER_CG (the reference's Solve('CG'))"); return PHI_ERR_UNSUPPORTED; }
    if (prm->balance_rhs || prm->project_mean || prm->matrix_offset != 0.f) {
        phi_set_error("diffuse_implicit: I - a L is not singular - balance_rhs, project_mean and matrix_offset must be 0"); return PHI_ERR_INVALID;
    }
    if (g->halo != 0) { phi_set_error("diffuse_implicit: z-slab grids are not supported"); return PHI_ERR_UNSUPPORTED; }
    for (int c = 0; c < components; ++c) {
        CHECK(phi_make_centered(g, &bc->comp[c], &cf[c]));
        for (int a = 0; a < g->dim; ++a)
            if (bc->comp[c].lo[a] != bc->comp[0].lo[a] || bc->comp[c].hi[a] != bc->comp[0].hi[a]) {
                phi_set_error("diffuse_implicit: boundary kinds must agree between components (axis %d)", a); return PHI_ERR_UNSUPPORTED;
            }
    }
    const size_t ws_need = phi_cg_workspace(l.g, nullptr).bytes;
    if (workspace_bytes < ws_need) { phi_set_error("diffuse_implicit: workspace %zu < %zu bytes", workspace_bytes, ws_need); return PHI_ERR_WORKSPACE; }
    if (!phi_ring_enabled() || !phi_cg_ring_fits(l.g, CgOp::Helmholtz)) {
        phi_set_error("diffuse_implicit: the grid does not fit the TMA-ring CG (batch <= 1024, grid lines short enough); this operator has no other kernel");
        return PHI_ERR_UNSUPPORTED;
    }
    PhiBC zero = bc->comp[0];                                    // L0: the operator sees the kinds, the constants go into the bias
    for (int a = 0; a < 3; ++a) { zero.clo[a] = 0.f; zero.chi[a] = 0.f; }
    CHECK(phi_make_centered(g, &zero, &l.pf));
    for (int c = components; c < 3; ++c) cf[c] = l.pf;
    l.rhs = y; l.x = x; l.prm = *prm; l.result = result; l.workspace = workspace; l.workspace_bytes = workspace_bytes;
    l.op.kind = CgOp::Helmholtz; l.op.amount = amount;
    const int e = phi_launch_diffuse_implicit(l, components, cf, (cudaStream_t)stream);
    if (e == -100) { phi_set_error("diffuse_implicit: the grid does not fit the TMA-ring CG on this device"); return PHI_ERR_UNSUPPORTED; }
    return cuda_fail(e, "diffuse_implicit");
}

int phicuda_diffuse_implicit_varying_f32(const PhiGrid* g, const PhiBC* bc, const float* diffusivity, int32_t diffusivity_batch,
                                         float dt, const float* y, float* x, const PhiCgParams* prm, PhiCgResult* result,
                                         void* workspace, size_t workspace_bytes, void* stream)
{
    // every check runs before the first CUDA call
    CgLaunch l; DField cf;
    CHECK(phi_make_dgrid(g, &l.g));
    if (!bc || !diffusivity || !y || !x || !prm || !result || !workspace) { phi_set_error("diffuse_implicit_varying: NULL argument"); return PHI_ERR_INVALID; }
    if (diffusivity_batch != 1 && diffusivity_batch != g->batch) {
        phi_set_error("diffuse_implicit_varying: diffusivity_batch must be 1 or the grid's batch %d, got %d", g->batch, diffusivity_batch); return PHI_ERR_INVALID;
    }
    if (!std::isfinite(dt)) { phi_set_error("diffuse_implicit_varying: dt is not finite"); return PHI_ERR_INVALID; }
    if (prm->method != PHI_SOLVER_CG) { phi_set_error("diffuse_implicit_varying: only PHI_SOLVER_CG (the reference's Solve('CG'))"); return PHI_ERR_UNSUPPORTED; }
    if (prm->balance_rhs || prm->project_mean || prm->matrix_offset != 0.f) {
        phi_set_error("diffuse_implicit_varying: I + D0 is not singular - balance_rhs, project_mean and matrix_offset must be 0"); return PHI_ERR_INVALID;
    }
    if (g->halo != 0) { phi_set_error("diffuse_implicit_varying: z-slab grids are not supported"); return PHI_ERR_UNSUPPORTED; }
    CHECK(phi_make_centered(g, bc, &cf));
    const size_t ws_need = phi_cg_workspace(l.g, nullptr).bytes;
    if (workspace_bytes < ws_need) { phi_set_error("diffuse_implicit_varying: workspace %zu < %zu bytes", workspace_bytes, ws_need); return PHI_ERR_WORKSPACE; }
    if (!phi_ring_enabled() || !phi_cg_ring_fits(l.g, CgOp::HelmholtzVarying)) {
        phi_set_error("diffuse_implicit_varying: the grid does not fit the TMA-ring CG (batch <= 1024, grid lines short enough); this operator has no other kernel");
        return PHI_ERR_UNSUPPORTED;
    }
    PhiBC zero = *bc;                                            // D0: the value ghosts of constant sides are 0, the constants go into
    for (int a = 0; a < 3; ++a) { zero.clo[a] = 0.f; zero.chi[a] = 0.f; }    // the bias and the coefficient ghosts
    CHECK(phi_make_centered(g, &zero, &l.pf));
    l.rhs = y; l.x = x; l.prm = *prm; l.result = result; l.workspace = workspace; l.workspace_bytes = workspace_bytes;
    l.op.kind = CgOp::HelmholtzVarying; l.op.k = diffusivity; l.op.kbcast = diffusivity_batch == 1 && g->batch > 1; l.op.ndt = -dt;
    for (int a = 0; a < 3; ++a) {
        l.op.kclo[a] = a < g->dim && cf.klo[a] == PHI_BC_CONST ? cf.clo[a] : 0.f;
        l.op.kchi[a] = a < g->dim && cf.khi[a] == PHI_BC_CONST ? cf.chi[a] : 0.f;
    }
    const int e = phi_launch_diffuse_implicit(l, 1, &cf, (cudaStream_t)stream);
    if (e == -100) { phi_set_error("diffuse_implicit_varying: the grid does not fit the TMA-ring CG on this device"); return PHI_ERR_UNSUPPORTED; }
    return cuda_fail(e, "diffuse_implicit_varying");
}

// div -> CG -> v = vin - grad p.  vin/vout may be the same arrays (make_incompressible) or scratch -> state (fused step).
// accessible != nullptr: the obstacle projection (N4), div *= accessible, masked CG, grad p *= hard_bcs.  The stencils take the float4
// kernels unless PHICUDA_SCALAR_KERNELS=1, with and without the mask.
static int project(const PhiGrid* g, const PhiVBC* vbc, const float* const vin[3], float* const vout[3], float* p, float* div,
                   const float* accessible, const PhiCgParams* prm, PhiCgResult* result, void* workspace, size_t workspace_bytes,
                   void* ev0, void* ev1, void* stream)
{
    DGrid dg; DVec dv; DVecOut out; DField cf, pf, af; PhiBC none, pbc; memset(&none, 0, sizeof(none));
    CHECK(phi_make_dgrid(g, &dg)); CHECK(make_vec(g, vbc, vin, &dv)); CHECK(phi_make_centered(g, &none, &cf));
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, &pf));
    if (accessible) CHECK(accessible_field(g, vbc, &af));
    if (!p || !div || !vout) { phi_set_error("make_incompressible: NULL argument"); return PHI_ERR_INVALID; }
    for (int c = 0; c < 3; ++c) {
        out.p[c] = c < g->dim ? vout[c] : nullptr;
        if (c < g->dim && !vout[c]) { phi_set_error("make_incompressible: output component %d is NULL", c); return PHI_ERR_INVALID; }
    }
    cudaStream_t st = (cudaStream_t)stream;
    const bool scalar = phi_scalar_kernels();
    const DField* afp = accessible ? &af : nullptr;
    CHECK(cuda_fail(scalar ? phi_launch_divergence(dg, dv, cf, div, accessible, st) : phi_launch_divergence_vec(dg, dv, cf, div, accessible, st), "divergence"));
    if (ev0) CHECK(cuda_fail(cudaEventRecord((cudaEvent_t)ev0, st), "cudaEventRecord"));
    if (accessible) CHECK(phicuda_cg_poisson_masked_f32(g, vbc, div, p, accessible, prm, result, workspace, workspace_bytes, stream));
    else            CHECK(phicuda_cg_poisson_f32(g, vbc, div, p, prm, result, workspace, workspace_bytes, stream));
    if (ev1) CHECK(cuda_fail(cudaEventRecord((cudaEvent_t)ev1, st), "cudaEventRecord"));
    return cuda_fail(scalar ? phi_launch_grad_sub(dg, dv, out, pf, p, afp, accessible, st) : phi_launch_grad_sub_vec(dg, dv, out, pf, p, afp, accessible, st), "grad_sub");
}

int phicuda_make_incompressible_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], float* p, float* div,
                                    const PhiCgParams* prm, PhiCgResult* result, void* workspace,
                                    size_t workspace_bytes, void* stream)
{
    return project(g, vbc, v, v, p, div, nullptr, prm, result, workspace, workspace_bytes, nullptr, nullptr, stream);
}

// ---- CenteredGrid velocities (wide stencil) -------------------------------------------------------------------------------
static int collocated_fields(const PhiGrid* g, const PhiVBC* vbc, DGrid* dg, DField vf[3], DField vf0[3], DField* pf, DField* cf)
{
    CHECK(phi_make_dgrid(g, dg));
    if (g->halo != 0) { phi_set_error("collocated: z-slabs are not supported for CenteredGrid velocities"); return PHI_ERR_UNSUPPORTED; }
    if (!vbc) { phi_set_error("collocated: boundary is NULL"); return PHI_ERR_INVALID; }
    PhiBC none, pbc; memset(&none, 0, sizeof(none));
    CHECK(phi_make_centered(g, &none, cf));
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, pf));
    for (int c = 0; c < 3; ++c) {
        if (c >= g->dim) { memset(&vf[c], 0, sizeof(DField)); memset(&vf0[c], 0, sizeof(DField)); continue; }
        CHECK(phi_make_centered(g, &vbc->comp[c], &vf[c]));
        PhiBC zero = vbc->comp[c];                               // extrapolation.remove_constant_offset (fluid.py:200)
        for (int a = 0; a < 3; ++a) { zero.clo[a] = 0.f; zero.chi[a] = 0.f; }
        CHECK(phi_make_centered(g, &zero, &vf0[c]));
    }
    return 0;
}

size_t phicuda_collocated_workspace_bytes(const PhiGrid* g)
{
    DGrid dg;
    if (phi_make_dgrid(g, &dg)) return 0;
    return phi_collocated_workspace_bytes(dg);
}

int phicuda_wide_laplace_f32(const PhiGrid* g, const PhiVBC* vbc, const float* x, float* y, void* workspace, size_t workspace_bytes, void* stream)
{
    DGrid dg; DField vf[3], vf0[3], pf, cf;
    CHECK(collocated_fields(g, vbc, &dg, vf, vf0, &pf, &cf));
    if (!x || !y || !workspace || x == y) { phi_set_error("wide_laplace: NULL / aliased argument"); return PHI_ERR_INVALID; }
    return cuda_fail(phi_wide_laplace(dg, vf0, pf, cf, x, y, workspace, workspace_bytes, (cudaStream_t)stream), "wide_laplace");
}

int phicuda_make_incompressible_centered_host_f32(const PhiGrid* g, const PhiVBC* vbc, float* const v[3], float* p, const PhiCgParams* prm,
                                                  PhiCgResult* result, void* workspace, size_t workspace_bytes, void* stream)
{
    DGrid dg; DField vf[3], vf0[3], pf, cf;
    CHECK(collocated_fields(g, vbc, &dg, vf, vf0, &pf, &cf));
    if (!v || !p || !prm || !result || !workspace) { phi_set_error("make_incompressible_centered: NULL argument"); return PHI_ERR_INVALID; }
    for (int c = 0; c < g->dim; ++c) if (!v[c]) { phi_set_error("make_incompressible_centered: component %d is NULL", c); return PHI_ERR_INVALID; }
    if (prm->method != PHI_SOLVER_CG_ADAPTIVE) { phi_set_error("make_incompressible_centered: the wide-stencil operator is not symmetric - use PHI_SOLVER_CG_ADAPTIVE (Solve('auto'))"); return PHI_ERR_UNSUPPORTED; }
    return cuda_fail(phi_make_incompressible_collocated(dg, vf, vf0, pf, cf, v, p, *prm, result, workspace, workspace_bytes,
                                                        (cudaStream_t)stream), "make_incompressible_centered");
}

static size_t centred_elems(const PhiGrid* g) { return (size_t)g->cext[0] * g->cext[1] * (g->dim == 3 ? g->cext[2] : 1) * g->batch; }
static size_t face_elems(const PhiGrid* g) { return (size_t)g->fext[0] * g->fext[1] * (g->dim == 3 ? g->fext[2] : 1) * g->batch; }

size_t phicuda_plume_scratch_bytes(const PhiGrid* g)
{
    return g ? (2 * centred_elems(g) + (size_t)g->dim * face_elems(g)) * sizeof(float) : 0;
}

// The step without the argument checks of its entry point.  faces / accessible: static obstacles (N4), nullptr = none.
static int plume_step(const PhiGrid* g, const PhiVBC* vbc, const PhiBC* sbc, float* const v[3], float* s, float* p,
                      const float* inflow, const float* accessible, const float* const* faces, const PhiPlumeParams* sp,
                      const PhiCgParams* prm, PhiCgResult* result, float* scratch, void* workspace, size_t workspace_bytes, void* stream)
{
    // Launch sequence (5 kernels + 1 device copy; round 1: 9 kernels + 4 copies):
    //   1. s_new = interp(s, x - dt v) + rate * inflow                      advection with the inflow as epilogue
    //   2. v*    = (interp(v, faces - dt v) + dt * buoyancy(s_new)) [* f]   all components in one launch, buoyancy and the
    //                                                                        obstacle face factors as epilogues
    //   3. s     <- s_new                                                    (the only copy: s cannot be advected in place)
    //   4. div   = divergence(v*)     5. p = CG(div, x0 = p)                 6. v = v* - grad p   (written into the caller's v)
    DGrid dg; DVec dv; DField sf;
    CHECK(phi_make_dgrid(g, &dg));
    if (!sp || !scratch || !s || !p || !v) { phi_set_error("plume_step: NULL argument"); return PHI_ERR_INVALID; }
    CHECK(make_vec(g, vbc, v, &dv)); CHECK(phi_make_centered(g, sbc, &sf));
    const size_t carr = centred_elems(g), farr = face_elems(g);
    float* s_new = scratch;                 // advected smoke
    float* tmp = scratch + carr;            // MacCormack scratch, later the divergence
    float* vn[3] = {nullptr, nullptr, nullptr};
    DVecOut out;
    for (int c = 0; c < 3; ++c) { vn[c] = c < g->dim ? scratch + 2 * carr + c * farr : nullptr; out.p[c] = vn[c]; }
    cudaStream_t st = (cudaStream_t)stream;
    const bool has_inflow = inflow && sp->inflow_rate != 0.f;
    const bool big = (long long)farr > (1ll << 31) - (1ll << 20);     // beyond 32-bit element offsets: 64-bit scalar kernels
    if (sp->static_scalar) {                // forced step: s is a stationary source field
        if (phi_scalar_kernels() || big) {
            CHECK(phicuda_advect_staggered_f32(g, vbc, v, vbc, v, vn, sp->dt, stream));
            CHECK(phicuda_add_buoyancy_f32(g, vbc, sbc, s, sp->buoyancy, sp->dt, vn, stream));
            if (faces) CHECK(phicuda_mul_faces_f32(g, vbc, vn, faces, stream));
        } else {
            CHECK(cuda_fail(phi_launch_advect_staggered_vec(dg, dv, dv, out, sp->dt, &sf, s, sp->buoyancy, faces, st), "advect_staggered"));
        }
        return project(g, vbc, vn, v, p, tmp, accessible, prm, result, workspace, workspace_bytes, sp->cg_start_event, sp->cg_stop_event, stream);
    }
    if (phi_scalar_kernels() || big) {      // round-1 sequence, kept for A/B comparisons
        if (sp->mac_cormack) CHECK(phicuda_mac_cormack_centered_f32(g, vbc, v, sbc, s, s_new, tmp, sp->dt, 1.0f, stream));
        else                 CHECK(phicuda_advect_centered_f32(g, vbc, v, sbc, s, s_new, sp->dt, stream));
        if (has_inflow) CHECK(phicuda_axpy_centered_f32(g, sp->inflow_rate, inflow, s_new, stream));
        CHECK(phicuda_advect_staggered_f32(g, vbc, v, vbc, v, vn, sp->dt, stream));
        CHECK(phicuda_add_buoyancy_f32(g, vbc, sbc, s_new, sp->buoyancy, sp->dt, vn, stream));
        if (faces) CHECK(phicuda_mul_faces_f32(g, vbc, vn, faces, stream));
    } else {
        if (sp->mac_cormack) {
            CHECK(cuda_fail(phi_launch_mac_cormack(dg, dv, sf, s, s_new, tmp, sp->dt, 1.0f, st), "mac_cormack"));
            if (has_inflow) CHECK(phicuda_axpy_centered_f32(g, sp->inflow_rate, inflow, s_new, stream));
        } else {
            CHECK(cuda_fail(phi_launch_advect_centered_vec(dg, dv, sf, s, s_new, sp->dt, has_inflow ? inflow : nullptr, sp->inflow_rate, st), "advect_centered"));
        }
        CHECK(cuda_fail(phi_launch_advect_staggered_vec(dg, dv, dv, out, sp->dt, &sf, s_new, sp->buoyancy, faces, st), "advect_staggered"));
    }
    cudaError_t e = cudaMemcpyAsync(s, s_new, carr * sizeof(float), cudaMemcpyDeviceToDevice, st);
    if (e) return cuda_fail(e, "plume_step copy s");
    return project(g, vbc, vn, v, p, tmp, accessible, prm, result, workspace, workspace_bytes, sp->cg_start_event, sp->cg_stop_event, stream);
}

int phicuda_plume_step_f32(const PhiGrid* g, const PhiVBC* vbc, const PhiBC* sbc, float* const v[3], float* s, float* p,
                           const float* inflow, const PhiPlumeParams* sp, const PhiCgParams* prm, PhiCgResult* result,
                           float* scratch, void* workspace, size_t workspace_bytes, void* stream)
{
    return plume_step(g, vbc, sbc, v, s, p, inflow, nullptr, nullptr, sp, prm, result, scratch, workspace, workspace_bytes, stream);
}

int phicuda_plume_step_masked_f32(const PhiGrid* g, const PhiVBC* vbc, const PhiBC* sbc, float* const v[3], float* s, float* p,
                                  const float* inflow, const float* accessible, const float* const face_factors[3],
                                  const PhiPlumeParams* sp, const PhiCgParams* prm, PhiCgResult* result,
                                  float* scratch, void* workspace, size_t workspace_bytes, void* stream)
{
    // every check of the step, its projection and its solve runs before the first CUDA call: a refused step leaves the state untouched
    DGrid dg; DVec dv; DField sf, cf, pf, af; PhiBC none, pbc; memset(&none, 0, sizeof(none));
    CHECK(phi_make_dgrid(g, &dg));
    if (!sp || !scratch || !s || !p || !v || !prm || !result || !workspace) { phi_set_error("plume_step_masked: NULL argument"); return PHI_ERR_INVALID; }
    if (!accessible || !face_factors) { phi_set_error("plume_step_masked: accessible / face_factors is NULL"); return PHI_ERR_INVALID; }
    for (int c = 0; c < g->dim; ++c)
        if (!face_factors[c]) { phi_set_error("plume_step_masked: face_factors[%d] is NULL", c); return PHI_ERR_INVALID; }
    if (g->halo != 0) { phi_set_error("plume_step_masked: z-slab grids are not supported (slab runs sequence the step in dist.py)"); return PHI_ERR_UNSUPPORTED; }
    CHECK(make_vec(g, vbc, v, &dv)); CHECK(phi_make_centered(g, sbc, &sf)); CHECK(phi_make_centered(g, &none, &cf));
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, &pf)); CHECK(accessible_field(g, vbc, &af));
    if (g->batch > CG_MAX_BATCH) { phi_set_error("cg: batch %d exceeds %d (split the batch)", g->batch, CG_MAX_BATCH); return PHI_ERR_UNSUPPORTED; }
    const size_t ws_need = phi_cg_workspace(dg, nullptr).bytes;
    if (workspace_bytes < ws_need) { phi_set_error("cg: workspace %zu < %zu bytes", workspace_bytes, ws_need); return PHI_ERR_WORKSPACE; }
    const bool adaptive = prm->method == PHI_SOLVER_CG_ADAPTIVE;
    if (prm->method != PHI_SOLVER_CG && !adaptive) { phi_set_error("cg: unknown solver method %d", prm->method); return PHI_ERR_INVALID; }
    if (prm->matrix_offset != 0.f) {
        phi_set_error(adaptive ? "cg: CG-adaptive does not take a matrix_offset" : "cg: matrix_offset is not supported together with obstacles");
        return PHI_ERR_UNSUPPORTED;
    }
    if (adaptive && (!phi_ring_enabled() || !phi_cg_ring_fits(dg, CgOp::Masked))) {     // the message of phi_launch_cg
        if (!phi_ring_enabled()) phi_set_error("cg: CG-adaptive runs on the TMA ring kernel only, which PHICUDA_NO_RING switches off");
        else phi_set_error("cg: CG-adaptive runs on the TMA ring kernel only; grid lines of %d cells do not fit it (%d-D%s, batch %d: at most %d cells)",
                           g->n[0], g->dim, " with obstacles", g->batch, phi_cg_ring_max_width(dg, CgOp::Masked, true));
        return PHI_ERR_UNSUPPORTED;
    }
    return plume_step(g, vbc, sbc, v, s, p, inflow, accessible, face_factors, sp, prm, result, scratch, workspace, workspace_bytes, stream);
}

static bool overlap(const void* a, size_t a_bytes, const void* b, size_t b_bytes) { return (const char*)a < (const char*)b + b_bytes && (const char*)b < (const char*)a + a_bytes; }

// a persistent stepper runs on its TMA ring only: refuses PHICUDA_NO_RING and lines longer than the ring takes, naming the widest
static int ring_only(const char* name, const PhiGrid* g, const DGrid& dg, int kernel)
{
    if (!phi_ring_enabled()) { phi_set_error("%s: runs on the TMA ring kernel only, which PHICUDA_NO_RING switches off", name); return PHI_ERR_UNSUPPORTED; }
    if (!phi_step_ring_fits(dg, kernel)) {
        phi_set_error("%s: grid lines of %d cells do not fit the TMA ring (%d-D: at most %d cells)", name, g->n[0], g->dim, phi_step_ring_max_width(dg, kernel));
        return PHI_ERR_UNSUPPORTED;
    }
    return 0;
}

size_t phicuda_reaction_diffusion_scratch_bytes(const PhiGrid* g)
{
    return g ? 2 * centred_elems(g) * sizeof(float) : 0;
}

int phicuda_reaction_diffusion_f32(const PhiGrid* g, const PhiVBC* bc, float* u, float* v, float du, float dv, float f, float k,
                                   float dt, int32_t substeps, float* scratch, size_t scratch_bytes, void* stream)
{
    // every check runs before the first CUDA call: a refused call leaves u and v untouched
    DGrid dg; DField fu, fv;
    CHECK(phi_make_dgrid(g, &dg));
    if (!bc || !u || !v || !scratch) { phi_set_error("reaction_diffusion: NULL argument"); return PHI_ERR_INVALID; }
    if (substeps < 0) { phi_set_error("reaction_diffusion: substeps must be >= 0, got %d", substeps); return PHI_ERR_INVALID; }
    if (!std::isfinite(du) || !std::isfinite(dv) || !std::isfinite(f) || !std::isfinite(k) || !std::isfinite(dt)) {
        phi_set_error("reaction_diffusion: du, dv, f, k and dt must be finite"); return PHI_ERR_INVALID;
    }
    const size_t n = centred_elems(g);
    const size_t need = phicuda_reaction_diffusion_scratch_bytes(g);
    if (scratch_bytes < need) { phi_set_error("reaction_diffusion: scratch %zu < %zu bytes", scratch_bytes, need); return PHI_ERR_INVALID; }
    if (overlap(u, 4 * n, v, 4 * n)) { phi_set_error("reaction_diffusion: u and v must be distinct arrays (they overlap)"); return PHI_ERR_INVALID; }
    if (overlap(scratch, need, u, 4 * n) || overlap(scratch, need, v, 4 * n)) {
        phi_set_error("reaction_diffusion: scratch overlaps u or v"); return PHI_ERR_INVALID;
    }
    if (g->halo != 0) { phi_set_error("reaction_diffusion: z-slab grids are not supported"); return PHI_ERR_UNSUPPORTED; }
    CHECK(phi_make_centered(g, &bc->comp[0], &fu)); CHECK(phi_make_centered(g, &bc->comp[1], &fv));
    for (int a = 0; a < g->dim; ++a) {
        if (bc->comp[0].lo[a] != bc->comp[1].lo[a] || bc->comp[0].hi[a] != bc->comp[1].hi[a]) {
            phi_set_error("reaction_diffusion: the boundary kinds of u and v must agree (axis %d)", a); return PHI_ERR_UNSUPPORTED;
        }
        for (int c = 0; c < 2; ++c)
            if ((bc->comp[c].lo[a] == PHI_BC_CONST && bc->comp[c].clo[a] != 0.f) || (bc->comp[c].hi[a] == PHI_BC_CONST && bc->comp[c].chi[a] != 0.f)) {
                phi_set_error("reaction_diffusion: non-zero constant boundary on axis %d of %s: the reference's step turns a constant c into "
                              "2c - c^2 (field (-) number keeps the field's extrapolation), so its ghosts are not fixed", a, c ? "v" : "u");
                return PHI_ERR_UNSUPPORTED;
            }
    }
    CHECK(ring_only("reaction_diffusion", g, dg, PHI_KERNEL_RD_RING));
    if (substeps == 0) return 0;
    RdParams p;
    p.du = du; p.dv = dv; p.f = f; p.fk = f + k; p.dt = dt;
    const int e = phi_launch_reaction_diffusion(dg, fu, u, v, scratch, scratch + n, p, substeps, (cudaStream_t)stream);
    if (e == -100) { phi_set_error("reaction_diffusion: the grid does not fit the TMA ring on this device"); return PHI_ERR_UNSUPPORTED; }
    return cuda_fail(e, "reaction_diffusion");
}

// scratch of the wave step: [one centred array, for an odd count][substeps WaveDisc][cell centres along each axis]
static size_t wave_tmp_bytes(const PhiGrid* g) { return (centred_elems(g) * sizeof(float) + 15) / 16 * 16; }
static size_t wave_table_bytes(const PhiGrid* g, int32_t substeps)
{
    return (size_t)substeps * sizeof(WaveDisc) + (size_t)(g->n[0] + g->n[1] + (g->dim == 3 ? g->n[2] : 0)) * sizeof(float);
}

size_t phicuda_wave_scratch_bytes(const PhiGrid* g, int32_t substeps)
{
    return g && substeps >= 0 ? wave_tmp_bytes(g) + wave_table_bytes(g, substeps) : 0;
}

int phicuda_wave_f32(const PhiGrid* g, const PhiBC* bc, float* h_c, float* h_p, float dd, float k_speed, float k_damp,
                     const PhiWaveDisc* discs, float radius_sq, const float* centers, int32_t substeps, void* scratch,
                     size_t scratch_bytes, void* stream)
{
    // every check runs before the first CUDA call: a refused call leaves h_c and h_p untouched
    DGrid dg; DField f;
    CHECK(phi_make_dgrid(g, &dg));
    if (!bc || !h_c || !h_p || !discs || !centers || !scratch) { phi_set_error("wave: NULL argument"); return PHI_ERR_INVALID; }
    if (substeps < 0) { phi_set_error("wave: substeps must be >= 0, got %d", substeps); return PHI_ERR_INVALID; }
    if (!std::isfinite(dd) || !std::isfinite(k_speed) || !std::isfinite(k_damp) || !std::isfinite(radius_sq)) {
        phi_set_error("wave: dd, k_speed, k_damp and radius_sq must be finite"); return PHI_ERR_INVALID;
    }
    const int naxis = g->n[0] + g->n[1] + (g->dim == 3 ? g->n[2] : 0);
    for (int i = 0; i < naxis; ++i)
        if (!std::isfinite(centers[i])) { phi_set_error("wave: cell centre %d is not finite", i); return PHI_ERR_INVALID; }
    for (int s = 0; s < substeps; ++s) {
        if (!discs[s].present) continue;
        bool ok = std::isfinite(discs[s].value);
        for (int a = 0; a < g->dim; ++a) ok = ok && std::isfinite(discs[s].center[a]);
        if (!ok) { phi_set_error("wave: disc %d has a non-finite centre or value", s); return PHI_ERR_INVALID; }
    }
    const size_t n = centred_elems(g);
    const size_t need = phicuda_wave_scratch_bytes(g, substeps);
    if (scratch_bytes < need) { phi_set_error("wave: scratch %zu < %zu bytes", scratch_bytes, need); return PHI_ERR_INVALID; }
    if (overlap(h_c, 4 * n, h_p, 4 * n)) { phi_set_error("wave: h_c and h_p must be distinct arrays (they overlap)"); return PHI_ERR_INVALID; }
    if (overlap(scratch, need, h_c, 4 * n) || overlap(scratch, need, h_p, 4 * n)) {
        phi_set_error("wave: scratch overlaps h_c or h_p"); return PHI_ERR_INVALID;
    }
    if (g->halo != 0) { phi_set_error("wave: z-slab grids are not supported"); return PHI_ERR_UNSUPPORTED; }
    CHECK(phi_make_centered(g, bc, &f));
    for (int a = 0; a < g->dim; ++a)
        if ((bc->lo[a] == PHI_BC_CONST && bc->clo[a] != 0.f) || (bc->hi[a] == PHI_BC_CONST && bc->chi[a] != 0.f)) {
            phi_set_error("wave: non-zero constant boundary on axis %d: the reference's step turns a constant c into c - c = 0 "
                          "(2.0 * h_c keeps h_c's extrapolation), so its ghosts are not fixed", a);
            return PHI_ERR_UNSUPPORTED;
        }
    CHECK(ring_only("wave", g, dg, PHI_KERNEL_WAVE_RING));
    if (substeps == 0) return 0;
    // the disc table: per axis the index range of cells whose own term fl(fl(p - c)^2) is <= r^2 (the float32 operations of the
    // kernel's test), which holds every cell of the disc because a float sum of non-negative terms is no smaller than any term
    std::vector<unsigned char> table(wave_table_bytes(g, substeps));
    WaveDisc* wd = reinterpret_cast<WaveDisc*>(table.data());
    for (int s = 0; s < substeps; ++s) {
        WaveDisc d; memset(&d, 0, sizeof(d));
        d.value = discs[s].value;
        for (int a = 0; a < 3; ++a) d.c[a] = a < g->dim ? discs[s].center[a] : 0.f;
        bool empty = !discs[s].present;
        const float* p = centers;
        for (int a = 0; a < g->dim && !empty; p += g->n[a], ++a) {
            int lo = g->n[a], hi = 0;
            for (int i = 0; i < g->n[a]; ++i) {
                const float t = p[i] - d.c[a];
                const float t2 = t * t;
                if (t2 <= radius_sq) { if (i < lo) lo = i; hi = i + 1; }
            }
            if (lo >= hi) empty = true;
            d.lo[a] = lo; d.hi[a] = hi;
        }
        if (g->dim == 2) { d.lo[2] = 0; d.hi[2] = 1; }
        if (empty) for (int a = 0; a < 3; ++a) d.lo[a] = d.hi[a] = 0;
        wd[s] = d;
    }
    memcpy(table.data() + (size_t)substeps * sizeof(WaveDisc), centers, (size_t)naxis * sizeof(float));
    unsigned char* dtab = (unsigned char*)scratch + wave_tmp_bytes(g);
    cudaError_t ce = cudaMemcpyAsync(dtab, table.data(), table.size(), cudaMemcpyHostToDevice, (cudaStream_t)stream);
    if (ce != cudaSuccess) return cuda_fail((int)ce, "wave");
    WaveParams wp;
    wp.dd = dd; wp.k_speed = k_speed; wp.k_damp = k_damp; wp.r2 = radius_sq;
    const int e = phi_launch_wave(dg, f, h_c, h_p, (float*)scratch, reinterpret_cast<const WaveDisc*>(dtab),
                                  reinterpret_cast<const float*>(dtab + (size_t)substeps * sizeof(WaveDisc)), wp, substeps, (cudaStream_t)stream);
    if (e == -100) { phi_set_error("wave: the grid does not fit the TMA ring on this device"); return PHI_ERR_UNSUPPORTED; }
    return cuda_fail(e, "wave");
}

// scratch of the Julia counts: [batch (re, im) pairs of c][n[0] x centres][n[1] y centres]
size_t phicuda_julia_scratch_bytes(const PhiGrid* g)
{
    return g ? (2 * (size_t)g->batch + (size_t)g->n[0] + (size_t)g->n[1]) * sizeof(float) : 0;
}

int phicuda_julia_f32(const PhiGrid* g, const float* centers, const float* c, int32_t iterations, int32_t* counts, void* scratch,
                      size_t scratch_bytes, void* stream)
{
    // every check runs before the first CUDA call: a refused call leaves counts untouched
    DGrid dg;
    CHECK(phi_make_dgrid(g, &dg));
    if (g->dim != 2) { phi_set_error("julia: 2-D grids only, got %d-D", g->dim); return PHI_ERR_UNSUPPORTED; }
    if (!centers || !c || !counts || !scratch) { phi_set_error("julia: NULL argument"); return PHI_ERR_INVALID; }
    if (iterations < 0) { phi_set_error("julia: iterations must be >= 0, got %d", iterations); return PHI_ERR_INVALID; }
    const int naxis = g->n[0] + g->n[1];
    for (int i = 0; i < naxis; ++i)
        if (!std::isfinite(centers[i])) { phi_set_error("julia: cell centre %d is not finite", i); return PHI_ERR_INVALID; }
    const size_t need = phicuda_julia_scratch_bytes(g);
    if (scratch_bytes < need) { phi_set_error("julia: scratch %zu < %zu bytes", scratch_bytes, need); return PHI_ERR_INVALID; }
    if (overlap(scratch, need, counts, centred_elems(g) * sizeof(int32_t))) { phi_set_error("julia: scratch overlaps counts"); return PHI_ERR_INVALID; }
    std::vector<float> table(need / sizeof(float));
    memcpy(table.data(), c, 2 * (size_t)g->batch * sizeof(float));
    memcpy(table.data() + 2 * (size_t)g->batch, centers, (size_t)naxis * sizeof(float));
    float* dtab = (float*)scratch;
    cudaError_t ce = cudaMemcpyAsync(dtab, table.data(), need, cudaMemcpyHostToDevice, (cudaStream_t)stream);
    if (ce != cudaSuccess) return cuda_fail((int)ce, "julia");
    const float* xc = dtab + 2 * (size_t)g->batch;
    return cuda_fail(phi_launch_julia(dg, dtab, xc, xc + g->n[0], iterations, counts, (cudaStream_t)stream), "julia");
}

int phicuda_advect_points_f32(const PhiGrid* g, const PhiVBC* vbc, const float* const vel[3], const PhiPointMap* map,
                              const float* points, int64_t npoints, int32_t points_batch, float dt, int32_t integrator,
                              int32_t steps, float* out, float* trajectory, void* stream)
{
    // every check runs before the first CUDA call: a refused call leaves out and trajectory untouched
    DGrid dg; DVec dv;
    CHECK(phi_make_dgrid(g, &dg));
    if (g->halo != 0) { phi_set_error("advect_points: z-slab grids are not supported"); return PHI_ERR_UNSUPPORTED; }
    CHECK(make_vec(g, vbc, vel, &dv));
    if (!map || !points || !out) { phi_set_error("advect_points: NULL argument"); return PHI_ERR_INVALID; }
    if (npoints < 0) { phi_set_error("advect_points: npoints must be >= 0, got %lld", (long long)npoints); return PHI_ERR_INVALID; }
    if (steps < 1) { phi_set_error("advect_points: steps must be >= 1, got %d", steps); return PHI_ERR_INVALID; }
    if (integrator != PHI_INTEGRATOR_EULER && integrator != PHI_INTEGRATOR_RK4) { phi_set_error("advect_points: unknown integrator %d", integrator); return PHI_ERR_INVALID; }
    if (points_batch < 1 || (points_batch != 1 && g->batch != 1 && points_batch != g->batch)) {
        phi_set_error("advect_points: points batch %d does not broadcast against grid batch %d", points_batch, g->batch); return PHI_ERR_INVALID;
    }
    for (int c = 0; c < g->dim; ++c) {
        const DField& f = dv.f[c];
        if ((long long)f.sb > INT_MAX) { phi_set_error("advect_points: component %d holds more than 2^31 elements per batch entry", c); return PHI_ERR_UNSUPPORTED; }
        for (int a = 0; a < g->dim; ++a) {
            const float lo = map->lower[c][a], sz = map->size[c][a], r = map->res[c][a];
            if (r != (float)(f.hi[a] - f.lo[a] + 1)) {
                phi_set_error("advect_points: map res[%d][%d] = %g but component %d stores %d values along axis %d", c, a, r, c, f.hi[a] - f.lo[a] + 1, a);
                return PHI_ERR_INVALID;
            }
            if (!(std::isfinite(sz) && sz > 0.f) || !std::isfinite(lo)) {
                phi_set_error("advect_points: map lower[%d][%d] = %g, size = %g (finite, size > 0 required)", c, a, lo, sz); return PHI_ERR_INVALID;
            }
        }
    }
    const long long B = g->batch > points_batch ? g->batch : points_batch;
    if ((unsigned __int128)npoints * (unsigned)B * (unsigned)(steps + 1) * (unsigned)g->dim * sizeof(float) > (unsigned __int128)INT64_MAX) {
        phi_set_error("advect_points: %lld points x %lld batch x %d steps exceeds 64-bit offsets", (long long)npoints, B, steps); return PHI_ERR_INVALID;
    }
    const size_t in_bytes = (size_t)npoints * points_batch * g->dim * sizeof(float), out_bytes = (size_t)npoints * B * g->dim * sizeof(float);
    const size_t traj_bytes = out_bytes * ((size_t)steps + 1);
    if (out != points && overlap(out, out_bytes, points, in_bytes)) { phi_set_error("advect_points: out overlaps points without being points"); return PHI_ERR_INVALID; }
    if (out == points && points_batch != B) { phi_set_error("advect_points: out may be points only when points are not broadcast (batch %d < %lld)", points_batch, B); return PHI_ERR_INVALID; }
    if (trajectory && (overlap(trajectory, traj_bytes, points, in_bytes) || overlap(trajectory, traj_bytes, out, out_bytes))) {
        phi_set_error("advect_points: trajectory overlaps points or out"); return PHI_ERR_INVALID;
    }
    const size_t fbytes = face_elems(g) * sizeof(float);
    for (int c = 0; c < g->dim; ++c)
        if (overlap(out, out_bytes, vel[c], fbytes) || (trajectory && overlap(trajectory, traj_bytes, vel[c], fbytes))) {
            phi_set_error("advect_points: out or trajectory overlaps velocity component %d", c); return PHI_ERR_INVALID;
        }
    if (npoints == 0) return 0;
    return cuda_fail(phi_launch_advect_points(dg, dv, *map, points, (long long)npoints, points_batch, dt, integrator, steps, out,
                                              trajectory, (cudaStream_t)stream), "advect_points");
}

// The kernel's SphParams from the public ones; 0 or the error code of the first check that fails.
static int sph_params(int64_t n, int32_t dim, const PhiSphParams* prm, SphParams* out)
{
    if (!prm) { phi_set_error("sph: NULL parameters"); return PHI_ERR_INVALID; }
    if (dim != 2 && dim != 3) { phi_set_error("sph: dim must be 2 or 3, got %d", dim); return PHI_ERR_INVALID; }
    if (n < 0 || n > (1 << 30)) { phi_set_error("sph: n must be in [0, 2^30], got %lld", (long long)n); return PHI_ERR_INVALID; }
    const float scalars[] = {prm->support, prm->smoothing_length, prm->kernel_norm, prm->mass, prm->pressure_norm, prm->viscous_norm,
                             prm->isotropic_exp, prm->base_density, prm->dt, prm->damping};
    for (float f : scalars)
        if (!std::isfinite(f)) { phi_set_error("sph: every parameter must be finite"); return PHI_ERR_INVALID; }
    if (!(prm->support > 0.f)) { phi_set_error("sph: support must be > 0, got %g", prm->support); return PHI_ERR_INVALID; }
    SphParams p = {};
    p.n = (int)n; p.dim = dim;
    double cells = 1;
    for (int a = 0; a < dim; ++a) {
        const float lo = prm->lower[a], up = prm->upper[a];
        if (!std::isfinite(lo) || !std::isfinite(up) || !std::isfinite(prm->gravity[a]) || !(lo < up)) {
            phi_set_error("sph: axis %d: lower %g < upper %g and gravity %g must be finite", a, lo, up, prm->gravity[a]); return PHI_ERR_INVALID;
        }
        // build_hash_grid in float32: res = max(1, ceil(max(upper - lower, s) / s)), edge = (s res) / res
        float size = up - lo;
        if (!(size >= prm->support)) size = prm->support;
        const float q = std::ceil(size / prm->support);
        if (!(q < (float)(1 << 30))) { phi_set_error("sph: axis %d needs %g hash cells", a, q); return PHI_ERR_INVALID; }
        const int r = q < 1.f ? 1 : (int)q;
        cells *= r;
        p.res[a] = r;
        p.lower[a] = lo; p.upper[a] = up;
        p.cell[a] = (prm->support * (float)r) / (float)r;
        p.gravity[a] = prm->gravity[a];
    }
    if (cells > (double)(1 << 30)) { phi_set_error("sph: %g hash cells exceed 2^30 (the support is too small for the domain)", cells); return PHI_ERR_INVALID; }
    p.ncells = (int)cells;
    p.s = prm->support; p.h = prm->smoothing_length; p.norm = prm->kernel_norm; p.m = prm->mass; p.P = prm->pressure_norm;
    p.V = prm->viscous_norm; p.iso = prm->isotropic_exp; p.base = prm->base_density; p.dt = prm->dt; p.damping = prm->damping;
    *out = p;
    return 0;
}

size_t phicuda_sph_scratch_bytes(int64_t n, int32_t dim, const PhiSphParams* prm)
{
    SphParams p;
    return sph_params(n, dim, prm, &p) ? 0 : phi_sph_scratch_bytes(p);
}

int phicuda_sph_f32(const float* x, const float* v, int64_t n, int32_t dim, const PhiSphParams* prm, int32_t substeps, float* x_out,
                    float* v_out, float* rho_out, void* scratch, size_t scratch_bytes, void* stream)
{
    // every check runs before the first CUDA call: a refused call leaves x_out, v_out and rho_out untouched
    SphParams p;
    CHECK(sph_params(n, dim, prm, &p));
    if (substeps < 1) { phi_set_error("sph: substeps must be >= 1, got %d", substeps); return PHI_ERR_INVALID; }
    if (n == 0) return 0;
    if (!x || !v || !x_out || !v_out || !scratch) { phi_set_error("sph: NULL argument"); return PHI_ERR_INVALID; }
    const size_t need = phi_sph_scratch_bytes(p);
    if (scratch_bytes < need) { phi_set_error("sph: scratch %zu < %zu bytes", scratch_bytes, need); return PHI_ERR_INVALID; }
    const size_t vec = (size_t)n * dim * sizeof(float), sc = (size_t)n * sizeof(float);
    const void* outs[] = {x_out, v_out, rho_out, scratch};
    const size_t out_bytes[] = {vec, vec, sc, need};
    for (int a = 0; a < 4; ++a) {
        if (!outs[a]) continue;
        if (overlap(outs[a], out_bytes[a], x, vec) || overlap(outs[a], out_bytes[a], v, vec)) {
            phi_set_error("sph: an output or the scratch overlaps x or v"); return PHI_ERR_INVALID;
        }
        for (int b = a + 1; b < 4; ++b)
            if (outs[b] && overlap(outs[a], out_bytes[a], outs[b], out_bytes[b])) {
                phi_set_error("sph: the outputs and the scratch must not overlap each other"); return PHI_ERR_INVALID;
            }
    }
    int max_ctas = SPH_MAX_CTAS;
    if (const char* e = getenv("PHICUDA_SPH_CTAS")) { const int c = atoi(e); if (c >= 1 && c < max_ctas) max_ctas = c; }   // launch-geometry tests
    return cuda_fail(phi_launch_sph(p, x, v, x_out, v_out, rho_out, scratch, substeps, max_ctas, (cudaStream_t)stream), "sph");
}

}  // extern "C"

// ---- N9: fp64 ------------------------------------------------------------------------------------------------------------
// The float fields of PhiGrid / PhiBC describe the layout and kinds and must equal the exact values rounded to float; the kernels
// take the exact values from PhiValues64.  Every check runs before the first CUDA call.
static const double kZero3[3] = {0.0, 0.0, 0.0};

static int check_values64(const PhiGrid* g, const PhiBC* bcs, int ncomp, const PhiValues64* val, const char* what)
{
    if (!val) { phi_set_error("%s: values (PhiValues64) is NULL", what); return PHI_ERR_INVALID; }
    if (g->halo != 0) { phi_set_error("%s: z-slab grids (halo %d) are not supported; the fp64 path runs on one GPU", what, g->halo); return PHI_ERR_UNSUPPORTED; }
    for (int a = 0; a < g->dim; ++a)
        if (!((float)val->dx[a] == g->dx[a])) {
            phi_set_error("%s: values.dx[%d] = %.17g does not round to grid.dx[%d] = %.9g", what, a, val->dx[a], a, (double)g->dx[a]);
            return PHI_ERR_INVALID;
        }
    for (int c = 0; c < ncomp; ++c)
        for (int a = 0; a < g->dim; ++a)
            if (!((float)val->clo[c][a] == bcs[c].clo[a]) || !((float)val->chi[c][a] == bcs[c].chi[a])) {
                phi_set_error("%s: values.clo/chi[%d][%d] = %.17g / %.17g do not round to the boundary's %.9g / %.9g", what, c, a,
                              val->clo[c][a], val->chi[c][a], (double)bcs[c].clo[a], (double)bcs[c].chi[a]);
                return PHI_ERR_INVALID;
            }
    return 0;
}

// after check_values64: the grid with the exact cell sizes, 1 / dx = RN(1 / dx) in double
static DGridT<double> dgrid64(const DGrid& f, const PhiValues64* val)
{
    DGridT<double> o;
    o.dim = f.dim; o.batch = f.batch; o.halo = f.halo;
    for (int a = 0; a < 3; ++a) {
        const bool used = a < f.dim;
        o.n[a] = f.n[a]; o.cext[a] = f.cext[a]; o.fext[a] = f.fext[a];
        o.dx[a] = used ? val->dx[a] : 1.0;
        o.inv_dx[a] = used ? 1.0 / val->dx[a] : 0.0;
        o.inv_dx2[a] = used ? 1.0 / (val->dx[a] * val->dx[a]) : 0.0;
    }
    return o;
}

static DFieldT<double> field64(const DField& f, const double clo[3], const double chi[3], int dim)
{
    DFieldT<double> o;
    for (int a = 0; a < 3; ++a) {
        o.lo[a] = f.lo[a]; o.hi[a] = f.hi[a]; o.klo[a] = f.klo[a]; o.khi[a] = f.khi[a];
        o.clo[a] = a < dim ? clo[a] : 0.0; o.chi[a] = a < dim ? chi[a] : 0.0;
    }
    o.sy = f.sy; o.sz = f.sz; o.sb = f.sb; o.halo = f.halo;
    return o;
}

static int make_vec64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* val, const double* const v[3], DVecT<double>* o)
{
    DVec f;
    if (!v) { phi_set_error("vector field / boundary is NULL"); return PHI_ERR_INVALID; }
    const float* vp[3] = {(const float*)v[0], (const float*)v[1], (const float*)v[2]};     // make_vec checks and keeps the addresses
    CHECK(make_vec(g, vbc, vp, &f));
    for (int c = 0; c < 3; ++c) {
        o->p[c] = c < g->dim ? v[c] : nullptr;
        o->f[c] = c < g->dim ? field64(f.f[c], val->clo[c], val->chi[c], g->dim) : field64(f.f[c], kZero3, kZero3, 0);
    }
    return 0;
}

// Every check of an fp64 pressure solve: fills l without a CUDA call.
static int cg_setup64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* val, const double* rhs, double* x, const PhiCgParams64* prm,
                      PhiCgResult64* result, void* workspace, size_t workspace_bytes, CgLaunch64* l)
{
    DGrid dg; PhiBC pbc; DField pf;
    CHECK(phi_make_dgrid(g, &dg));
    if (!vbc || !rhs || !x || !prm || !result || !workspace) { phi_set_error("cg_f64: NULL argument"); return PHI_ERR_INVALID; }
    for (int a = 0; a < g->dim; ++a) CHECK(check_bc(&vbc->comp[a], g->dim));
    CHECK(check_values64(g, vbc->comp, g->dim, val, "cg_f64"));
    if (prm->method == PHI_SOLVER_CG_ADAPTIVE) { phi_set_error("cg_f64: CG-adaptive runs on the fp32 TMA ring kernel only; fp64 solves take PHI_SOLVER_CG"); return PHI_ERR_UNSUPPORTED; }
    if (prm->method != PHI_SOLVER_CG) { phi_set_error("cg_f64: unknown solver method %d", prm->method); return PHI_ERR_INVALID; }
    if (g->batch > CG_MAX_BATCH) { phi_set_error("cg_f64: batch %d exceeds %d (split the batch)", g->batch, CG_MAX_BATCH); return PHI_ERR_UNSUPPORTED; }
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, &pf));
    l->g = dgrid64(dg, val);
    l->pf = field64(pf, kZero3, kZero3, g->dim);              // the pressure boundary has no constants
    const size_t need = phi_cg_workspace_bytes_f64(l->g);
    if (workspace_bytes < need) { phi_set_error("cg_f64: workspace %zu < %zu bytes", workspace_bytes, need); return PHI_ERR_WORKSPACE; }
    l->rhs = rhs; l->x = x; l->prm = *prm; l->result = result; l->workspace = workspace; l->workspace_bytes = workspace_bytes;
    return 0;
}

extern "C" {

static int laplace64(const PhiGrid* g, const PhiBC* bc, const PhiValues64* val, const double* x, double coeff, double* y, bool axpy,
                     void* stream, const char* what)
{
    DGrid dg; DField f;
    CHECK(phi_make_dgrid(g, &dg)); CHECK(phi_make_centered(g, bc, &f));
    CHECK(check_values64(g, bc, 1, val, what));
    if (!x || !y || x == y) { phi_set_error("%s: x and y must be distinct non-NULL arrays", what); return PHI_ERR_INVALID; }
    return cuda_fail(phi_launch_laplace(dgrid64(dg, val), field64(f, val->clo[0], val->chi[0], g->dim), x, y, coeff, axpy,
                                        (cudaStream_t)stream), what);
}

int phicuda_laplace_f64(const PhiGrid* g, const PhiBC* bc, const PhiValues64* values, const double* x, double* y, void* stream)
{
    return laplace64(g, bc, values, x, 0.0, y, false, stream, "laplace_f64");
}

int phicuda_laplace_axpy_f64(const PhiGrid* g, const PhiBC* bc, const PhiValues64* values, const double* x, double coeff, double* y,
                             void* stream)
{
    return laplace64(g, bc, values, x, coeff, y, true, stream, "laplace_axpy_f64");
}

int phicuda_divergence_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* values, const double* const v[3], double* div,
                           void* stream)
{
    DGrid dg; DVecT<double> dv; DField cf; PhiBC none; memset(&none, 0, sizeof(none));
    CHECK(phi_make_dgrid(g, &dg));
    if (!vbc) { phi_set_error("divergence_f64: boundary is NULL"); return PHI_ERR_INVALID; }
    CHECK(check_values64(g, vbc->comp, g->dim, values, "divergence_f64"));
    CHECK(make_vec64(g, vbc, values, v, &dv)); CHECK(phi_make_centered(g, &none, &cf));
    if (!div) { phi_set_error("divergence_f64: div is NULL"); return PHI_ERR_INVALID; }
    return cuda_fail(phi_launch_divergence(dgrid64(dg, values), dv, field64(cf, kZero3, kZero3, g->dim), div, (cudaStream_t)stream),
                     "divergence_f64");
}

int phicuda_grad_sub_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* values, double* const v[3], const double* p,
                         void* stream)
{
    DGrid dg; DVecT<double> dv; DVecOutT<double> out; PhiBC pbc; DField pf;
    CHECK(phi_make_dgrid(g, &dg));
    if (!vbc) { phi_set_error("grad_sub_f64: boundary is NULL"); return PHI_ERR_INVALID; }
    CHECK(check_values64(g, vbc->comp, g->dim, values, "grad_sub_f64"));
    CHECK(make_vec64(g, vbc, values, v, &dv));
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, &pf));
    if (!p) { phi_set_error("grad_sub_f64: p is NULL"); return PHI_ERR_INVALID; }
    for (int c = 0; c < 3; ++c) out.p[c] = c < g->dim ? v[c] : nullptr;
    return cuda_fail(phi_launch_grad_sub(dgrid64(dg, values), dv, out, field64(pf, kZero3, kZero3, g->dim), p, (cudaStream_t)stream),
                     "grad_sub_f64");
}

int phicuda_advect_centered_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* vvalues, const double* const vel[3],
                                const PhiBC* fbc, const PhiValues64* fvalues, const double* src, double* dst, double dt, void* stream)
{
    DGrid dg; DVecT<double> dv; DField ff;
    CHECK(phi_make_dgrid(g, &dg));
    if (!vbc) { phi_set_error("advect_centered_f64: boundary is NULL"); return PHI_ERR_INVALID; }
    CHECK(check_values64(g, vbc->comp, g->dim, vvalues, "advect_centered_f64"));
    CHECK(make_vec64(g, vbc, vvalues, vel, &dv)); CHECK(phi_make_centered(g, fbc, &ff));
    CHECK(check_values64(g, fbc, 1, fvalues, "advect_centered_f64"));
    if (!src || !dst || src == dst) { phi_set_error("advect_centered_f64: src and dst must be distinct non-NULL arrays"); return PHI_ERR_INVALID; }
    return cuda_fail(phi_launch_advect(dgrid64(dg, vvalues), dv, field64(ff, fvalues->clo[0], fvalues->chi[0], g->dim), -1, src, dst, dt,
                                       (cudaStream_t)stream), "advect_centered_f64");
}

int phicuda_advect_staggered_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* vvalues, const double* const vel[3],
                                 const PhiVBC* fbc, const PhiValues64* fvalues, const double* const src[3], double* const dst[3],
                                 double dt, void* stream)
{
    DGrid dg; DVecT<double> dv, df;
    CHECK(phi_make_dgrid(g, &dg));
    if (!vbc || !fbc || !dst) { phi_set_error("advect_staggered_f64: NULL argument"); return PHI_ERR_INVALID; }
    CHECK(check_values64(g, vbc->comp, g->dim, vvalues, "advect_staggered_f64"));
    CHECK(check_values64(g, fbc->comp, g->dim, fvalues, "advect_staggered_f64"));
    CHECK(make_vec64(g, vbc, vvalues, vel, &dv)); CHECK(make_vec64(g, fbc, fvalues, src, &df));
    for (int c = 0; c < g->dim; ++c) {
        if (!dst[c]) { phi_set_error("advect_staggered_f64: dst[%d] is NULL", c); return PHI_ERR_INVALID; }
        for (int k = 0; k < g->dim; ++k) if (dst[c] == src[k] || dst[c] == vel[k]) { phi_set_error("advect_staggered_f64: dst must not alias src or vel"); return PHI_ERR_INVALID; }
    }
    const DGridT<double> dg64 = dgrid64(dg, vvalues);
    for (int c = 0; c < g->dim; ++c)
        CHECK(cuda_fail(phi_launch_advect(dg64, dv, df.f[c], c, src[c], dst[c], dt, (cudaStream_t)stream), "advect_staggered_f64"));
    return 0;
}

size_t phicuda_cg_workspace_bytes_f64(const PhiGrid* g)
{
    DGrid dg;
    if (phi_make_dgrid(g, &dg)) return 0;
    const PhiValues64 unit = {{1.0, 1.0, 1.0}, {}, {}};          // the size depends on the extents and the batch only
    return phi_cg_workspace_bytes_f64(dgrid64(dg, &unit));
}

int phicuda_cg_poisson_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* values, const double* rhs, double* x,
                           const PhiCgParams64* prm, PhiCgResult64* result, void* workspace, size_t workspace_bytes, void* stream)
{
    CgLaunch64 l;
    CHECK(cg_setup64(g, vbc, values, rhs, x, prm, result, workspace, workspace_bytes, &l));
    return cuda_fail(phi_launch_cg(l, (cudaStream_t)stream), "cg_f64");
}

int phicuda_make_incompressible_f64(const PhiGrid* g, const PhiVBC* vbc, const PhiValues64* values, double* const v[3], double* p,
                                    double* div, const PhiCgParams64* prm, PhiCgResult64* result, void* workspace,
                                    size_t workspace_bytes, void* stream)
{
    // every check of the projection and its solve runs before the first CUDA call
    CgLaunch64 l; DGrid dg; DVecT<double> dv; DVecOutT<double> out; DField cf, pf; PhiBC none, pbc; memset(&none, 0, sizeof(none));
    CHECK(cg_setup64(g, vbc, values, div, p, prm, result, workspace, workspace_bytes, &l));
    CHECK(phi_make_dgrid(g, &dg));
    CHECK(make_vec64(g, vbc, values, v, &dv)); CHECK(phi_make_centered(g, &none, &cf));
    CHECK(phi_pressure_bc(vbc, g->dim, &pbc)); CHECK(phi_make_centered(g, &pbc, &pf));
    if (div == p) { phi_set_error("make_incompressible_f64: div and p must be distinct arrays"); return PHI_ERR_INVALID; }
    for (int c = 0; c < g->dim; ++c) {                // divergence reads v while it writes div, grad_sub writes v while it reads p
        if (v[c] == div || v[c] == p) { phi_set_error("make_incompressible_f64: div and p must not alias v[%d]", c); return PHI_ERR_INVALID; }
        for (int k = 0; k < c; ++k) if (v[k] == v[c]) { phi_set_error("make_incompressible_f64: v[%d] and v[%d] are the same array", k, c); return PHI_ERR_INVALID; }
    }
    for (int c = 0; c < 3; ++c) out.p[c] = c < g->dim ? v[c] : nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    CHECK(cuda_fail(phi_launch_divergence(l.g, dv, field64(cf, kZero3, kZero3, g->dim), div, st), "make_incompressible_f64 divergence"));
    CHECK(cuda_fail(phi_launch_cg(l, st), "make_incompressible_f64 cg"));
    return cuda_fail(phi_launch_grad_sub(l.g, dv, out, l.pf, p, st), "make_incompressible_f64 grad_sub");
}

}  // extern "C"
