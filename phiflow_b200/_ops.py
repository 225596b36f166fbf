"""
Array-level host API over the C ABI: device layout, conversions from/to the reference's array layout, and one Python
function per exported entry point.  torch is used for device memory and streams only.

Boundary specs use the same plain encoding as the reference-side tests: a tuple over axes (x, y[, z]) of
(lower, upper) sides, each 'periodic', 'zg' (ZERO_GRADIENT == BOUNDARY) or a float constant.
"""
import ctypes as C
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import PhiGrid, PhiBC, PhiVBC, PhiCgParams, PhiCgResult, PhiPlumeParams, F3

PERIODIC, ZG, HALO = 'periodic', 'zg', 'halo'
_RESULT_DTYPE = np.dtype([('iterations', np.int32), ('converged', np.int32), ('diverged', np.int32),
                          ('residual_sq', np.float32), ('tol_sq', np.float32), ('initial_residual_sq', np.float32)])


def _kind(side):
    if side == PERIODIC:
        return _lib.BC_PERIODIC
    if side == ZG:
        return _lib.BC_ZERO_GRADIENT
    if side == HALO:
        return _lib.BC_HALO
    return _lib.BC_CONST


def make_bc(spec) -> PhiBC:
    bc = PhiBC()
    for a, (lo, hi) in enumerate(spec):
        bc.lo[a], bc.hi[a] = _kind(lo), _kind(hi)
        bc.clo[a] = float(lo) if not isinstance(lo, str) else 0.0
        bc.chi[a] = float(hi) if not isinstance(hi, str) else 0.0
    return bc


def make_vbc(spec, dim) -> PhiVBC:
    """spec: one boundary spec for all components, or a list of `dim` specs (per-component constants)."""
    per_comp = spec if isinstance(spec, list) else [spec] * dim
    vbc = PhiVBC()
    for c in range(dim):
        vbc.comp[c] = make_bc(per_comp[c])
    return vbc


def stored_faces(vspec, axis):
    """(lower stored, upper stored) - PhiML/phiml/math/extrapolation.py:57-62."""
    spec = vspec[0] if isinstance(vspec, list) else vspec
    lo, hi = spec[axis]
    return (lo == ZG or lo == PERIODIC or lo == HALO), (hi == ZG)


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("phiflow_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback.")


def _ptr(t: Optional[torch.Tensor], off: int = 0):
    """Device address of the first OWNED plane (off = byte offset of the lower halo planes, 0 on a single GPU)."""
    return C.c_void_p(t.data_ptr() + off) if t is not None else C.c_void_p(0)


def _f3(ts: Sequence[torch.Tensor], off: int = 0):
    arr = F3()
    for i in range(3):
        arr[i] = ts[i].data_ptr() + off if i < len(ts) else None
    return arr


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Domain:
    """Resolution, cell size, batch size and the allocation extents of centred / staggered arrays (include/phicuda.h)."""

    def __init__(self, resolution: Sequence[int], dx: Sequence[float], batch: int = 1, vbc=None, device='cuda', halo: int = 0):
        self.dim = len(resolution)
        assert self.dim in (2, 3), "only 2-D and 3-D grids"
        self.res = tuple(int(r) for r in resolution)
        self.dx = tuple(float(d) for d in dx)
        self.batch = int(batch)
        self.device = torch.device(device)
        self.upper = tuple(stored_faces(vbc, a)[1] if vbc is not None else False for a in range(self.dim))
        r4 = lambda v: (v + 3) // 4 * 4
        self.halo = int(halo)                 # z-slab halo planes on each side (multi-GPU); `resolution` is the OWNED slab
        assert self.halo == 0 or self.dim == 3
        pad = lambda a: 2 * self.halo if a == 2 else 0
        self.cext = (r4(self.res[0]),) + tuple(self.res[a] + pad(a) for a in range(1, self.dim))
        self.fext = (r4(self.res[0] + int(self.upper[0])),) + tuple(self.res[a] + int(self.upper[a]) + pad(a) for a in range(1, self.dim))
        self.coff = 4 * self.halo * self.cext[0] * self.cext[1]       # byte offset of the first owned plane
        self.foff = 4 * self.halo * self.fext[0] * self.fext[1]
        g = PhiGrid()
        g.dim, g.batch = self.dim, self.batch
        for a in range(3):
            g.n[a] = self.res[a] if a < self.dim else 1
            g.cext[a] = self.cext[a] if a < self.dim else 1
            g.fext[a] = self.fext[a] if a < self.dim else 1
            g.dx[a] = self.dx[a] if a < self.dim else 1.0
        g.halo = self.halo
        self.grid = g
        self._ws = None
        self._result = None
        self._scratch = None

    # ---- allocation ---------------------------------------------------------------------------------------------
    def _shape(self, ext):
        return (self.batch,) + tuple(reversed(ext))

    def alloc_centered(self) -> torch.Tensor:
        return torch.zeros(self._shape(self.cext), dtype=torch.float32, device=self.device)

    def alloc_faces(self) -> List[torch.Tensor]:
        return [torch.zeros(self._shape(self.fext), dtype=torch.float32, device=self.device) for _ in range(self.dim)]

    def workspace(self):
        if self._ws is None:
            n = _lib.load().phicuda_cg_workspace_bytes(C.byref(self.grid))
            self._ws = torch.zeros(n, dtype=torch.uint8, device=self.device)
        return self._ws, self.results()

    def results(self):
        """Device buffer of one PhiCgResult per batch entry (what read_results returns)."""
        if self._result is None:
            self._result = torch.zeros(self.batch * 6, dtype=torch.int32, device=self.device)
        return self._result

    def scratch(self):
        if self._scratch is None:
            n = _lib.load().phicuda_plume_scratch_bytes(C.byref(self.grid))
            self._scratch = torch.zeros(n // 4, dtype=torch.float32, device=self.device)
        return self._scratch

    # ---- conversions: reference layout (x, y[, z]) <-> device layout (b, [z,] y, x) ------------------------------------
    def _to_dev(self, a: np.ndarray, ext, offset_axis=None, offset=0) -> torch.Tensor:
        a = np.asarray(a, dtype=np.float32)
        if a.ndim == self.dim:
            a = a[None]
        assert a.ndim == self.dim + 1 and a.shape[0] in (1, self.batch), f"bad array shape {a.shape}"
        if a.shape[0] != self.batch:
            a = np.broadcast_to(a, (self.batch,) + a.shape[1:])
        t = torch.zeros(self._shape(ext), dtype=torch.float32, device=self.device)
        src = torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0,) + tuple(range(self.dim, 0, -1)))))
        idx = [slice(None)]
        for ax in range(self.dim - 1, -1, -1):               # device axis order: z, y, x
            start = (offset if ax == offset_axis else 0) + (self.halo if ax == 2 else 0)
            idx.append(slice(start, start + a.shape[1 + ax]))
        t[tuple(idx)] = src.to(self.device)
        return t

    def _to_host(self, t: torch.Tensor, shape, offset_axis=None, offset=0) -> np.ndarray:
        idx = [slice(None)]
        for ax in range(self.dim - 1, -1, -1):
            start = (offset if ax == offset_axis else 0) + (self.halo if ax == 2 else 0)
            idx.append(slice(start, start + shape[ax]))
        a = t[tuple(idx)].cpu().numpy()
        return np.ascontiguousarray(np.transpose(a, (0,) + tuple(range(self.dim, 0, -1))))

    def centered_from_numpy(self, a) -> torch.Tensor:
        return self._to_dev(a, self.cext)

    def centered_to_numpy(self, t, squeeze=True) -> np.ndarray:
        a = self._to_host(t, self.res)
        return a[0] if (squeeze and self.batch == 1) else a

    def face_shapes(self, vspec):
        shapes, offsets = [], []
        for c in range(self.dim):
            lo, hi = stored_faces(vspec, c)
            s = list(self.res); s[c] = self.res[c] - 1 + int(lo) + int(hi)
            shapes.append(tuple(s)); offsets.append(0 if lo else 1)
        return shapes, offsets

    def faces_from_numpy(self, comps, vspec) -> List[torch.Tensor]:
        shapes, offsets = self.face_shapes(vspec)
        out = []
        for c in range(self.dim):
            a = np.asarray(comps[c], dtype=np.float32)
            assert tuple(a.shape[-self.dim:]) == shapes[c], f"component {c}: shape {a.shape} != stored faces {shapes[c]}"
            out.append(self._to_dev(a, self.fext, c, offsets[c]))
        return out

    def faces_to_numpy(self, ts, vspec, squeeze=True):
        shapes, offsets = self.face_shapes(vspec)
        out = []
        for c in range(self.dim):
            a = self._to_host(ts[c], shapes[c], c, offsets[c])
            out.append(a[0] if (squeeze and self.batch == 1) else a)
        return out


# ---- one function per exported entry point ---------------------------------------------------------------------------------

def laplace(dom: Domain, bc, x: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
    """field.laplace order 2 (phi/field/_field_math.py:118-145)."""
    require_cuda()
    out = dom.alloc_centered() if out is None else out
    _lib.check(_lib.load().phicuda_laplace_f32(C.byref(dom.grid), C.byref(make_bc(bc)), _ptr(x, dom.coff), _ptr(out, dom.coff), _stream()))
    return out


def laplace_axpy(dom: Domain, bc, x, coeff: float, out=None):
    """x + coeff * laplace(x): one explicit diffusion sub-step (phi/physics/diffuse.py:13-60)."""
    require_cuda()
    out = dom.alloc_centered() if out is None else out
    _lib.check(_lib.load().phicuda_laplace_axpy_f32(C.byref(dom.grid), C.byref(make_bc(bc)), _ptr(x, dom.coff), C.c_float(coeff), _ptr(out, dom.coff), _stream()))
    return out


def laplace_axpy_faces(dom: Domain, vbc, v: List[torch.Tensor], coeff: float, substeps: int = 1) -> List[torch.Tensor]:
    """diffuse.explicit of a STAGGERED field (phi/physics/diffuse.py:13-60 -> phi/field/_field_math.py:118-145 with `fields = [u]`:
    `math.laplace` of the non-uniform component stack pads every component by one layer of ITS boundary, so component c is an
    independent array of its stored faces with the boundary spec of component c - verified against the vendored PhiML in
    tests/test_staggered_diffusion.py).  Not on the north-star path (row N3): composed on the host from the laplace kernel - each
    component is copied into a centred array of a domain whose resolution is the component's face count (the x component of a
    walled grid starts at face 1, i.e. 4 bytes off the 16-byte alignment the TMA ring needs), `substeps` x laplace_axpy, copied back."""
    require_cuda()
    assert dom.halo == 0, "staggered diffusion is not offered on z-slabs"
    shapes, offsets = dom.face_shapes(vbc)
    out = []
    for c in range(dom.dim):
        sub = Domain(shapes[c], dom.dx, dom.batch, device=dom.device)
        spec = vbc[c] if isinstance(vbc, list) else vbc
        src = (slice(None),) + tuple(slice(offsets[c] if a == c else 0, (offsets[c] if a == c else 0) + shapes[c][a]) for a in range(dom.dim - 1, -1, -1))
        dst = (slice(None),) + tuple(slice(0, shapes[c][a]) for a in range(dom.dim - 1, -1, -1))
        a, b = sub.alloc_centered(), sub.alloc_centered()
        a[dst] = v[c][src]
        for _ in range(substeps):
            laplace_axpy(sub, spec, a, coeff, out=b)
            a, b = b, a
        res = v[c].clone()
        res[src] = a[dst]
        out.append(res)
    return out


def divergence(dom: Domain, vbc, v: List[torch.Tensor], out=None, accessible=None):
    """field.divergence of a staggered grid (phi/field/_field_math.py:617-626); accessible: div *= active mask (fluid.py:138-141)."""
    require_cuda()
    out = dom.alloc_centered() if out is None else out
    if accessible is not None:
        _lib.check(_lib.load().phicuda_divergence_masked_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(v, dom.foff),
                                                            _ptr(accessible, dom.coff), _ptr(out, dom.coff), _stream()))
        return out
    _lib.check(_lib.load().phicuda_divergence_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(v, dom.foff), _ptr(out, dom.coff), _stream()))
    return out


def grad_sub(dom: Domain, vbc, v: List[torch.Tensor], p: torch.Tensor, accessible=None):
    """v -= spatial_gradient(p, at='face') in place (phi/physics/fluid.py:158-161); accessible: gradient *= hard_bcs (:159-160)."""
    require_cuda()
    if accessible is not None:
        _lib.check(_lib.load().phicuda_grad_sub_masked_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(v, dom.foff), _ptr(p, dom.coff),
                                                          _ptr(accessible, dom.coff), _stream()))
        return v
    _lib.check(_lib.load().phicuda_grad_sub_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(v, dom.foff), _ptr(p, dom.coff), _stream()))
    return v


def advect_centered(dom: Domain, vbc, vel, fbc, src, dt: float, out=None):
    """advect.semi_lagrangian of a centred field (phi/physics/advect.py:156-179)."""
    require_cuda()
    out = dom.alloc_centered() if out is None else out
    _lib.check(_lib.load().phicuda_advect_centered_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(vel, dom.foff),
                                                       C.byref(make_bc(fbc)), _ptr(src, dom.coff), _ptr(out, dom.coff), C.c_float(dt), _stream()))
    return out


def advect_staggered(dom: Domain, vbc, vel, fbc, src, dt: float, out=None):
    """advect.semi_lagrangian of a staggered field (self-advection when src is vel)."""
    require_cuda()
    out = dom.alloc_faces() if out is None else out
    _lib.check(_lib.load().phicuda_advect_staggered_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(vel, dom.foff),
                                                        C.byref(make_vbc(fbc, dom.dim)), _f3(src, dom.foff), _f3(out, dom.foff), C.c_float(dt), _stream()))
    return out


def grid_sample(dom: Domain, bc, grid: torch.Tensor, coords: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
    """math.grid_sample (PhiML/phiml/math/_ops.py:936-1015): grid = centred array in device layout, coords = float32 tensor
    (batch, npoints, dim) of index-space positions (x first, 0 = first cell centre).  Returns (batch, npoints)."""
    require_cuda()
    assert coords.dtype == torch.float32 and coords.is_contiguous() and coords.shape[0] == dom.batch and coords.shape[-1] == dom.dim
    npoints = coords.shape[1]
    out = torch.empty((dom.batch, npoints), dtype=torch.float32, device=dom.device) if out is None else out
    _lib.check(_lib.load().phicuda_grid_sample_f32(C.byref(dom.grid), C.byref(make_bc(bc)), _ptr(grid, dom.coff), _ptr(coords),
                                                   C.c_int64(npoints), _ptr(out), _stream()))
    return out


def mac_cormack_centered(dom: Domain, vbc, vel, fbc, src, dt: float, correction_strength=1.0, out=None):
    """advect.mac_cormack of a centred field (phi/physics/advect.py:182-215)."""
    require_cuda()
    out = dom.alloc_centered() if out is None else out
    tmp = dom.alloc_centered()
    _lib.check(_lib.load().phicuda_mac_cormack_centered_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(vel, dom.foff),
                                                            C.byref(make_bc(fbc)), _ptr(src, dom.coff), _ptr(out, dom.coff), _ptr(tmp, dom.coff),
                                                            C.c_float(dt), C.c_float(correction_strength), _stream()))
    return out


def axpy_centered(dom: Domain, a: float, x, y):
    require_cuda()
    _lib.check(_lib.load().phicuda_axpy_centered_f32(C.byref(dom.grid), C.c_float(a), _ptr(x, dom.coff), _ptr(y, dom.coff), _stream()))
    return y


def add_buoyancy(dom: Domain, vbc, sbc, s, factor: Sequence[float], dt: float, v):
    """v += dt * resample(s * factor, to=v) in place (phi/field/_resample.py:272-276).  The product keeps the boundary of s
    (phi/field/_field.py:809): faces next to a constant side c of s average c itself, unscaled, also where factor is 0."""
    require_cuda()
    b = (C.c_float * 3)(*[float(factor[i]) if i < len(factor) else 0.0 for i in range(3)])
    _lib.check(_lib.load().phicuda_add_buoyancy_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), C.byref(make_bc(sbc)),
                                                    _ptr(s, dom.coff), b, C.c_float(dt), _f3(v, dom.foff), _stream()))
    return v


def max_abs_velocity(dom: Domain, vbc, v, out: torch.Tensor = None) -> torch.Tensor:
    """Device tensor of 3 floats: max |v_c| per component over the stored faces of the owned planes (CFL number of the
    unbounded semi-Lagrangian back-trace, phi/physics/advect.py:20-24)."""
    require_cuda()
    out = torch.zeros(3, dtype=torch.float32, device=dom.device) if out is None else out
    _lib.check(_lib.load().phicuda_max_abs_velocity_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(v, dom.foff), _ptr(out), _stream()))
    return out


def last_launch_info() -> dict:
    """Which kernel variant this thread's most recent laplace / CG launch selected (include/phicuda.h PhiLaunchInfo)."""
    info = _lib.PhiLaunchInfo()
    _lib.check(_lib.load().phicuda_last_launch_info(C.byref(info)))
    out = {k: int(getattr(info, k)) for k, _ in _lib.PhiLaunchInfo._fields_}
    out['passes'] = int(_lib.load().phicuda_last_cg_passes())      # sweeps per CG iteration of the last CG launch
    return out


CG_OPERATORS = {0: None, 1: 'poisson', 2: 'helmholtz', 3: 'helmholtz_varying'}       # include/phicuda.h PHI_CG_OP_*


def last_cg_operator():
    """Operator of this thread's most recent CG launch: 'poisson', 'helmholtz' (diffuse_implicit), 'helmholtz_varying'
    (diffuse_implicit_varying), or None before the first one."""
    return CG_OPERATORS[int(_lib.load().phicuda_last_cg_operator())]


def _is_flexible(vspec) -> bool:
    spec = vspec[0] if isinstance(vspec, list) else vspec
    return any(side == ZG for ax in spec for side in ax)


def cg_params(vbc, rtol=1e-5, atol=1e-5, max_iter=1000, matrix_offset=0.0, balance=None, method='CG') -> PhiCgParams:
    """Solver parameters with the defaults of fluid.make_incompressible (phi/physics/fluid.py:145-148):
    non-flexible velocity boundaries (closed / periodic) -> balanced right-hand side and rank deficiency 1."""
    rank_def = not _is_flexible(vbc)
    prm = PhiCgParams()
    prm.rtol, prm.atol, prm.max_iter = rtol, atol, int(max_iter)
    prm.balance_rhs = int(rank_def if balance is None else balance)
    prm.project_mean = int(rank_def)
    prm.matrix_offset = float(matrix_offset) if rank_def else 0.0
    prm.method = {'CG': 0, 'CG-adaptive': 1}[method]
    return prm


def read_results(dom: Domain, components: int = 1) -> np.ndarray:
    """Synchronises and returns the per-batch solve results as a structured array.  components = C > 1: the records of the last
    diffuse_implicit of C components on `dom`, one per (batch entry, component), entry b * C + c."""
    d = dom if components == 1 else dom._stacked[components]
    return d.results().cpu().numpy().view(_RESULT_DTYPE)


def cg_poisson(dom: Domain, vbc, rhs, x0=None, prm: PhiCgParams = None):
    """Pressure solve: CG on the matrix-free Poisson operator (phi/physics/fluid.py:156). Returns x (x0 updated in place)."""
    require_cuda()
    ws, res = dom.workspace()
    x = dom.alloc_centered() if x0 is None else x0
    prm = prm or cg_params(vbc)
    _lib.check(_lib.load().phicuda_cg_poisson_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _ptr(rhs, dom.coff), _ptr(x, dom.coff), C.byref(prm),
                                                  _ptr(res), _ptr(ws), C.c_size_t(ws.numel()), _stream()))
    return x


def diffuse_implicit(dom: Domain, spec, u, amount: float, rtol=1e-5, atol=1e-5, max_iter=1000, x0=None):
    """diffuse.implicit (phi/physics/diffuse.py:63-95): solves x - amount * laplace(x) = u with CG, amount = diffusivity * dt.
    u: a centred array with boundary spec `spec`, or a list of C <= 3 same-shaped component arrays (a vector CenteredGrid, or the
    components of a periodic StaggeredGrid) with one spec or a list of per-component specs.  Every component of every batch entry is
    its own system, as in the reference (its tracer keeps the uncoupled vector dim out of the matrix).  x0: start value of the same
    form, default u (diffuse.py:93-94).  Returns new arrays in the form of u; the inputs are not modified.
    read_results(dom, components=C) then holds one record per system, entry b * C + c = component c of batch entry b."""
    require_cuda()
    comps = list(u) if isinstance(u, (list, tuple)) else [u]
    n = len(comps)
    assert 1 <= n <= 3 and all(c.shape == comps[0].shape for c in comps), "1 to 3 components of the same shape"
    assert dom.halo == 0, "implicit diffusion is not offered on z-slabs"
    if n == 1:
        sdom, y = dom, comps[0]
    else:                                   # entry s * n + c = component c of system s
        cache = dom.__dict__.setdefault('_stacked', {})
        if n not in cache:
            cache[n] = Domain(dom.res, dom.dx, dom.batch * n, device=dom.device)
        sdom = cache[n]
        y = torch.stack(comps, 1).reshape((dom.batch * n,) + tuple(comps[0].shape[1:]))
    if x0 is None:
        x = y.clone()
    else:
        x0s = list(x0) if isinstance(x0, (list, tuple)) else [x0]
        x = x0s[0].clone() if n == 1 else torch.stack(x0s, 1).reshape(y.shape)
    ws, _ = sdom.workspace()
    prm = PhiCgParams()                     # plain CG; I - amount * L is not singular: no balancing, projection or offset
    prm.rtol, prm.atol, prm.max_iter = rtol, atol, int(max_iter)
    _lib.check(_lib.load().phicuda_diffuse_implicit_f32(C.byref(sdom.grid), C.byref(make_vbc(spec, n)), C.c_int32(n), C.c_float(amount),
                                                        _ptr(y), _ptr(x), C.byref(prm), _ptr(sdom.results()), _ptr(ws), C.c_size_t(ws.numel()),
                                                        _stream()))
    if n == 1:
        return x if not isinstance(u, (list, tuple)) else [x]
    x = x.reshape((dom.batch, n) + tuple(comps[0].shape[1:]))
    return [x[:, c].clone() for c in range(n)]


def diffuse_implicit_varying(dom: Domain, spec, u, k, dt: float, rtol=1e-5, atol=1e-5, max_iter=1000, x0=None):
    """diffuse.implicit(u, k, dt) with a spatially varying diffusivity (phi/physics/diffuse.py:90-95, 129-141): solves
    sharpen(x) = explicit(x, k, -dt) = u with CG.  Every face takes min(-dt k_lo, -dt k_hi), whose ghosts follow u's boundary `spec`
    (a constant side with value c gives min(-dt k_edge, c)); for dt > 0 that is the face MAXIMUM of k.
    u: centred array of `dom`; k: centred array with 1 (shared by every entry) or dom.batch entries.  x0: start value, default u.
    Returns a new array; the inputs are not modified.  read_results(dom) then holds one record per batch entry."""
    require_cuda()
    assert dom.halo == 0, "implicit diffusion is not offered on z-slabs"
    assert tuple(u.shape) == dom._shape(dom.cext), f"u: shape {tuple(u.shape)} is not a centred array of the domain"
    assert k.dtype == torch.float32 and k.is_contiguous() and tuple(k.shape[1:]) == tuple(u.shape[1:]) and k.shape[0] in (1, dom.batch), \
        f"k: shape {tuple(k.shape)} is not a centred array of the domain with 1 or {dom.batch} entries"
    x = (u if x0 is None else x0).clone()
    ws, _ = dom.workspace()
    prm = PhiCgParams()                     # plain CG; I + D0 is not singular: no balancing, projection or offset
    prm.rtol, prm.atol, prm.max_iter = rtol, atol, int(max_iter)
    _lib.check(_lib.load().phicuda_diffuse_implicit_varying_f32(C.byref(dom.grid), C.byref(make_bc(spec)), _ptr(k), C.c_int32(k.shape[0]),
                                                                C.c_float(dt), _ptr(u), _ptr(x), C.byref(prm), _ptr(dom.results()), _ptr(ws),
                                                                C.c_size_t(ws.numel()), _stream()))
    return x


def _cached_scratch(dom: Domain, attr: str, nbytes: int) -> torch.Tensor:
    """A float32 scratch tensor of at least nbytes bytes, cached on dom as `attr` and replaced by a larger one when a call needs more.
    Each caller keeps its own attribute: calls of different functions may run on different streams."""
    s = getattr(dom, attr, None)
    if s is None or 4 * s.numel() < nbytes:
        s = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=dom.device)
        setattr(dom, attr, s)
    return s


def reaction_diffusion(dom: Domain, spec, u, v, du: float, dv: float, f: float, k: float, dt: float, substeps: int = 1):
    """`substeps` Gray-Scott substeps of the Reaction_Diffusion notebook in one launch (include/phicuda.h, N7):
    uvv = u * v**2, u += dt * (du * laplace(u) - uvv + f * (1 - u)), v += dt * (dv * laplace(v) + uvv - (f + k) * v).
    u, v: centred arrays of `dom`; spec: one boundary spec for both, or [spec_u, spec_v] (same kinds, constants 0).
    Returns new arrays (u', v'); the inputs are not modified and may be the same tensor."""
    require_cuda()
    assert dom.halo == 0, "reaction-diffusion is not offered on z-slabs"
    shape = dom._shape(dom.cext)
    assert tuple(u.shape) == shape and tuple(v.shape) == shape, f"u, v: shapes {tuple(u.shape)}, {tuple(v.shape)} are not centred arrays of the domain"
    un, vn = u.clone(), v.clone()
    s = _cached_scratch(dom, '_rd_scratch', _lib.load().phicuda_reaction_diffusion_scratch_bytes(C.byref(dom.grid)))
    _lib.check(_lib.load().phicuda_reaction_diffusion_f32(C.byref(dom.grid), C.byref(make_vbc(spec, 2)), _ptr(un), _ptr(vn), C.c_float(du),
                                                          C.c_float(dv), C.c_float(f), C.c_float(k), C.c_float(dt), C.c_int32(substeps),
                                                          _ptr(s), C.c_size_t(4 * s.numel()), _stream()))
    return un, vn


def wave(dom: Domain, spec, h_c, h_p, dd: float, k_speed: float, k_damp: float, discs, radius_sq: float, centers, substeps: int = 1):
    """`substeps` steps of the Waves notebook's wave equation in one launch (include/phicuda.h, N8): per substep s the disc s is
    stamped on both states, then h_n = 2 h_c - h_p + dd (k_speed laplace(h_c) - k_damp (h_c - h_p)) and (h_c, h_p) = (h_n, h_c).
    discs: `substeps` entries (center, value), or None for a substep without a disc; radius_sq: float32 r^2; centers: per-axis cell
    centres (x, then y[, z]) as float32.  Returns new arrays (h_c', h_p'); the inputs are not modified and may be the same tensor."""
    require_cuda()
    assert dom.halo == 0, "the wave step is not offered on z-slabs"
    shape = dom._shape(dom.cext)
    assert tuple(h_c.shape) == shape and tuple(h_p.shape) == shape, f"h_c, h_p: shapes {tuple(h_c.shape)}, {tuple(h_p.shape)} are not centred arrays of the domain"
    assert len(discs) == substeps, f"{len(discs)} discs for {substeps} substeps"
    table = (_lib.PhiWaveDisc * max(substeps, 1))()
    for d, entry in zip(table, discs):
        if entry is not None:
            center, value = entry
            for a, c in enumerate(center):
                d.center[a] = float(c)
            d.value, d.present = float(value), 1
    coords = np.ascontiguousarray(centers, dtype=np.float32)
    assert coords.size == sum(dom.res), f"{coords.size} cell centres for resolution {dom.res}"
    hc, hp = h_c.clone(), h_p.clone()
    lib = _lib.load()
    scratch = _cached_scratch(dom, '_wave_scratch', lib.phicuda_wave_scratch_bytes(C.byref(dom.grid), substeps))
    _lib.check(lib.phicuda_wave_f32(C.byref(dom.grid), C.byref(make_bc(spec)), _ptr(hc), _ptr(hp), C.c_float(dd), C.c_float(k_speed),
                                    C.c_float(k_damp), table, C.c_float(radius_sq), coords.ctypes.data_as(C.POINTER(C.c_float)),
                                    C.c_int32(substeps), _ptr(scratch), C.c_size_t(4 * scratch.numel()), _stream()))
    return hc, hp


def mul_faces(dom: Domain, vbc, v, mask):
    """v_c *= mask_c on the stored faces (apply_boundary_conditions for stationary obstacles, fluid.py:212-240)."""
    require_cuda()
    _lib.check(_lib.load().phicuda_mul_faces_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(v, dom.foff), _f3(mask, dom.foff), _stream()))
    return v


def make_incompressible(dom: Domain, vbc, v, p=None, prm: PhiCgParams = None, accessible=None):
    """fluid.make_incompressible on raw arrays: v and p are updated in place.  accessible: centred obstacle mask (N4)."""
    require_cuda()
    ws, res = dom.workspace()
    p = dom.alloc_centered() if p is None else p
    div = dom.alloc_centered()
    prm = prm or cg_params(vbc)
    if accessible is not None:
        _lib.check(_lib.load().phicuda_make_incompressible_masked_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(v, dom.foff),
                                                                      _ptr(p, dom.coff), _ptr(div, dom.coff), _ptr(accessible, dom.coff),
                                                                      C.byref(prm), _ptr(res), _ptr(ws), C.c_size_t(ws.numel()), _stream()))
        return v, p
    _lib.check(_lib.load().phicuda_make_incompressible_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(v, dom.foff), _ptr(p, dom.coff), _ptr(div, dom.coff),
                                                           C.byref(prm), _ptr(res), _ptr(ws), C.c_size_t(ws.numel()), _stream()))
    return v, p


def _collocated_workspace(dom: Domain):
    if getattr(dom, '_co_ws', None) is None:
        n = _lib.load().phicuda_collocated_workspace_bytes(C.byref(dom.grid))
        dom._co_ws = torch.zeros(n, dtype=torch.uint8, device=dom.device)
    return dom._co_ws


def wide_laplace(dom: Domain, vbc, x: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
    """fluid.masked_laplace(wide_stencil=True) without obstacles (phi/physics/fluid.py:197-202): centred divergence of the centred
    gradient, the pressure operator of CenteredGrid velocities."""
    require_cuda()
    out = dom.alloc_centered() if out is None else out
    ws = _collocated_workspace(dom)
    _lib.check(_lib.load().phicuda_wide_laplace_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _ptr(x), _ptr(out), _ptr(ws),
                                                    C.c_size_t(ws.numel()), _stream()))
    return out


def estimate_matrix_offset(dom: Domain, vbc, seed: int = 0) -> float:
    """The rank-1 offset the reference adds to rank-deficient systems (PhiML/phiml/math/_optimize.py:705-714):
    sqrt(mean|A x| * 9 / N) for a uniform random x - here with the wide-stencil operator."""
    g = torch.Generator(device='cpu').manual_seed(seed)
    x = dom.alloc_centered()
    idx = (slice(None),) + tuple(slice(0, dom.res[a]) for a in range(dom.dim - 1, -1, -1))
    x[idx] = torch.rand((dom.batch,) + tuple(reversed(dom.res)), generator=g).to(dom.device)
    y = wide_laplace(dom, vbc, x)
    n = float(np.prod(dom.res))
    return float(torch.sqrt(y[idx].abs().mean() * 9.0 / n).item())


def make_incompressible_centered(dom: Domain, vbc, v: List[torch.Tensor], p: torch.Tensor = None, rtol=1e-5, atol=1e-5, max_iter=1000,
                                 matrix_offset=None):
    """fluid.make_incompressible for a CenteredGrid velocity (wide stencil, phi/physics/fluid.py:138-161 with :154-155): v = `dim`
    CENTRED arrays, updated in place; returns (v, p).  Solver: CG-adaptive, what the reference's default Solve() runs.
    Synchronises the stream (the iteration loop polls the stopping flags from the host)."""
    require_cuda()
    res = dom.results()
    ws = _collocated_workspace(dom)
    p = dom.alloc_centered() if p is None else p
    prm = cg_params(vbc, rtol=rtol, atol=atol, max_iter=max_iter, method='CG-adaptive')
    if prm.project_mean and matrix_offset is None:
        matrix_offset = estimate_matrix_offset(dom, vbc)
    prm.matrix_offset = float(matrix_offset or 0.0) if prm.project_mean else 0.0
    _lib.check(_lib.load().phicuda_make_incompressible_centered_host_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), _f3(v), _ptr(p),
                                                                        C.byref(prm), _ptr(res), _ptr(ws), C.c_size_t(ws.numel()), _stream()))
    return v, p


def plume_step(dom: Domain, vbc, sbc, v, s, p, inflow, dt, inflow_rate, buoyancy, prm: PhiCgParams, mac_cormack=False, cg_events=None,
               static_scalar=False, accessible=None, factors=None):
    """incompressible_step: the notebook step (examples/grids/Smoke_Plume.ipynb:58-68) as one C-ABI call; state updated in place.
    cg_events: optional pair of torch.cuda.Event(enable_timing=True) that the library records around the pressure solve.
    static_scalar: `s` is a stationary forcing field (v* = advect(v) + dt * resample(s * buoyancy, to=v)), not advected smoke.
    accessible, factors: static obstacles (Batched_Smoke, Fluid_Logo) - the centred accessible mask and the per-component face factors
    of apply_boundary_conditions (flow._obstacle_masks), both with the full batch (one obstacle per entry); v* is multiplied by the
    factors and projected with the masked operator (phicuda_plume_step_masked_f32)."""
    require_cuda()
    assert dom.halo == 0, "plume_step is the single-GPU fused call; z-slab runs sequence the step in phiflow_b200.dist"
    assert (accessible is None) == (factors is None), "obstacles need both the accessible mask and the face factors"
    ws, res = dom.workspace()
    sp = PhiPlumeParams()
    sp.dt, sp.inflow_rate, sp.mac_cormack, sp.static_scalar = dt, inflow_rate, int(mac_cormack), int(static_scalar)
    for i in range(3):
        sp.buoyancy[i] = float(buoyancy[i]) if i < len(buoyancy) else 0.0
    if cg_events is not None:
        for ev in cg_events:
            if not ev.cuda_event:                   # torch creates the cudaEvent_t lazily at the first record
                ev.record()
        sp.cg_start_event, sp.cg_stop_event = cg_events[0].cuda_event, cg_events[1].cuda_event
    if accessible is not None:
        _lib.check(_lib.load().phicuda_plume_step_masked_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), C.byref(make_bc(sbc)), _f3(v),
                                                             _ptr(s), _ptr(p), _ptr(inflow), _ptr(accessible), _f3(factors), C.byref(sp),
                                                             C.byref(prm), _ptr(res), _ptr(dom.scratch()), _ptr(ws), C.c_size_t(ws.numel()),
                                                             _stream()))
        return v, s, p
    _lib.check(_lib.load().phicuda_plume_step_f32(C.byref(dom.grid), C.byref(make_vbc(vbc, dom.dim)), C.byref(make_bc(sbc)), _f3(v),
                                                  _ptr(s), _ptr(p), _ptr(inflow), C.byref(sp), C.byref(prm), _ptr(res),
                                                  _ptr(dom.scratch()), _ptr(ws), C.c_size_t(ws.numel()), _stream()))
    return v, s, p


class HostPlume:
    """The reference-facing form of the step: the state (v components, s, p) lives in HOST arrays in the reference's
    (x, y[, z]) order (`Field.numpy()` order, phi/field/_field.py:170-172); every call uploads it from pinned memory,
    transposes to the device layout (DESIGN.md section 2), runs phicuda_plume_step_f32, transposes back and downloads the
    new state.  This is what bench.py times as `e2e`."""

    def __init__(self, dom: Domain, vbc, sbc):
        require_cuda()
        self.dom, self.vbc, self.sbc = dom, vbc, sbc
        shapes, self.offsets = dom.face_shapes(vbc)
        pin = lambda shape: torch.zeros(shape, dtype=torch.float32).pin_memory()
        self.v = [pin(shapes[c]) for c in range(dom.dim)]
        self.s, self.p = pin(dom.res), pin(dom.res)
        self.dv, self.ds, self.dp = dom.alloc_faces(), dom.alloc_centered(), dom.alloc_centered()
        self.bytes_per_direction = 4 * (sum(t.numel() for t in self.v) + self.s.numel() + self.p.numel())
        self._perm = tuple(range(dom.dim - 1, -1, -1))

    def _view(self, t, shape, axis=None, offset=0):
        idx = [0]
        for ax in range(self.dom.dim - 1, -1, -1):
            start = offset if ax == axis else 0
            idx.append(slice(start, start + shape[ax]))
        return t[tuple(idx)]

    def load(self, v_dev, s_dev, p_dev):
        """Seeds the host state from device arrays (set-up, untimed)."""
        shapes, offs = self.dom.face_shapes(self.vbc)
        for c in range(self.dom.dim):
            self.v[c].copy_(self._view(v_dev[c], shapes[c], c, offs[c]).permute(*self._perm))
        self.s.copy_(self._view(s_dev, self.dom.res).permute(*self._perm))
        self.p.copy_(self._view(p_dev, self.dom.res).permute(*self._perm))
        torch.cuda.synchronize()

    def step(self, inflow_dev, dt, inflow_rate, buoyancy, prm, **kw):
        dom, dev = self.dom, self.dom.device
        shapes, offs = dom.face_shapes(self.vbc)
        for c in range(dom.dim):
            self._view(self.dv[c], shapes[c], c, offs[c]).copy_(self.v[c].to(dev, non_blocking=True).permute(*self._perm))
        self._view(self.ds, dom.res).copy_(self.s.to(dev, non_blocking=True).permute(*self._perm))
        self._view(self.dp, dom.res).copy_(self.p.to(dev, non_blocking=True).permute(*self._perm))
        plume_step(dom, self.vbc, self.sbc, self.dv, self.ds, self.dp, inflow_dev, dt, inflow_rate, buoyancy, prm, **kw)
        for c in range(dom.dim):
            self.v[c].copy_(self._view(self.dv[c], shapes[c], c, offs[c]).permute(*self._perm), non_blocking=True)
        self.s.copy_(self._view(self.ds, dom.res).permute(*self._perm), non_blocking=True)
        self.p.copy_(self._view(self.dp, dom.res).permute(*self._perm), non_blocking=True)
