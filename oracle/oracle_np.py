"""
CPU oracle for the incompressible-fluid hot path  --  TEST INFRASTRUCTURE ONLY.

This is a NumPy/SciPy *restatement* of the algorithm the reference (tum-pbs/PhiFlow 3.4.0 with its
NumPy backend, vendored PhiML 1.7.2) executes for
    advect.semi_lagrangian / advect.mac_cormack  ->  field.divergence  ->  CG math.solve_linear over
    the laplace matrix  ->  field.spatial_gradient subtraction     (fluid.make_incompressible).
It is NOT a product path: only tests/, __graft_entry__.smoke() and the cpu_baseline / --impl reference
legs of bench.py may import it.  Nothing in phiflow_b200/ imports it, and phiflow_b200 fails loudly when
its CUDA library is missing instead of falling back to this file.

Parity pinning: every function here is checked (tests/test_oracle_golden.py) against
  * the reference's own known-answer tests (SURVEY.md §4), re-expressed on raw arrays, and
  * golden fixtures tests/golden/*.npz produced by tests/golden/make_golden.py, which imports the vendored
    `phiml.math` and runs the reference's own pad / laplace / spatial_gradient /
    grid_sample / sample_subgrid / jit_compile_linear(...).sparse_matrix / solve_linear on seeded inputs.
  * more shapes and boundary mixes recorded from PhiML 1.7.2 by tests/golden/make_live_golden.py (tests/test_oracle_live_phiml.py,
    tests/test_vector_boundaries.py): pad / laplace / grid_sample / closest_grid_values / the staggered laplace, and cg() against
    phiml.backend.NUMPY.linear_solve - bitwise-equal iterates.
`phi` itself (the Field layer) cannot be imported in the build container (it needs phiml>=1.14, only 1.7.2 is
vendored), so the thin phi.field glue is restated here from the cited lines and pinned by the known-answer tests.

Conventions (all mirror the reference):
  * arrays are float32, axis order (x, y[, z]) exactly as `Field.numpy()` returns them
    (phi/field/_field.py:170-172); no batch axis - callers loop over batch entries, which the reference treats
    as independent systems (PhiML/phiml/backend/_linalg.py:72-87).
  * a boundary condition is a tuple over axes of (lower, upper) sides; each side is 'periodic', 'zg'
    (ZERO_GRADIENT == BOUNDARY) or a float constant (ZERO is 0.0)
    (PhiML/phiml/math/extrapolation.py:247, 544, 648, 1135-1156, combine_sides :1209).
  * a staggered field is a list of per-component arrays whose extent along their own axis is
    n-1 / n / n+1 faces depending on the boundary (tests/commit/field/test__grid.py:25-37).
"""
from __future__ import annotations

import contextlib
import itertools
from typing import List, Sequence, Tuple

import numpy as np
import scipy.sparse as sp

F32 = np.float32
PERIODIC = 'periodic'
ZG = 'zg'          # ZERO_GRADIENT a.k.a. BOUNDARY
ZERO = 0.0


@contextlib.contextmanager
def precision(bits: int):
    """Evaluate the oracle in float64 (bits=64) to obtain an 'exact arithmetic' yardstick for tolerance statements."""
    global F32
    old = F32
    F32 = np.float64 if bits == 64 else np.float32
    try:
        yield
    finally:
        F32 = old


# --------------------------------------------------------------------------------------------------
# boundary-condition helpers
# --------------------------------------------------------------------------------------------------

def uniform_bc(dim: int, side) -> tuple:
    """Same extrapolation on every side (the singletons of extrapolation.py:1135-1156)."""
    return tuple((side, side) for _ in range(dim))


def is_const(side) -> bool:
    return not isinstance(side, str)


def kinds_of(bc):
    """A vector boundary is one spec for all components, or a LIST of `dim` specs when constants differ per component
    (ConstantExtrapolation of a vector, e.g. the lid `{'y+': vec(x=1, y=0)}` of Lid_Driven_Cavity.ipynb).  The KINDS (constant /
    ZERO_GRADIENT / PERIODIC per side) are the same in every entry - they decide the stored faces, extrapolation.py:57-62."""
    return bc[0] if isinstance(bc, list) else bc


def valid_outer_faces(bc, axis) -> Tuple[bool, bool]:
    """extrapolation.py:57-62 + determines_boundary_values: ZERO/const -> both determined (:284-285),
    copy pads (ZERO_GRADIENT) -> not determined (:451-452), PERIODIC -> only the upper face (:657-662)."""
    lo, hi = kinds_of(bc)[axis]
    lo_stored = (lo == ZG) or (lo == PERIODIC)
    hi_stored = (hi == ZG)
    return lo_stored, hi_stored


def is_flexible(bc) -> bool:
    """extrapolation.py:288 (const: False), :565 (ZERO_GRADIENT: True), :665 (PERIODIC: False);
    mixed: any() (:1288-1289)."""
    return any(side == ZG for ax in kinds_of(bc) for side in ax)


def pressure_bc(vbc) -> tuple:
    """fluid._pressure_extrapolation, phi/physics/fluid.py:264-274 (applied per side for mixed BCs)."""
    def conv(side):
        if side == PERIODIC:
            return PERIODIC
        if side == ZG:
            return ZERO
        return ZG
    return tuple((conv(lo), conv(hi)) for lo, hi in kinds_of(vbc))


def staggered_shapes(res: Sequence[int], vbc) -> List[tuple]:
    """Stored extent of each component: tests/commit/field/test__grid.py:25-37."""
    shapes = []
    for c in range(len(res)):
        lo, hi = valid_outer_faces(vbc, c)
        s = list(res)
        s[c] = res[c] - 1 + int(lo) + int(hi)
        shapes.append(tuple(s))
    return shapes


# --------------------------------------------------------------------------------------------------
# A8  pad
# --------------------------------------------------------------------------------------------------

def pad_axis(a: np.ndarray, axis: int, lo_w: int, hi_w: int, bc_axis) -> np.ndarray:
    """math.pad along one axis (PhiML/phiml/math/_ops.py:791-838).
    constant: extrapolation.py:291-325; ZERO_GRADIENT (edge copy): :568-573; PERIODIC (wrap): :671-675.
    Negative widths crop (tests/commit/math/test_extrapolation.py:53-160)."""
    lo_side, hi_side = bc_axis
    # positive widths are padded first, negative widths are sliced off afterwards (_ops.py:830-838)
    crop_lo, crop_hi = max(0, -lo_w), max(0, -hi_w)
    lo_w, hi_w = max(0, lo_w), max(0, hi_w)
    parts = []
    if lo_w > 0:
        if lo_side == PERIODIC:
            parts.append(np.take(a, np.arange(a.shape[axis] - lo_w, a.shape[axis]), axis=axis))
        elif lo_side == ZG:
            parts.append(np.repeat(np.take(a, [0], axis=axis), lo_w, axis=axis))
        else:
            shp = list(a.shape); shp[axis] = lo_w
            parts.append(np.full(shp, lo_side, dtype=a.dtype))
    parts.append(a)
    if hi_w > 0:
        if hi_side == PERIODIC:
            parts.append(np.take(a, np.arange(0, hi_w), axis=axis))
        elif hi_side == ZG:
            parts.append(np.repeat(np.take(a, [a.shape[axis] - 1], axis=axis), hi_w, axis=axis))
        else:
            shp = list(a.shape); shp[axis] = hi_w
            parts.append(np.full(shp, hi_side, dtype=a.dtype))
    out = np.concatenate(parts, axis=axis) if len(parts) > 1 else a
    if crop_lo or crop_hi:
        out = np.take(out, np.arange(crop_lo, out.shape[axis] - crop_hi), axis=axis)
    return out


def pad(a: np.ndarray, widths: Sequence[Tuple[int, int]], bc) -> np.ndarray:
    for axis, (lo_w, hi_w) in enumerate(widths):
        if lo_w or hi_w:
            a = pad_axis(a, axis, lo_w, hi_w, bc[axis])
    return a


# --------------------------------------------------------------------------------------------------
# A7  laplace      A5  divergence      A6  gradient at faces
# --------------------------------------------------------------------------------------------------

def laplace(x: np.ndarray, dx: Sequence[float], bc) -> np.ndarray:
    """math.laplace, PhiML/phiml/math/_nd.py:825-861 via shift (:480-535):
    sum_d (left + right - 2*center) / dx_d**2 with one ghost layer from `bc`."""
    x = x.astype(F32)
    result = None
    for axis in range(x.ndim):
        p = pad_axis(x, axis, 1, 1, bc[axis])
        n = x.shape[axis]
        left = np.take(p, np.arange(0, n), axis=axis)
        right = np.take(p, np.arange(2, n + 2), axis=axis)
        term = (left + right - F32(2) * x) / (F32(dx[axis]) ** 2)
        result = term if result is None else result + term
    return result


def bake_staggered(v: List[np.ndarray], vbc_comp) -> List[np.ndarray]:
    """field.bake_extrapolation for staggered grids, phi/field/_field_math.py:20-39:
    pad component d along d to n_d+1 faces with its own boundary."""
    out = []
    for c, comp in enumerate(v):
        lo, hi = valid_outer_faces(vbc_comp[c], c)
        out.append(pad_axis(comp, c, 0 if lo else 1, 0 if hi else 1, vbc_comp[c][c]))
    return out


def divergence_staggered(v: List[np.ndarray], dx: Sequence[float], vbc_comp) -> np.ndarray:
    """field.divergence order 2, staggered branch, phi/field/_field_math.py:617-626:
    sum_d forward-difference(baked v_d)/dx_d (math.spatial_gradient 'forward', _nd.py:813-815)."""
    baked = bake_staggered(v, vbc_comp)
    result = None
    for c, comp in enumerate(baked):
        n = comp.shape[c] - 1
        left = np.take(comp, np.arange(0, n), axis=c)
        right = np.take(comp, np.arange(1, n + 1), axis=c)
        term = (right - left) / F32(dx[c])
        result = term if result is None else result + term
    return result


def gradient_faces(p: np.ndarray, dx: Sequence[float], pbc, vbc) -> List[np.ndarray]:
    """field.spatial_gradient(p, at='face') order 2 = stagger(), phi/field/_field_math.py:229-236, 535-581:
    (upper - lower)/dx on the faces that `vbc` stores; pad widths per :564-572, ghost p from `pbc`."""
    out = []
    for c in range(p.ndim):
        lo, hi = valid_outer_faces(vbc, c)
        if lo and hi:
            wl, wu = (1, 0), (0, 1)
        elif lo and not hi:
            wl, wu = (1, -1), (0, 0)
        elif (not lo) and hi:
            wl, wu = (0, 0), (-1, 1)
        else:
            wl, wu = (0, -1), (-1, 0)
        lower = pad_axis(p, c, wl[0], wl[1], pbc[c])
        upper = pad_axis(p, c, wu[0], wu[1], pbc[c])
        out.append((upper - lower) / F32(dx[c]))
    return out


# --------------------------------------------------------------------------------------------------
# Appendix A of SURVEY.md: the CenteredGrid-velocity ("collocated", wide stencil) variant of the projection
# --------------------------------------------------------------------------------------------------

def gradient_centered(p: np.ndarray, dx: Sequence[float], pbc) -> List[np.ndarray]:
    """field.spatial_gradient(p, at='center') order 2 (phi/field/_field_math.py:230-233) = math.spatial_gradient
    'central' (PhiML/phiml/math/_nd.py:810-812): (p[i+1] - p[i-1]) / (2 dx) with ghost p from the pressure boundary."""
    out = []
    for c in range(p.ndim):
        q = pad_axis(p, c, 1, 1, pbc[c])
        n = p.shape[c]
        out.append((np.take(q, np.arange(2, n + 2), axis=c) - np.take(q, np.arange(0, n), axis=c)) / (F32(dx[c]) * F32(2)))
    return out


def divergence_centered(v: List[np.ndarray], dx: Sequence[float], vbc_comp) -> np.ndarray:
    """field.divergence of a CenteredGrid, order 2 (phi/field/_field_math.py:627-632): sum_d (v_d[i+1] - v_d[i-1]) / (2 dx_d)
    with ghost values from the velocity boundary of component d."""
    result = None
    for c, comp in enumerate(v):
        q = pad_axis(comp, c, 1, 1, vbc_comp[c][c])
        n = comp.shape[c]
        term = (np.take(q, np.arange(2, n + 2), axis=c) - np.take(q, np.arange(0, n), axis=c)) / (F32(dx[c]) * F32(2))
        result = term if result is None else result + term
    return result


def remove_constant_offset(bc):
    """extrapolation.remove_constant_offset: constants become 0, the rest is kept (fluid.py:200)."""
    return tuple(tuple(s if isinstance(s, str) else 0.0 for s in ax) for ax in bc)


def wide_laplace(p: np.ndarray, dx: Sequence[float], pbc, vbc) -> np.ndarray:
    """fluid.masked_laplace(wide_stencil=True) without obstacles (phi/physics/fluid.py:197-202): centred divergence of the
    centred gradient; the gradient's ghosts follow the velocity boundary with constants removed."""
    d = p.ndim
    vbc0 = remove_constant_offset(vbc)
    return divergence_centered(gradient_centered(p, dx, pbc), dx, [vbc0] * d)


def wide_poisson_matrix(res: Sequence[int], dx: Sequence[float], vbc) -> sp.csr_matrix:
    """Matrix of wide_laplace (what jit_compile_linear traces for CenteredGrid velocities): interior rows
    [1 0 -2 0 1] / (4 dx^2) per axis.  Built column by column from unit vectors (small grids only); C order of (x, y, z)."""
    n = int(np.prod(res))
    pbc = pressure_bc(vbc)
    cols = []
    for j in range(n):
        e = np.zeros(n, F32)
        e[j] = 1
        cols.append(wide_laplace(e.reshape(res), dx, pbc, vbc).ravel())
    return sp.csr_matrix(np.stack(cols, axis=1).astype(F32))


def make_incompressible_centered(v: List[np.ndarray], vbc, res, dx, rtol=1e-5, atol=1e-5, max_iter=1000, rng=None, method='CG-adaptive'):
    """fluid.make_incompressible for a CenteredGrid velocity (phi/physics/fluid.py:138-161 with wide_stencil=True, :154-155):
    centred divergence -> (balance) -> solve on the wide operator (+ the rank-1 offset of _optimize.py:705-714 when the system
    is rank deficient) -> v -= centred gradient of p.
    The default Solve() has method 'auto', which the vendored PhiML maps to CG-adaptive (backend/_backend.py:1446-1447).
    That matters here: the boundary rows of the wide operator are not symmetric (the ghosts of the gradient follow the
    pressure boundary, those of the divergence the velocity boundary), and plain CG does not reach rtol 1e-5 within 1000
    iterations on the reference test's systems, CG-adaptive needs 28-43 (measured with this oracle)."""
    d = len(res)
    div = divergence_centered(v, dx, component_bcs(vbc, d))
    pbc = pressure_bc(vbc)
    A = wide_poisson_matrix(res, dx, vbc)
    offset = None
    if not is_flexible(vbc):
        div = div - np.mean(div, dtype=F32)
        offset = estimate_matrix_offset(A, div.size, rng if rng is not None else np.random.default_rng(0))
    info = (cg_adaptive if method == 'CG-adaptive' else cg)(A, div, np.zeros(res, F32), rtol, atol, max_iter, offset)
    p = info['x'].reshape(res)
    grad = gradient_centered(p, dx, pbc)
    return [v[c] - grad[c] for c in range(d)], p, info


# --------------------------------------------------------------------------------------------------
# A11  grid_sample (the NumPy backend has no native grid_sample -> python fallback is the oracle)
# --------------------------------------------------------------------------------------------------

def _closest_setup(grid: np.ndarray, coords: np.ndarray, bc):
    """math._closest_grid_values, PhiML/phiml/math/_ops.py:902-933."""
    d = grid.ndim
    widths = []
    shift = np.zeros(d, dtype=F32)
    for ax in range(d):
        lo, hi = bc[ax]
        lo_p = 1 if is_const(lo) else 0     # not extrap.is_copy_pad(dim, False)
        hi_p = 1 if is_const(hi) else 0
        widths.append((lo_p, hi_p))
        shift[ax] = lo_p
    padded = pad(grid, widths, bc)
    c = (coords + shift).astype(F32)
    i0 = np.floor(c).astype(np.int32)
    i1 = i0 + 1

    def transform(idx):
        out = np.empty_like(idx)
        for ax in range(d):
            lo, hi = bc[ax]
            n = padded.shape[ax]
            if lo == PERIODIC and hi == PERIODIC:
                out[..., ax] = np.mod(idx[..., ax], n)          # extrapolation.py:668-669
            else:
                out[..., ax] = np.clip(idx[..., ax], 0, n - 1)  # extrapolation.py:160-176 (also mixed :1313-1326)
        return out
    return padded, transform(i0), transform(i1)


def closest_grid_values(grid: np.ndarray, coords: np.ndarray, bc) -> np.ndarray:
    """Returns the 2^d neighbour values, shape coords.shape[:-1] + (2,)*d (PhiML test__ops.py:317-321)."""
    d = grid.ndim
    padded, lo_idx, hi_idx = _closest_setup(grid.astype(F32), coords, bc)
    out = np.empty(coords.shape[:-1] + (2,) * d, dtype=F32)
    for corner in itertools.product((0, 1), repeat=d):
        idx = tuple(np.where(corner[ax], hi_idx[..., ax], lo_idx[..., ax]) for ax in range(d))
        out[(Ellipsis,) + corner] = padded[idx]
    return out


def grid_sample(grid: np.ndarray, coords: np.ndarray, bc) -> np.ndarray:
    """math.grid_sample -> _grid_sample fallback, PhiML/phiml/math/_ops.py:936-1015:
    weights = prod_axis(binary*frac + (1-binary)*(1-frac)), frac = coords % 1; result = sum(neighbors*weights)."""
    d = grid.ndim
    coords = coords.astype(F32)
    neighbors = closest_grid_values(grid, coords, bc)
    frac = np.mod(coords, F32(1)).astype(F32)
    weights = np.empty_like(neighbors)
    for corner in itertools.product((0, 1), repeat=d):
        w = None
        for ax in range(d):
            f = frac[..., ax] if corner[ax] else (F32(1) - frac[..., ax])
            w = f if w is None else w * f
        weights[(Ellipsis,) + corner] = w
    prod = neighbors * weights
    return prod.reshape(prod.shape[:-d] + (-1,)).sum(-1, dtype=F32)


# --------------------------------------------------------------------------------------------------
# geometry of sample points
# --------------------------------------------------------------------------------------------------

def cell_centers_1d(lower: float, size: float, n: int) -> np.ndarray:
    """UniformGrid.center, phi/geom/_grid.py:60-64: lower + linspace(.5/n, 1-.5/n, n) * size."""
    local = np.linspace(0.5 / n, 1 - 0.5 / n, n).astype(F32)
    return (local * F32(size) + F32(lower)).astype(F32)


def component_grid(lower, upper, res, vbc, c):
    """UniformGrid.stagger(dim, lower, upper), phi/geom/_grid.py:204-209 -> (lower', upper', res')."""
    lo_st, hi_st = valid_outer_faces(vbc, c)
    lower = [F32(v) for v in lower]
    upper = [F32(v) for v in upper]
    unit = (upper[c] - lower[c]) / F32(res[c])
    lo2 = list(lower); up2 = list(upper); r2 = list(res)
    lo2[c] = lower[c] + unit * F32(-0.5 if lo_st else 0.5)
    up2[c] = upper[c] + unit * F32(0.5 if hi_st else -0.5)
    r2[c] = res[c] + int(lo_st) + int(hi_st) - 1
    return lo2, up2, r2


def points_of(lower, upper, res) -> np.ndarray:
    """Cell centres of a uniform grid, shape res + (d,)."""
    axes = [cell_centers_1d(lower[a], F32(upper[a]) - F32(lower[a]), res[a]) for a in range(len(res))]
    mesh = np.meshgrid(*axes, indexing='ij')
    return np.stack(mesh, -1).astype(F32)


def to_index_space(points: np.ndarray, lower, upper, res) -> np.ndarray:
    """sample_grid_at_centers, phi/field/_resample.py:257-258:
    bounds.global_to_local(points) * resolution - 0.5 (Box.global_to_local, phi/geom/_box.py:134-152)."""
    lower = np.asarray(lower, dtype=F32)
    size = (np.asarray(upper, dtype=F32) - lower).astype(F32)
    local = ((points - lower) / size).astype(F32)
    return (local * np.asarray(res, dtype=F32) - F32(0.5)).astype(F32)


# --------------------------------------------------------------------------------------------------
# A10  staggered velocity at cell centres / at the faces of component c (shift resampling)
# --------------------------------------------------------------------------------------------------

def _half_shift_average(a: np.ndarray, axis: int) -> np.ndarray:
    """math.sample_subgrid with start%1 == .5 along `axis` (_nd.py:973-1003):
    upper*0.5 + lower*0.5 over neighbouring entries (result is one shorter)."""
    n = a.shape[axis]
    lower = np.take(a, np.arange(0, n - 1), axis=axis)
    upper = np.take(a, np.arange(1, n), axis=axis)
    return upper * F32(0.5) + lower * F32(0.5)


def sample_component_on_grid(comp: np.ndarray, c: int, res, vbc_c, target_face_axis, target_vbc) -> np.ndarray:
    """Component `c` of a staggered grid sampled at
         * the cell centres              (target_face_axis is None), or
         * the stored faces of component `target_face_axis`
       through sample_staggered_grid -> sample_grid_at_centers -> _shift_resample -> sample_subgrid
       (phi/field/_resample.py:279-287, 241-256, 341-364).  Source and target share dx, so the resampling is a
       pad (with the component's own boundary) followed by 0.5/0.5 averages along every half-offset axis."""
    d = comp.ndim
    a = comp.astype(F32)
    if target_face_axis == c:
        return a
    # pad (field.pad with the component's boundary): n_c+1 faces along its own axis ...
    lo_st, hi_st = valid_outer_faces(vbc_c, c)
    a = pad_axis(a, c, 0 if lo_st else 1, 0 if hi_st else 1, vbc_c[c])
    t = target_face_axis
    if t is not None:
        # ... and cells -1 .. n_t along the target's face axis (the component is cell-centred there)
        a = pad_axis(a, t, 1, 1, vbc_c[t])
    # sample_subgrid lerps the half-offset axes in spatial order (x, y, z)
    for ax in sorted([c] + ([t] if t is not None else [])):
        a = _half_shift_average(a, ax)
    if t is None:
        return a
    t_lo, t_hi = valid_outer_faces(target_vbc, t)
    n_t = res[t]
    first = 0 if t_lo else 1
    last = n_t if t_hi else n_t - 1
    return np.take(a, np.arange(first, last + 1), axis=t)


def component_bcs(vbc, dim):
    """Per-component boundary of a vector field: the same spec for every component, or the given list (see kinds_of)."""
    return list(vbc) if isinstance(vbc, list) else [vbc for _ in range(dim)]


# --------------------------------------------------------------------------------------------------
# A9  semi-Lagrangian advection, N1 MacCormack
# --------------------------------------------------------------------------------------------------

def _velocity_at_centers(v, res, vbc):
    d = len(res)
    comp = component_bcs(vbc, d)
    return np.stack([sample_component_on_grid(v[c], c, res, comp[c], None, vbc) for c in range(d)], -1)


def _velocity_at_faces(v, res, vbc, target_axis, target_vbc):
    d = len(res)
    comp = component_bcs(vbc, d)
    return np.stack([sample_component_on_grid(v[c], c, res, comp[c], target_axis, target_vbc) for c in range(d)], -1)


def semi_lagrangian_centered(s: np.ndarray, sbc, v: List[np.ndarray], vbc, lower, upper, dt: float) -> np.ndarray:
    """advect.semi_lagrangian for a CenteredGrid advected by a StaggeredGrid of the same resolution,
    phi/physics/advect.py:156-179 with euler (:20-24)."""
    res = s.shape
    v0 = _velocity_at_centers(v, res, vbc)
    pts = points_of(lower, upper, res)
    lookup = (pts + v0 * F32(-dt)).astype(F32)
    return grid_sample(s.astype(F32), to_index_space(lookup, lower, upper, res), sbc)


def semi_lagrangian_staggered(f: List[np.ndarray], fbc, v: List[np.ndarray], vbc, res, lower, upper, dt: float):
    """advect.semi_lagrangian for a StaggeredGrid `f` advected by StaggeredGrid `v` on the same cells
    (self-advection when f is v).  Sample points = stored faces of `f`; velocity there via A10; every component is
    then interpolated on its own staggered sub-grid (reduce_sample, phi/field/_resample.py:66-72, 148-153)."""
    d = len(res)
    fbc_comp = component_bcs(fbc, d)
    out = []
    for c in range(d):
        v0 = _velocity_at_faces(v, res, vbc, c, fbc)
        lo_c, up_c, res_c = component_grid(lower, upper, res, fbc, c)
        pts = points_of(lo_c, up_c, res_c)
        lookup = (pts + v0 * F32(-dt)).astype(F32)
        out.append(grid_sample(f[c].astype(F32), to_index_space(lookup, lo_c, up_c, res_c), fbc_comp[c]))
    return out


def mac_cormack_centered(s, sbc, v, vbc, lower, upper, dt: float, correction_strength=1.0):
    """advect.mac_cormack, phi/physics/advect.py:182-215, CenteredGrid advected by a StaggeredGrid."""
    res = s.shape
    s = s.astype(F32)
    v0 = _velocity_at_centers(v, res, vbc)
    pts = points_of(lower, upper, res)
    p_bwd = (pts + v0 * F32(-dt)).astype(F32)
    p_fwd = (pts + v0 * F32(dt)).astype(F32)
    c_bwd = to_index_space(p_bwd, lower, upper, res)
    c_fwd = to_index_space(p_fwd, lower, upper, res)
    fwd_adv = grid_sample(s, c_bwd, sbc)
    bwd_adv = grid_sample(fwd_adv, c_fwd, sbc)
    new = fwd_adv + F32(correction_strength * 0.5) * (s - bwd_adv)
    limits = closest_grid_values(s, c_bwd, sbc)
    flat = limits.reshape(limits.shape[:-len(res)] + (-1,))
    return np.clip(new, flat.min(-1), flat.max(-1)).astype(F32)


# --------------------------------------------------------------------------------------------------
# centred -> faces resampling (buoyancy), N2
# --------------------------------------------------------------------------------------------------

def centered_to_faces(s: np.ndarray, sbc, vbc) -> List[np.ndarray]:
    """resample(CenteredGrid, to=StaggeredGrid) = sample_grid_at_faces (phi/field/_resample.py:272-276):
    each staggered sub-grid has the same dx and a half-cell offset -> _shift_resample: pad with the scalar's
    boundary, 0.5/0.5 average of the two cells adjacent to every stored face."""
    out = []
    for c in range(s.ndim):
        lo_st, hi_st = valid_outer_faces(vbc, c)
        a = pad_axis(s.astype(F32), c, 1, 1, sbc[c])
        a = _half_shift_average(a, c)            # faces 0..n
        n = s.shape[c]
        first = 0 if lo_st else 1
        last = n if hi_st else n - 1
        out.append(np.take(a, np.arange(first, last + 1), axis=c))
    return out


# --------------------------------------------------------------------------------------------------
# A2 / A12  the pressure matrix and CG
# --------------------------------------------------------------------------------------------------

def poisson_matrix(res: Sequence[int], dx: Sequence[float], pbc) -> sp.csr_matrix:
    """The CSR matrix the reference obtains by tracing fluid.masked_laplace (phi/physics/fluid.py:165-202)
    with matrix_from_function (PhiML/phiml/math/_trace.py:665-732); rows per boundary type: SURVEY.md Appendix A.
    Flattening order = C order of (x, y, z) (reshaped_native, _optimize.py:696-697)."""
    d = len(res)
    mats = []
    for ax in range(d):
        n = res[ax]
        lo, hi = pbc[ax]
        main = np.full(n, -2.0)
        off = np.ones(n - 1)
        m = sp.diags([off, main, off], [-1, 0, 1], shape=(n, n), format='lil')
        if lo == PERIODIC:
            m[0, n - 1] += 1.0
            m[n - 1, 0] += 1.0
        else:
            if lo == ZG:
                m[0, 0] += 1.0       # ghost = edge  -> [-1 1]
            if hi == ZG:
                m[n - 1, n - 1] += 1.0
            # constant 0 ghost (Dirichlet) keeps [-2 1]
        inv = F32(1) / (F32(dx[ax]) ** 2)
        mats.append((m.tocsr() * float(inv)))
    total = None
    for ax in range(d):
        term = None
        for a2 in range(d):
            factor = mats[ax] if a2 == ax else sp.identity(res[a2], format='csr')
            term = factor if term is None else sp.kron(term, factor, format='csr')
        total = term if total is None else total + term
    total = total.tocsr().astype(F32)
    total.sort_indices()
    return total


def estimate_matrix_offset(A: sp.csr_matrix, n: int, rng: np.random.Generator) -> float:
    """_linear_solve_forward, PhiML/phiml/math/_optimize.py:705-714: random-probe estimate of the matrix scale."""
    random_x = rng.uniform(0, 1, size=n).astype(F32)
    random_y = A.dot(random_x)
    random_y_std = np.mean(np.abs(random_y), dtype=F32)
    return float(np.sqrt(random_y_std * F32(9) / F32(n)))


def cg(A, y: np.ndarray, x0: np.ndarray, rtol: float, atol: float, max_iter: int, matrix_offset=None):
    """Backend-generic CG, PhiML/phiml/backend/_linalg.py:52-90, with stop_on_l2 (:23-40) and
    linear() incl. the rank-1 offset (:784-789).  One batch entry.  Returns dict(x, residual, iterations,
    converged, diverged)."""
    y = y.astype(F32).ravel()
    x = x0.astype(F32).ravel().copy()

    def linear(vec, without=False):
        res = A.dot(vec).astype(F32)
        res_wo = res
        if matrix_offset is not None:
            res = res + np.sum(vec, dtype=F32) * F32(matrix_offset)
        return (res, res_wo) if without else res

    y0, y0_tol = linear(x, True)
    residual, residual_tol = y - y0, y - y0_tol
    dx = residual
    delta0 = np.sum(residual * dx, dtype=F32)
    delta0_tol = np.sum(residual_tol * residual_tol, dtype=F32)
    tol_sq = max(F32(rtol) ** 2 * abs(delta0_tol), F32(atol) ** 2)
    rsq0 = abs(delta0)
    iterations = 0

    def check(it, rsq, first):
        rsq = abs(rsq)
        converged = bool(rsq <= tol_sq)
        if first:
            diverged = not np.isfinite(rsq)
        else:
            with np.errstate(divide='ignore', invalid='ignore'):
                diverged = bool((rsq / rsq0 > 1e5) and it >= 8) or not np.isfinite(rsq)
        return (not converged) and (not diverged) and it < max_iter, converged, diverged

    cont, converged, diverged = check(0, delta0, True)
    delta = delta0
    while cont:
        iterations += 1
        dy = linear(dx)
        dx_dy = np.sum(dx * dy, dtype=F32)
        step = F32(0) if dx_dy == 0 else F32(delta / dx_dy)
        x = x + step * dx
        residual = residual - step * dy
        delta_old = delta
        delta = np.sum(residual * residual, dtype=F32)
        beta = F32(0) if delta_old == 0 else F32(delta / delta_old)
        dx = residual + beta * dx
        cont, converged, diverged = check(iterations, delta, False)
    return dict(x=x, residual=residual, iterations=iterations, converged=converged, diverged=diverged,
                residual_sq=float(abs(delta)), tol_sq=float(tol_sq))


def cg_adaptive(A, y: np.ndarray, x0: np.ndarray, rtol: float, atol: float, max_iter: int, matrix_offset=None):
    """CG-adaptive (Hestenes-Stiefel variant), PhiML/phiml/backend/_linalg.py:93-128.  Differences to cg(): the step is
    (dx.r)/(dx.dy), the new direction is r - ((r.dy)/(dx.dy)) dx with dy = A dx kept from the previous iteration, and the
    tolerance is relative to |y|^2 (:109), not to the initial residual.  One batch entry; dict as cg() + function_evaluations."""
    y = y.astype(F32).ravel()
    x = x0.astype(F32).ravel().copy()

    def linear(vec):
        res = A.dot(vec).astype(F32)
        if matrix_offset is not None:
            res = res + np.sum(vec, dtype=F32) * F32(matrix_offset)
        return res

    def div_no_nan(a, b):
        return F32(0) if b == 0 else F32(a / b)

    dx = residual = y - linear(x)
    dy = linear(dx)
    iterations, function_evaluations = 0, 1
    rsq = np.sum(residual ** 2, dtype=F32)
    tol_sq = max(F32(rtol) ** 2 * np.sum(y ** 2, dtype=F32), F32(atol) ** 2)
    rsq0 = abs(rsq)

    def check(it, r2, first):
        r2 = abs(r2)
        converged = bool(r2 <= tol_sq)
        if first:
            diverged = not np.isfinite(r2)
        else:
            with np.errstate(divide='ignore', invalid='ignore'):
                diverged = bool((r2 / rsq0 > 1e5) and it >= 8) or not np.isfinite(r2)
        return (not converged) and (not diverged) and it < max_iter, converged, diverged

    cont, converged, diverged = check(0, rsq, True)
    while cont:
        iterations += 1
        dx_dy = np.sum(dx * dy, dtype=F32)
        step = div_no_nan(np.sum(dx * residual, dtype=F32), dx_dy)
        x = x + step * dx
        residual = residual - step * dy
        rsq = np.sum(residual ** 2, dtype=F32)
        dx = residual - div_no_nan(np.sum(residual * dy, dtype=F32), dx_dy) * dx
        dy = linear(dx)
        function_evaluations += 1
        cont, converged, diverged = check(iterations, rsq, False)
    return dict(x=x, residual=residual, iterations=iterations, function_evaluations=function_evaluations, converged=converged,
                diverged=diverged, residual_sq=float(abs(rsq)), tol_sq=float(tol_sq))


def make_incompressible(v: List[np.ndarray], vbc, res, dx, rtol=1e-5, atol=1e-5, max_iter=1000, x0=None,
                        use_matrix_offset=True, rng=None, matrix=None):
    """fluid.make_incompressible, no obstacles, order 2, StaggeredGrid: phi/physics/fluid.py:94-162.
    Returns (v_new components, pressure array, solve info)."""
    d = len(res)
    vbc_comp = component_bcs(vbc, d)
    div = divergence_staggered(v, dx, vbc_comp)                                  # :138
    pbc = pressure_bc(vbc)                                                       # :149-151
    rank_deficient = not is_flexible(vbc)                                        # :145-148
    if rank_deficient:
        div = div - np.mean(div, dtype=F32)                                      # _balance_divergence :205-209
    A = matrix if matrix is not None else poisson_matrix(res, dx, pbc)
    offset = None
    if rank_deficient and use_matrix_offset:
        offset = estimate_matrix_offset(A, int(np.prod(res)), rng or np.random.default_rng(0))
    x0 = np.zeros(res, F32) if x0 is None else x0
    info = cg(A, div, x0, rtol, atol, max_iter, offset)                          # :156
    p = info['x'].reshape(res)
    grad = gradient_faces(p, dx, pbc, vbc)                                       # :158
    v_new = [a - g for a, g in zip(v, grad)]                                     # :161
    return v_new, p, info


def diffuse_explicit(u, bc, dx, diffusivity: float, dt: float, substeps: int = 1):
    """diffuse.explicit, phi/physics/diffuse.py:13-60: `substeps` x  u += amount * laplace(u), amount = diffusivity * (dt / substeps).
    `u` = centred array with its boundary spec, or a list of staggered components with the vector boundary: the reference's
    staggered laplace (phi/field/_field_math.py:118-145, `fields = [u]`, math.laplace pads every component of the non-uniform stack
    by one layer of the component's own boundary) is the per-component laplace - checked against the vendored PhiML in
    tests/test_staggered_diffusion.py."""
    amount = F32(diffusivity * (dt / substeps))
    if isinstance(u, list):
        comp = component_bcs(bc, len(u))
        return [diffuse_explicit(a, comp[c], dx, diffusivity, dt, substeps) for c, a in enumerate(u)]
    u = u.astype(F32)
    for _ in range(substeps):
        u = (u + amount * laplace(u, dx, bc)).astype(F32)
    return u


# --------------------------------------------------------------------------------------------------
# the notebook step = incompressible_step (examples/grids/Smoke_Plume.ipynb:58-68)
# --------------------------------------------------------------------------------------------------

def sphere_soft_mask(center, radius, lower, upper, res) -> np.ndarray:
    """resample(Sphere, to=CenteredGrid, soft=True): Geometry.approximate_fraction_inside
    (phi/geom/_geom.py:278-308, balance 0.5) with Sphere.approximate_signed_distance (phi/geom/_sphere.py:107-120)
    and the cells' bounding radius |half_size|."""
    pts = points_of(lower, upper, res)
    diff = pts - np.asarray(center, dtype=F32)
    dist = np.sqrt(np.maximum(np.sum(diff * diff, -1, dtype=F32), F32(1e-3) ** 2)).astype(F32)   # vec_length(eps=1e-3)
    half = [(F32(upper[a]) - F32(lower[a])) / F32(res[a]) * F32(0.5) for a in range(len(res))]
    cell_radius = np.sqrt(np.sum(np.asarray(half, F32) ** 2, dtype=F32))
    frac = F32(0.5) - (dist - F32(radius)) / cell_radius
    return np.clip(frac, 0, 1).astype(F32)


def plume_step(v, s, p, dt, vbc, sbc, lower, upper, res, inflow_mask, inflow_rate, buoyancy, rtol=1e-3, atol=1e-5,
               max_iter=1000, smoke_advection='semi_lagrangian', use_matrix_offset=True, rng=None, matrix=None):
    """One smoke-plume step (Smoke_Plume.ipynb `step`): advect smoke + inflow, buoyancy, self-advect velocity,
    pressure projection with warm start x0=p."""
    d = len(res)
    dx = [(F32(upper[a]) - F32(lower[a])) / F32(res[a]) for a in range(d)]
    if smoke_advection == 'mac_cormack':
        s_adv = mac_cormack_centered(s, sbc, v, vbc, lower, upper, dt)
    else:
        s_adv = semi_lagrangian_centered(s, sbc, v, vbc, lower, upper, dt)
    s_new = (s_adv + F32(inflow_rate) * inflow_mask).astype(F32)
    # buoyancy = resample(s * (0, 0.1), to=v): scale the centred field first, then average to the faces
    faces = [centered_to_faces(s_new * F32(buoyancy[c]), sbc, vbc)[c] for c in range(d)]
    v_adv = semi_lagrangian_staggered(v, vbc, v, vbc, res, lower, upper, dt)
    v_b = [(v_adv[c] + faces[c] * F32(dt)).astype(F32) for c in range(d)]
    v_new, p_new, info = make_incompressible(v_b, vbc, res, dx, rtol, atol, max_iter, x0=p,
                                             use_matrix_offset=use_matrix_offset, rng=rng, matrix=matrix)
    return v_new, s_new, p_new, info


# --------------------------------------------------------------------------------------------------
# N4  static obstacles: accessible / hard_bcs masks (phi/physics/fluid.py:130-137, 165-202, 212-240)
# --------------------------------------------------------------------------------------------------

def accessible_bc(vbc) -> tuple:
    """fluid._accessible_extrapolation (phi/physics/fluid.py:277-288): PERIODIC -> PERIODIC, BOUNDARY -> ONE, constant -> ZERO."""
    def conv(side):
        if side == PERIODIC:
            return PERIODIC
        return 1.0 if side == ZG else 0.0
    return tuple((conv(lo), conv(hi)) for lo, hi in vbc)


def hard_bcs_faces(accessible: np.ndarray, vbc) -> List[np.ndarray]:
    """field.stagger(accessible, math.minimum, velocity.boundary, at='face') (fluid.py:134, _field_math.py:535-581):
    1 on faces between two accessible cells, 0 on faces touching an obstacle; ghost cells from accessible_bc."""
    abc = accessible_bc(vbc)
    out = []
    for c in range(accessible.ndim):
        lo, hi = valid_outer_faces(vbc, c)
        if lo and hi:
            wl, wu = (1, 0), (0, 1)
        elif lo and not hi:
            wl, wu = (1, -1), (0, 0)
        elif (not lo) and hi:
            wl, wu = (0, 0), (-1, 1)
        else:
            wl, wu = (0, -1), (-1, 0)
        lower = pad_axis(accessible.astype(F32), c, wl[0], wl[1], abc[c])
        upper = pad_axis(accessible.astype(F32), c, wu[0], wu[1], abc[c])
        out.append(np.minimum(lower, upper))
    return out


DENSE_MASKED_MATRIX_LIMIT = 3000     # cells; above this the column-by-column builder (n x n dense, O(n^2) memory) is replaced by the assembly below


def masked_poisson_matrix_sparse(res, dx, vbc, accessible: np.ndarray) -> sp.csr_matrix:
    """The same operator assembled face by face in O(n): every face between two cells carries the flux
    min(acc_lower, acc_upper) * (p_upper - p_lower) / dx^2 (hard_bcs = field.stagger(accessible, minimum), fluid.py:134, 197-202);
    open sides (pressure Dirichlet 0) see an accessible ghost cell with p = 0, walls (pressure Neumann) no flux, periodic sides
    the wrapped neighbour; obstacle cells are identity rows.  tests/test_oracle_golden.py checks it against the column-by-column
    builder (which is pinned against the phiml-traced matrix) for every boundary kind."""
    d = len(res)
    n = int(np.prod(res))
    pbc = pressure_bc(vbc)
    acc = accessible.astype(F32)
    idx = np.arange(n).reshape(res)
    rows, cols, vals = [], [], []

    def face(i_l, i_u, w):
        rows.extend([i_l, i_l, i_u, i_u]); cols.extend([i_l, i_u, i_u, i_l]); vals.extend([-w, w, -w, w])

    for ax in range(d):
        inv = F32(1) / (F32(dx[ax]) * F32(dx[ax]))
        lo, hi = pbc[ax]
        lower = [slice(None)] * d; upper = [slice(None)] * d
        lower[ax], upper[ax] = slice(0, -1), slice(1, None)
        if res[ax] > 1:
            face(idx[tuple(lower)].ravel(), idx[tuple(upper)].ravel(), (np.minimum(acc[tuple(lower)], acc[tuple(upper)]) * inv).ravel())
        first = [slice(None)] * d; last = [slice(None)] * d
        first[ax], last[ax] = 0, res[ax] - 1
        if lo == PERIODIC:
            face(idx[tuple(last)].ravel(), idx[tuple(first)].ravel(), (np.minimum(acc[tuple(last)], acc[tuple(first)]) * inv).ravel())
        else:
            for side, sel in ((lo, first), (hi, last)):
                if is_const(side):                              # Dirichlet 0 behind an accessible ghost cell: -acc_i * p_i / dx^2
                    i = idx[tuple(sel)].ravel()
                    rows.append(i); cols.append(i); vals.append((-acc[tuple(sel)] * inv).ravel())
    A = sp.coo_matrix((np.concatenate(vals).astype(np.float64), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n)).tocsr()
    A = A + sp.diags((acc.ravel() == 0).astype(np.float64))
    A = A.astype(F32)
    A.sum_duplicates(); A.sort_indices()
    return A


def masked_poisson_matrix(res, dx, vbc, accessible: np.ndarray) -> sp.csr_matrix:
    """Matrix of fluid.masked_laplace with obstacles (fluid.py:197-202): div(hard_bcs * grad p) on active cells,
    identity on inactive ones (`where(active, div, pressure)`).  Built column-block-wise from the oracle's own
    gradient / divergence so that it follows the same restated glue (validated against a phiml-traced matrix)."""
    d = len(res)
    pbc = pressure_bc(vbc)
    n = int(np.prod(res))
    if n > DENSE_MASKED_MATRIX_LIMIT:
        return masked_poisson_matrix_sparse(res, dx, vbc, accessible)
    vbc0 = tuple(tuple(0.0 if is_const(s) else s for s in ax) for ax in vbc)      # remove_constant_offset
    hard = hard_bcs_faces(accessible, vbc)
    cols = []
    eye = np.eye(n, dtype=F32)
    for j in range(n):
        pj = eye[j].reshape(res)
        grad = gradient_faces(pj, dx, pbc, vbc0)
        grad = [g * h for g, h in zip(grad, hard)]
        div = divergence_staggered(grad, dx, component_bcs(vbc0, d))
        cols.append(np.where(accessible > 0, div, pj).ravel())
    return sp.csr_matrix(np.stack(cols, 1).astype(F32))


def make_incompressible_obstacles(v: List[np.ndarray], vbc, res, dx, accessible: np.ndarray, vmask: List[np.ndarray] = None,
                                  rtol=1e-5, atol=1e-5, max_iter=1000, x0=None, matrix=None):
    """fluid.make_incompressible with stationary obstacles (phi/physics/fluid.py:121-162):
    v <- v * (1 - obstacle mask at faces) [apply_boundary_conditions, :212-240], div *= active, balanced with
    div - active*mean(div)/mean(active) [:205-209], masked CG, v -= hard_bcs * grad p."""
    d = len(res)
    accessible = accessible.astype(F32)
    if vmask is not None:
        v = [a * m for a, m in zip(v, vmask)]
    div = divergence_staggered(v, dx, component_bcs(vbc, d)) * accessible
    if not is_flexible(vbc):
        div = div - accessible * (np.mean(div, dtype=F32) / np.mean(accessible, dtype=F32))
    A = matrix if matrix is not None else masked_poisson_matrix(res, dx, vbc, accessible)
    x0 = np.zeros(res, F32) if x0 is None else x0
    info = cg(A, div, x0, rtol, atol, max_iter, None)
    p = info['x'].reshape(res)
    grad = gradient_faces(p, dx, pressure_bc(vbc), vbc)
    hard = hard_bcs_faces(accessible, vbc)
    v_new = [a - g * h for a, g, h in zip(v, grad, hard)]
    return v_new, p, info
