"""
Reference-side adapter: real `phiml` objects in, real `phiml` objects out, libphicuda.so in between  (SURVEY.md section 8b,
boundary 1; row B1 of the scope table).

    phiml.math.extrapolation.Extrapolation  --to_spec / to_vspec-->  boundary spec of phiflow_b200._ops (-> PhiBC / PhiVBC)
    phiml.math.Tensor (named dims)          --pull_* / push_*---->   device arrays in the layout of DESIGN.md section 2
    "can the fast path do this?"            --eligible()--------->   reason string, or None when eligible

Every function here works on `phiml` Tensors and Extrapolations only, i.e. on what `Field.values`, `Field.extrapolation` and
`Field.dx` hold (phi/field/_field.py:51-82); `flow.py` next to this file applies them to real Fields.  Ineligible cases are
never computed approximately: callers get `NotEligible` and fall through to the stock implementation (the reference's own
convention for "this backend cannot do that": return NotImplemented, PhiML/phiml/math/_ops.py:983-1015).

The compute engine is `phiflow_b200._ops` (CUDA only, raises without a GPU).  Tests may substitute `ENGINE` / `DEVICE` with an
oracle-backed stand-in to exercise the plumbing on a CPU box; the product never does.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _ops

ENGINE = _ops          # the module that provides Domain, make_incompressible, advect_*, ... (tests may swap it)
DEVICE = 'cuda'


class NotEligible(Exception):
    """The case is valid PhiFlow but outside the fast path; the caller must run the stock implementation."""


def _phiml():
    try:
        from phiml import math
        from phiml.math import extrapolation
    except ImportError as err:  # pragma: no cover
        raise ImportError("phiflow_b200.phi_cuda needs PhiML / PhiFlow importable (pip install phiflow)") from err
    return math, extrapolation


# ----------------------------------------------------------------------------------------------------------------------
# (i) boundary translation  (PhiML/phiml/math/extrapolation.py:247 ConstantExtrapolation, :544 _ZeroGradient, :648 _Periodic...,
#     :1236 _MixedExtrapolation = combine_sides)
# ----------------------------------------------------------------------------------------------------------------------
def _side(ext, component: Optional[str]):
    math, E = _phiml()
    if isinstance(ext, E.ConstantExtrapolation):
        value = ext.value
        shape = getattr(value, 'shape', None)
        if shape is not None and shape.rank > 0:
            if shape.names == ('vector',) and component is not None and component in shape.get_item_names('vector'):
                value = value.vector[component]
            elif shape.volume == 1:
                value = math.reshaped_numpy(value, [shape])[0]
            else:
                raise NotEligible(f"constant boundary with shape {shape} (only scalars or per-component vectors)")
        try:
            return float(value)
        except Exception:
            raise NotEligible(f"constant boundary value {value!r} is not a plain number")
    if ext is E.ZERO_GRADIENT or type(ext).__name__ == '_ZeroGradient':
        return 'zg'
    if ext is E.PERIODIC or type(ext).__name__ == '_PeriodicExtrapolation':
        return 'periodic'
    raise NotEligible(f"boundary {ext!r} (fast path: constant, ZERO_GRADIENT, PERIODIC and per-side mixes)")


def to_spec(ext, dims: Sequence[str], component: Optional[str] = None) -> tuple:
    """Boundary of ONE scalar array: ((lower, upper) per axis in `dims` order), sides 'periodic' | 'zg' | float."""
    math, E = _phiml()
    spec = []
    for d in dims:
        if isinstance(ext, E._MixedExtrapolation):
            try:
                lo, hi = ext._at_boundary(d + '-'), ext._at_boundary(d + '+')
            except KeyError:
                raise NotEligible(f"mixed boundary {ext!r} does not cover dimension '{d}'")
            if isinstance(lo, E._MixedExtrapolation) or isinstance(hi, E._MixedExtrapolation):
                raise NotEligible("nested mixed boundaries")
        else:
            lo = hi = ext
        lo, hi = _side(lo, component), _side(hi, component)
        if (lo == 'periodic') != (hi == 'periodic'):
            raise NotEligible(f"dimension '{d}': PERIODIC on one side only")
        spec.append((lo, hi))
    return tuple(spec)


def to_vspec(ext, dims: Sequence[str]):
    """Boundary of a vector field: one spec when all components agree, else a list of per-component specs (constants may
    differ per component, the KINDS must not: they decide which faces are stored, extrapolation.py:57-62)."""
    per = [to_spec(ext, dims, component=d) for d in dims]
    kinds = [[tuple(s if isinstance(s, str) else 'c' for s in ax) for ax in p] for p in per]
    if any(k != kinds[0] for k in kinds):
        raise NotEligible("boundary kinds differ between vector components")
    return per[0] if all(p == per[0] for p in per) else per


def stored_face_counts(vspec, resolution: Sequence[int]) -> List[tuple]:
    """Shapes (x, y[, z]) of the stored staggered components (tests/commit/field/test__grid.py:25-37)."""
    spec = vspec[0] if isinstance(vspec, list) else vspec
    shapes = []
    for c in range(len(resolution)):
        lo, hi = _ops.stored_faces(spec, c)
        s = list(resolution)
        s[c] = resolution[c] - 1 + int(lo) + int(hi)
        shapes.append(tuple(s))
    return shapes


# ----------------------------------------------------------------------------------------------------------------------
# (ii) layouts: named-dim Tensors <-> device arrays  (Tensor.native(order), PhiML/phiml/math/_tensors.py:48-65)
# ----------------------------------------------------------------------------------------------------------------------
def _batch_of(*tensors):
    math, _ = _phiml()
    shape = math.merge_shapes(*[t.shape.batch for t in tensors])
    return shape


def _native(t, batch_shape, dims: Sequence[str]) -> torch.Tensor:
    """(batch, z, y, x) float32 torch tensor on DEVICE from a phiml Tensor with spatial dims `dims` (any backend)."""
    math, _ = _phiml()
    extra = t.shape.without(batch_shape).without(dims)
    if extra.volume != 1:
        raise NotEligible(f"unexpected dimensions {extra} on a grid array")
    t = math.expand(t, batch_shape)
    nat = math.reshaped_native(t, [batch_shape, *reversed(list(dims))], force_expand=True)
    if not isinstance(nat, torch.Tensor):
        nat = torch.from_numpy(np.ascontiguousarray(np.asarray(nat)))
    return nat.to(device=DEVICE, dtype=torch.float32)


def pull_centered(dom, t, batch_shape, dims) -> torch.Tensor:
    out = dom.alloc_centered()
    idx = (slice(None),) + tuple(slice(0, dom.res[a]) for a in range(dom.dim - 1, -1, -1))
    out[idx] = _native(t, batch_shape, dims)
    return out


def push_centered(dom, dev: torch.Tensor, batch_shape, dims, like=None):
    math, _ = _phiml()
    from phiml.math import spatial
    idx = (slice(None),) + tuple(slice(0, dom.res[a]) for a in range(dom.dim - 1, -1, -1))
    groups = [batch_shape] + [spatial(**{d: dom.res[a]}) for a, d in reversed(list(enumerate(dims)))]
    return math.reshaped_tensor(dev[idx].contiguous(), groups, convert=False)    # results stay on the device (no silent D2H copy)


def split_components(values, dims: Sequence[str]):
    """The per-component tensors of staggered values.  Wall / open boundaries store different face counts per component, so the
    values are a non-uniform TensorStack along the dual dim `~vector` that cannot be exported as ONE native array
    (SURVEY.md section 8b): export per component."""
    names = values.shape.names
    vdim = '~vector' if '~vector' in names else 'vector'
    if vdim not in names:
        raise NotEligible("staggered values without a vector dimension")
    return [values[{vdim: d}] for d in dims]


def pull_staggered(dom, comps: Sequence, vspec, batch_shape, dims) -> List[torch.Tensor]:
    shapes, offsets = dom.face_shapes(vspec)
    out = dom.alloc_faces()
    for c, t in enumerate(comps):
        got = tuple(t.shape.get_size(d) for d in dims)
        if got != shapes[c]:
            raise NotEligible(f"component '{dims[c]}' has shape {got}, the boundary stores {shapes[c]} faces")
        idx = [slice(None)]
        for ax in range(dom.dim - 1, -1, -1):
            start = offsets[c] if ax == c else 0
            idx.append(slice(start, start + shapes[c][ax]))
        out[c][tuple(idx)] = _native(t, batch_shape, dims)
    return out


def push_staggered(dom, dev: Sequence[torch.Tensor], vspec, batch_shape, dims):
    """-> stacked Tensor along dual(vector=dims), rebuilt like phi/field/_grid.py:179-187 does."""
    math, _ = _phiml()
    from phiml.math import spatial, dual
    shapes, offsets = dom.face_shapes(vspec)
    comps = []
    for c in range(dom.dim):
        idx = [slice(None)]
        for ax in range(dom.dim - 1, -1, -1):
            start = offsets[c] if ax == c else 0
            idx.append(slice(start, start + shapes[c][ax]))
        groups = [batch_shape] + [spatial(**{d: shapes[c][a]}) for a, d in reversed(list(enumerate(dims)))]
        comps.append(math.reshaped_tensor(dev[c][tuple(idx)].contiguous(), groups, convert=False))
    return math.stack(comps, dual(vector=tuple(dims)))


# ----------------------------------------------------------------------------------------------------------------------
# (iii) eligibility  (SURVEY.md section 3.4: UniformGrid, order 2, fp32, ZERO / ZERO_GRADIENT / PERIODIC per side, CG family)
# ----------------------------------------------------------------------------------------------------------------------
FAST_SOLVERS = ('CG', 'CG-adaptive', 'auto')


def eligible(dims: Sequence[str], ext=None, order: int = 2, solve_method: Optional[str] = None, obstacles=(), active=None,
             preconditioner=None, staggered: bool = True, uniform: bool = True) -> Optional[str]:
    """None when the fast path applies, else the reason it does not (the caller falls through to the stock implementation)."""
    math, _ = _phiml()
    if len(dims) not in (2, 3):
        return f"{len(dims)}-D grids"
    if not uniform:
        return "non-uniform geometry (meshes, graphs, point clouds)"
    if not staggered:
        return "CenteredGrid velocity (wide stencil, SURVEY.md Appendix A)"
    if order != 2:
        return f"order {order} (fast path: 2)"
    if math.get_precision() != 32:
        return f"precision {math.get_precision()} (fast path: 32; never silently downcast)"
    if active is not None:
        return "`active` masks"
    if obstacles:
        return "obstacles through this adapter (the C ABI supports stationary masks; moving obstacles never)"
    if preconditioner is not None:
        return "preconditioned solves"
    if solve_method is not None and solve_method not in FAST_SOLVERS:
        return f"solver '{solve_method}' (fast path: {', '.join(FAST_SOLVERS)})"
    if ext is not None:
        try:
            to_vspec(ext, dims) if staggered else to_spec(ext, dims)
        except NotEligible as err:
            return str(err)
    return None


# ----------------------------------------------------------------------------------------------------------------------
# (iv) the hot-path functions on phiml Tensors
# ----------------------------------------------------------------------------------------------------------------------
def _domain(res, dx, batch, vspec):
    return ENGINE.Domain(res, dx, batch, vbc=vspec, device=DEVICE)


def _dx_tuple(dx, dims) -> Tuple[float, ...]:
    if isinstance(dx, dict):
        return tuple(float(dx[d]) for d in dims)
    if hasattr(dx, 'vector'):
        return tuple(float(dx.vector[d]) for d in dims)
    return tuple(float(v) for v in dx)


def make_incompressible(values, ext, dx, dims: Sequence[str], resolution: Sequence[int], method='auto', rel_tol=1e-5, abs_tol=1e-5,
                        max_iterations=1000, x0=None):
    """fluid.make_incompressible (phi/physics/fluid.py:94-162) on the VALUES of a StaggeredGrid.
    values: stacked staggered Tensor (dual/channel dim `vector`), ext: its Extrapolation, dx: cell size per dim.
    Returns (new values, pressure Tensor, info dict with iterations / residual / converged / diverged per batch entry)."""
    reason = eligible(dims, ext, solve_method=method)
    if reason:
        raise NotEligible(reason)
    vspec = to_vspec(ext, dims)
    comps = split_components(values, dims)
    batch_shape = _batch_of(*comps, *([x0] if x0 is not None else []))
    dom = _domain(tuple(resolution), _dx_tuple(dx, dims), max(1, batch_shape.volume), vspec)
    v = pull_staggered(dom, comps, vspec, batch_shape, dims)
    p = pull_centered(dom, x0, batch_shape, dims) if x0 is not None else dom.alloc_centered()
    adaptive = method in ('auto', 'CG-adaptive')            # the reference maps 'auto' to CG-adaptive (_backend.py:1446-1447)
    prm = ENGINE.cg_params(vspec, rtol=rel_tol, atol=abs_tol, max_iter=max_iterations, method='CG-adaptive' if adaptive else 'CG')
    ENGINE.make_incompressible(dom, vspec, v, p, prm)
    res = ENGINE.read_results(dom)
    info = {k: np.array(res[k]) for k in ('iterations', 'converged', 'diverged', 'residual_sq', 'tol_sq')}
    return push_staggered(dom, v, vspec, batch_shape, dims), push_centered(dom, p, batch_shape, dims), info


def make_incompressible_centered(values, ext, dx, dims: Sequence[str], resolution: Sequence[int], method='auto', rel_tol=1e-5, abs_tol=1e-5,
                                 max_iterations=1000):
    """fluid.make_incompressible for a CenteredGrid velocity (wide stencil, phi/physics/fluid.py:154-155): values = Tensor with a
    channel dim `vector` over `dims`.  Only 'auto' / 'CG-adaptive' - the operator is not symmetric at the boundary rows and the
    reference's plain CG does not converge on it either (DESIGN.md section 1)."""
    reason = eligible(dims, ext, solve_method=method)
    if reason:
        raise NotEligible(reason)
    if method not in ('auto', 'CG-adaptive'):
        raise NotEligible(f"solver '{method}' on the wide-stencil (CenteredGrid) operator: fast path runs CG-adaptive only")
    math, _ = _phiml()
    vspec = to_vspec(ext, dims)
    comps = [values.vector[d] for d in dims]
    batch_shape = _batch_of(*comps)
    dom = _domain(tuple(resolution), _dx_tuple(dx, dims), max(1, batch_shape.volume), None)
    v = [pull_centered(dom, c, batch_shape, dims) for c in comps]
    v, p = ENGINE.make_incompressible_centered(dom, vspec, v, None, rtol=rel_tol, atol=abs_tol, max_iter=max_iterations)
    res = ENGINE.read_results(dom)
    info = {k: np.array(res[k]) for k in ('iterations', 'converged', 'diverged', 'residual_sq', 'tol_sq')}
    from phiml.math import channel
    out = math.stack([push_centered(dom, t, batch_shape, dims) for t in v], channel(vector=tuple(dims)))
    return out, push_centered(dom, p, batch_shape, dims), info


def semi_lagrangian_staggered(values, ext, velocity_values, velocity_ext, dx, dims, resolution, dt: float):
    """advect.semi_lagrangian of a StaggeredGrid by a StaggeredGrid on the same grid (phi/physics/advect.py:156-179)."""
    reason = eligible(dims, velocity_ext) or eligible(dims, ext)
    if reason:
        raise NotEligible(reason)
    vspec, fspec = to_vspec(velocity_ext, dims), to_vspec(ext, dims)
    vcomps, fcomps = split_components(velocity_values, dims), split_components(values, dims)
    batch_shape = _batch_of(*vcomps, *fcomps)
    dom = _domain(tuple(resolution), _dx_tuple(dx, dims), max(1, batch_shape.volume), vspec)
    if dom.face_shapes(fspec) != dom.face_shapes(vspec):
        raise NotEligible("advected field and velocity store different faces")
    v = pull_staggered(dom, vcomps, vspec, batch_shape, dims)
    f = v if values is velocity_values else pull_staggered(dom, fcomps, fspec, batch_shape, dims)
    out = ENGINE.advect_staggered(dom, vspec, v, fspec, f, float(dt))
    return push_staggered(dom, out, fspec, batch_shape, dims)


def semi_lagrangian_centered(values, ext, velocity_values, velocity_ext, dx, dims, resolution, dt: float, mac_cormack=False,
                             correction_strength=1.0):
    """advect.semi_lagrangian / advect.mac_cormack of a CenteredGrid by a StaggeredGrid on the same grid."""
    reason = eligible(dims, velocity_ext)
    if reason:
        raise NotEligible(reason)
    vspec, sspec = to_vspec(velocity_ext, dims), to_spec(ext, dims)
    vcomps = split_components(velocity_values, dims)
    batch_shape = _batch_of(*vcomps, values)
    dom = _domain(tuple(resolution), _dx_tuple(dx, dims), max(1, batch_shape.volume), vspec)
    v = pull_staggered(dom, vcomps, vspec, batch_shape, dims)
    s = pull_centered(dom, values, batch_shape, dims)
    if mac_cormack:
        out = ENGINE.mac_cormack_centered(dom, vspec, v, sspec, s, float(dt), correction_strength)
    else:
        out = ENGINE.advect_centered(dom, vspec, v, sspec, s, float(dt))
    return push_centered(dom, out, batch_shape, dims)


def laplace(values, ext, dx, dims, resolution):
    """field.laplace order 2 of a CenteredGrid (phi/field/_field_math.py:118-145)."""
    math, _ = _phiml()
    if math.get_precision() != 32:
        raise NotEligible(f"precision {math.get_precision()}")
    spec = to_spec(ext, dims)
    batch_shape = _batch_of(values)
    dom = _domain(tuple(resolution), _dx_tuple(dx, dims), max(1, batch_shape.volume), None)
    return push_centered(dom, ENGINE.laplace(dom, spec, pull_centered(dom, values, batch_shape, dims)), batch_shape, dims)


def divergence(values, ext, dx, dims, resolution):
    """field.divergence of a StaggeredGrid (phi/field/_field_math.py:617-626)."""
    reason = eligible(dims, ext)
    if reason:
        raise NotEligible(reason)
    vspec = to_vspec(ext, dims)
    comps = split_components(values, dims)
    batch_shape = _batch_of(*comps)
    dom = _domain(tuple(resolution), _dx_tuple(dx, dims), max(1, batch_shape.volume), vspec)
    v = pull_staggered(dom, comps, vspec, batch_shape, dims)
    return push_centered(dom, ENGINE.divergence(dom, vspec, v), batch_shape, dims)


def diffuse_implicit(values, ext, dx, dims, resolution, amount: float, staggered: bool, rel_tol=1e-5, abs_tol=1e-5, max_iterations=1000,
                     x0=None):
    """diffuse.implicit (phi/physics/diffuse.py:63-95) on the VALUES of a grid: a scalar CenteredGrid, a CenteredGrid with one channel
    dim of <= 3 components, or a PERIODIC StaggeredGrid.  Every component of every batch entry is its own system, as in the reference,
    whose tracer (PhiML/phiml/math/_trace.py) keeps the uncoupled vector dim out of the matrix.  x0: values of the same
    form (default: `values`).  Returns (new values, info dict with one record per system, ordered (batch entry, component), and
    'components': the vector dim, or None for a scalar field)."""
    math, _ = _phiml()
    if math.get_precision() != 32:
        raise NotEligible(f"precision {math.get_precision()} (fast path: 32; never silently downcast)")
    if len(dims) not in (2, 3):
        raise NotEligible(f"{len(dims)}-D grids")
    if staggered:
        vspec = to_vspec(ext, dims)
        if any(s != 'periodic' for ax in (vspec[0] if isinstance(vspec, list) else vspec) for s in ax):
            raise NotEligible("implicit diffusion of a non-periodic StaggeredGrid (the reference supports PERIODIC only, "
                              "tests/commit/physics/test_diffuse.py:25,28)")
        comps = split_components(values, dims)
        x0c = split_components(x0, dims) if x0 is not None else None
        names, spec = list(dims), vspec
    else:
        chan = values.shape.channel
        if chan.rank > 1 or chan.volume > 3:
            raise NotEligible(f"channel dims {chan} (fast path: scalar or one channel dim of <= 3 components)")
        names = list(chan.get_item_names(chan.name) or range(chan.volume)) if chan.rank else [None]
        comps = [values[{chan.name: n}] for n in names] if chan.rank else [values]
        x0c = ([x0[{chan.name: n}] for n in names] if chan.rank else [x0]) if x0 is not None else None
        specs = [to_spec(ext, dims, component=n if isinstance(n, str) else None) for n in names]
        kinds = [[tuple(s if isinstance(s, str) else 'c' for s in ax) for ax in sp] for sp in specs]
        if any(k != kinds[0] for k in kinds):
            raise NotEligible("boundary kinds differ between vector components")
        spec = specs if len(specs) > 1 else specs[0]
    batch_shape = _batch_of(*comps, *(x0c or []))
    dom = _domain(tuple(resolution), _dx_tuple(dx, dims), max(1, batch_shape.volume), None)
    u = [pull_centered(dom, c, batch_shape, dims) for c in comps]
    x = [pull_centered(dom, c, batch_shape, dims) for c in x0c] if x0c is not None else None
    out = ENGINE.diffuse_implicit(dom, spec, u if len(u) > 1 or staggered else u[0], float(amount), rel_tol, abs_tol, max_iterations,
                                  x0=(x if len(u) > 1 or staggered else x[0]) if x is not None else None)
    out = out if isinstance(out, list) else [out]
    res = ENGINE.read_results(dom, components=len(u)) if len(u) > 1 else ENGINE.read_results(dom)
    info = {k: np.array(res[k]) for k in ('iterations', 'converged', 'diverged', 'residual_sq', 'tol_sq')}
    pushed = [push_centered(dom, t, batch_shape, dims) for t in out]
    from phiml.math import dual
    info['components'] = dual(vector=tuple(dims)) if staggered else (values.shape.channel if values.shape.channel.rank else None)
    if staggered:
        return math.stack(pushed, dual(vector=tuple(dims))), info
    if not values.shape.channel.rank:
        return pushed[0], info
    chan = values.shape.channel
    item_names = chan.get_item_names(chan.name)
    from phiml.math import channel
    return math.stack(pushed, channel(**{chan.name: tuple(item_names) if item_names else len(pushed)})), info


def diffuse_implicit_varying(values, ext, dx, dims, resolution, diffusivity, dt: float, rel_tol=1e-5, abs_tol=1e-5, max_iterations=1000,
                             x0=None):
    """diffuse.implicit with a spatially varying diffusivity (phi/physics/diffuse.py:48-59, 90-95, 129-141) on the VALUES of a scalar
    CenteredGrid.  diffusivity: the values of k on the same grid (the field's spatial dims and sizes, no channel dim, batch dims a
    subset of the field's).  Every face takes min(-dt k_lo, -dt k_hi); the coefficient ghosts follow `ext` (amount.at(u),
    phi/field/_resample.py:56-63).  Returns (new values, info dict with one record per batch entry)."""
    math, _ = _phiml()
    if math.get_precision() != 32:
        raise NotEligible(f"precision {math.get_precision()} (fast path: 32; never silently downcast)")
    if len(dims) not in (2, 3):
        raise NotEligible(f"{len(dims)}-D grids")
    if values.shape.channel.rank:
        raise NotEligible(f"channel dims {values.shape.channel} with a varying diffusivity (the reference supports scalar fields only)")
    if diffusivity.shape.channel.rank or diffusivity.shape.dual.rank or diffusivity.shape.instance.rank:
        raise NotEligible(f"diffusivity dims {diffusivity.shape} (fast path: one value per cell; no anisotropic diffusivity)")
    if tuple(sorted(diffusivity.shape.spatial.names)) != tuple(sorted(dims)) or \
            any(diffusivity.shape.get_size(d) != n for d, n in zip(dims, resolution)):
        raise NotEligible(f"diffusivity on a different grid ({diffusivity.shape.spatial}; it would need resampling)")
    batch_shape = _batch_of(values, *([x0] if x0 is not None else []))
    kb = diffusivity.shape.batch
    if any(n not in batch_shape.names for n in kb.names):
        raise NotEligible(f"diffusivity batch dims {kb} that the field does not have")
    spec = to_spec(ext, dims)
    dom = _domain(tuple(resolution), _dx_tuple(dx, dims), max(1, batch_shape.volume), None)
    u = pull_centered(dom, values, batch_shape, dims)
    x = pull_centered(dom, x0, batch_shape, dims) if x0 is not None else None
    if kb.rank:
        k = pull_centered(dom, diffusivity, batch_shape, dims)             # one k per entry (expanded over the field's other batch dims)
    else:
        k = pull_centered(_domain(tuple(resolution), _dx_tuple(dx, dims), 1, None), diffusivity, kb, dims)    # one k for every entry
    out = ENGINE.diffuse_implicit_varying(dom, spec, u, k, float(dt), rel_tol, abs_tol, max_iterations, x0=x)
    res = ENGINE.read_results(dom)
    info = {k_: np.array(res[k_]) for k_ in ('iterations', 'converged', 'diverged', 'residual_sq', 'tol_sq')}
    return push_centered(dom, out, batch_shape, dims), info


def grid_sample_native(grid: torch.Tensor, coords: torch.Tensor, mode: str):
    """Backend.grid_sample contract (PhiML/phiml/backend/_backend.py:1578-1593): grid (batch, x, y[, z], channel), coordinates
    (batch, points..., d) in index space, mode in 'zeros' | 'boundary' | 'periodic'.  Anything else -> NotImplemented, the
    reference then runs its own fallback (_ops.py:983-1015)."""
    spec_side = {'zeros': 0.0, 'boundary': 'zg', 'periodic': 'periodic'}.get(mode)
    if spec_side is None or grid.dtype != torch.float32 or grid.device.type != torch.device(DEVICE).type:
        return NotImplemented
    d = grid.dim() - 2
    if d not in (2, 3) or coords.shape[-1] != d:
        return NotImplemented
    batch, channels = max(grid.shape[0], coords.shape[0]), grid.shape[-1]
    res = tuple(grid.shape[1:1 + d])
    dom = ENGINE.Domain(res, (1.0,) * d, batch * channels, device=grid.device)
    dev = dom.alloc_centered()
    src = grid.expand(batch, *grid.shape[1:]).permute(0, d + 1, *range(d, 0, -1)).reshape(batch * channels, *reversed(res))
    dev[(slice(None),) + tuple(slice(0, res[a]) for a in range(d - 1, -1, -1))] = src
    pts = coords.expand(batch, *coords.shape[1:]).reshape(batch, -1, d).to(torch.float32)
    pts = pts.repeat_interleave(channels, dim=0).contiguous()
    out = ENGINE.grid_sample(dom, ((spec_side, spec_side),) * d, dev, pts).reshape(batch, channels, *coords.shape[1:-1])
    return out.permute(0, *range(2, out.dim()), 1)                       # (batch, points..., channel)
