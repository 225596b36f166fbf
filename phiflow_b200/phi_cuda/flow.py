# pylint: disable-msg = wildcard-import, unused-wildcard-import, unused-import
"""
Standard import for the H100 fast path:   from phiflow_b200.phi_cuda.flow import *      (installed into the phi tree: phi.cuda.flow)

Extends `from phi.flow import *` exactly like phi/torch/flow.py:14-35 does for PyTorch: same names, the `phicuda` backend becomes
the default backend (unless imported inside a backend context), and the module objects `fluid`, `advect`, `field`, `diffuse` are
replaced by shallow clones whose hot-path functions try libphicuda first and FALL THROUGH to the stock implementation when a
case is not eligible (SURVEY.md section 3.4 / 8b).  Notebooks reach these functions as module attributes (`fluid.make_incompressible`,
phi/flow.py:18-19), so the clones are exported under the stock names; `phi.physics.fluid` itself is not modified - plain
`phi.flow` users in the same process keep the stock behaviour.

This file needs PhiFlow (phi >= 3) importable; everything it calls in phiflow_b200.phi_cuda._adapter works on phiml objects only.
"""
import types as _types
import warnings as _warnings

from phi.flow import *  # noqa: F401,F403
from phi import math as _math
from phi.field import Field as _Field
from phi.field import StaggeredGrid as _StaggeredGrid, CenteredGrid as _CenteredGrid
from phi.physics import fluid as _fluid, advect as _advect, diffuse as _diffuse
from phi import field as _field
from phiml import backend as _backend

from . import _adapter
from ._adapter import NotEligible
from ._backend import get_backend as _get_backend

PHICUDA = _get_backend()
if not _backend.context_backend():
    _backend.set_global_default_backend(PHICUDA)
else:  # same behaviour as phi/torch/flow.py:33-35
    _backend.ML_LOGGER.warning(f"Importing '{__name__}' within a backend context will not set the default backend.")

FALLTHROUGH_LOG = []          # (function name, reason): which calls ran on the stock implementation and why


def _grid_info(f: _Field):
    """dims, resolution, dx of a uniform grid field, or NotEligible."""
    if not (f.is_grid and getattr(f.geometry, 'is_uniform', True)):       # UniformGrid only (phi/geom/_grid.py:41-215)
        raise NotEligible("not a uniform grid")
    dims = tuple(f.resolution.names)
    res = tuple(int(f.resolution.get_size(d)) for d in dims)
    return dims, res, {d: float(f.dx.vector[d]) for d in dims}


def _fall(name, reason, stock, *args, **kwargs):
    FALLTHROUGH_LOG.append((name, str(reason)))
    return stock(*args, **kwargs)


def _report(solve, info, x, components=None):
    """SolveTape / NotConverged / Diverged protocol of math.solve_linear (PhiML/phiml/math/_optimize.py:190-204, 735-743).
    `x` is the pressure Field; the per-entry records of the kernel become Tensors over its batch dims.  The kernel keeps |r|^2 per
    entry, not the residual vector: `SolveInfo.residual` holds the residual NORM per entry (the "Max residual" of the not-converged
    message is then that norm).  components: the vector dim when every component was its own system (records ordered (batch entry,
    component)), as SolveInfo has them for the reference's batched solves."""
    import numpy as _np
    from phiml.math._optimize import SolveInfo, _SOLVE_TAPES
    batch_shape = x.values.shape.batch

    def per_entry(a):
        a = _np.asarray(a)
        if components is not None:
            groups = ([batch_shape] if batch_shape.rank else []) + [components]
            return _math.reshaped_tensor(a.reshape([max(1, batch_shape.volume)] * bool(batch_shape.rank) + [components.volume]), groups, convert=False)
        return _math.reshaped_tensor(a, [batch_shape], convert=False) if batch_shape.rank else _math.wrap(a.reshape(-1)[0])
    # one non-batch dim, so that per-entry slices stay Tensors like a real residual vector does (_optimize.py:207-214)
    residual = _math.expand(per_entry(_np.sqrt(_np.maximum(info['residual_sq'], 0.0))), _math.channel(l2_norm=1))
    res = SolveInfo(solve, x, residual, per_entry(info['iterations']), per_entry(info['iterations'] + 1),
                    per_entry(info['converged'].astype(bool)), per_entry(info['diverged'].astype(bool)), "phicuda", None, None)
    for tape in _SOLVE_TAPES:
        tape._add(solve, False, res)
    res.convergence_check(False)          # raises NotConverged / Diverged unless suppressed by the Solve


def make_incompressible(velocity, obstacles=(), solve=Solve(), active=None, order=2, correct_skew=False, wide_stencil=None):  # noqa: F405
    """fluid.make_incompressible (phi/physics/fluid.py:94-100), fast path for StaggeredGrids on uniform grids."""
    stock = _fluid.make_incompressible
    original_solve = solve
    try:
        if not isinstance(velocity, _Field) or not velocity.is_grid:
            raise NotEligible("not a grid")
        solve = solve.with_defaults('solve')     # Solve() leaves the tolerances None until the solve (_optimize.py:104-111, 130-136)
        if not velocity.is_staggered:            # CenteredGrid velocity: wide stencil, CG-adaptive only (fluid.py:154-155)
            dims, res, dx = _grid_info(velocity)
            if _fluid._get_obstacles_for(obstacles, velocity) or active is not None or order != 2 or correct_skew or wide_stencil is False \
                    or solve.x0 is not None or solve.preconditioner is not None:
                raise NotEligible("CenteredGrid velocity with obstacles / active / x0 / narrow stencil")
            values, p, info = _adapter.make_incompressible_centered(velocity.values, velocity.extrapolation, dx, dims, res, method=solve.method,
                                                                    rel_tol=float(solve.rel_tol), abs_tol=float(solve.abs_tol),
                                                                    max_iterations=int(_math.max(solve.max_iterations)))
            pressure = _CenteredGrid(p, _fluid._pressure_extrapolation(velocity.extrapolation), velocity.bounds, velocity.resolution)
            _report(solve, info, pressure)
            return velocity.with_values(values), pressure
        dims, res, dx = _grid_info(velocity)
        reason = _adapter.eligible(dims, velocity.extrapolation, order=order, solve_method=solve.method, obstacles=_fluid._get_obstacles_for(obstacles, velocity),
                                   active=active, preconditioner=solve.preconditioner)
        if reason or correct_skew or wide_stencil:
            raise NotEligible(reason or "correct_skew / wide_stencil")
        x0 = solve.x0.values if isinstance(solve.x0, _Field) else None
        values, p, info = _adapter.make_incompressible(velocity.values, velocity.extrapolation, dx, dims, res, method=solve.method,
                                                       rel_tol=float(solve.rel_tol), abs_tol=float(solve.abs_tol),
                                                       max_iterations=int(_math.max(solve.max_iterations)), x0=x0)
    except NotEligible as why:
        return _fall('make_incompressible', why, stock, velocity, obstacles, original_solve, active, order, correct_skew, wide_stencil)
    pressure = _CenteredGrid(p, _fluid._pressure_extrapolation(velocity.extrapolation), velocity.bounds, velocity.resolution)
    _report(solve, info, pressure)
    return velocity.with_values(values), pressure


def semi_lagrangian(field, velocity, dt, integrator=_advect.euler):
    """advect.semi_lagrangian (phi/physics/advect.py:156-159) with the euler integrator on uniform grids."""
    stock = _advect.semi_lagrangian
    try:
        if integrator is not _advect.euler or not isinstance(velocity, _Field) or not velocity.is_staggered or not isinstance(field, _Field):
            raise NotEligible("integrator / field types")
        dims, res, dx = _grid_info(velocity)
        if not (field.is_grid and field.bounds == velocity.bounds and field.resolution == velocity.resolution):
            raise NotEligible("field and velocity on different grids")
        if field.is_staggered:
            out = _adapter.semi_lagrangian_staggered(field.values, field.extrapolation, velocity.values, velocity.extrapolation, dx, dims, res, float(dt))
        else:
            if field.shape.channel.volume > 1:
                raise NotEligible("multi-channel centred field")
            out = _adapter.semi_lagrangian_centered(field.values, field.extrapolation, velocity.values, velocity.extrapolation, dx, dims, res, float(dt))
    except (NotEligible, TypeError, ValueError) as why:
        return _fall('semi_lagrangian', why, stock, field, velocity, dt, integrator)
    return field.with_values(out)


def mac_cormack(field, velocity, dt, correction_strength=1.0, integrator=_advect.euler):
    stock = _advect.mac_cormack
    try:
        if integrator is not _advect.euler or not isinstance(field, _Field) or field.is_staggered or not velocity.is_staggered:
            raise NotEligible("integrator / field types")
        dims, res, dx = _grid_info(velocity)
        if not (field.is_grid and field.bounds == velocity.bounds and field.resolution == velocity.resolution) or field.shape.channel.volume > 1:
            raise NotEligible("field and velocity on different grids")
        out = _adapter.semi_lagrangian_centered(field.values, field.extrapolation, velocity.values, velocity.extrapolation, dx, dims, res, float(dt),
                                                mac_cormack=True, correction_strength=float(correction_strength))
    except (NotEligible, TypeError, ValueError) as why:
        return _fall('mac_cormack', why, stock, field, velocity, dt, correction_strength, integrator)
    return field.with_values(out)


def laplace(u, axes=_math.spatial, gradient=None, order=2, implicit=None, weights=None, upwind=None, correct_skew=True):
    stock = _field.laplace
    try:
        if not isinstance(u, _Field) or not u.is_grid or u.is_staggered or order != 2 or implicit or weights is not None or gradient is not None \
                or upwind is not None or axes is not _math.spatial or u.shape.channel.volume > 1:
            raise NotEligible("laplace variant")
        dims, res, dx = _grid_info(u)
        out = _adapter.laplace(u.values, u.extrapolation, dx, dims, res)
    except (NotEligible, TypeError, ValueError) as why:
        return _fall('laplace', why, stock, u, axes, gradient, order, implicit, weights, upwind, correct_skew)
    return u.with_values(out).with_extrapolation(u.extrapolation.spatial_gradient().spatial_gradient())


def divergence(field, order=2, implicit=None, upwind=None):
    stock = _field.divergence
    try:
        if not isinstance(field, _Field) or not field.is_staggered or order != 2 or implicit or upwind is not None:
            raise NotEligible("divergence variant")
        dims, res, dx = _grid_info(field)
        out = _adapter.divergence(field.values, field.extrapolation, dx, dims, res)
    except (NotEligible, TypeError, ValueError) as why:
        return _fall('divergence', why, stock, field, order, implicit, upwind)
    return _CenteredGrid(out, field.extrapolation.spatial_gradient(), field.bounds, field.resolution)


def _number(v):
    """float of a plain number or a phiml scalar Tensor, else NotEligible (Fields, vectors, per-batch values run on the stock path)."""
    if isinstance(v, bool):
        raise NotEligible("boolean diffusivity / dt")
    if isinstance(v, (int, float)):
        return float(v)
    if isinstance(v, _math.Tensor) and v.shape.rank == 0:
        return float(v)
    raise NotEligible(f"diffusivity / dt {type(v).__name__} that is not a plain number (Field, vector or per-batch values)")


def implicit(field, diffusivity, dt, solve=Solve('CG'), gradient=None, upwind=None, correct_skew=True, gradient_for_diffusivity=True):  # noqa: F405
    """diffuse.implicit (phi/physics/diffuse.py:63-95), fast path for scalar / <= 3-channel CenteredGrids and periodic StaggeredGrids on
    uniform grids with a numeric diffusivity and dt, Solve('CG') without preconditioner, fp32."""
    stock = _diffuse.implicit
    original_solve = solve
    try:
        if not isinstance(field, _Field) or not field.is_grid:
            raise NotEligible("not a grid")
        if gradient is not None or upwind is not None:
            raise NotEligible("gradient / upwind (FVM arguments)")
        k_values = _varying_diffusivity(field, diffusivity)
        if k_values is not None:
            return _implicit_varying(field, k_values, dt, solve, stock, (field, diffusivity, dt, original_solve, gradient, upwind,
                                                                         correct_skew, gradient_for_diffusivity))
        amount = _number(diffusivity) * _number(dt)
        solve = solve.with_defaults('solve')
        if solve.method != 'CG' or solve.preconditioner is not None:
            raise NotEligible(f"solver '{solve.method}' / preconditioner {solve.preconditioner} (fast path: Solve('CG'))")
        dims, res, dx = _grid_info(field)
        x0 = solve.x0.values if isinstance(solve.x0, _Field) else None
        if solve.x0 is not None and x0 is None:
            raise NotEligible("x0 that is not a Field")
        values, info = _adapter.diffuse_implicit(field.values, field.extrapolation, dx, dims, res, amount, field.is_staggered,
                                                 rel_tol=float(solve.rel_tol), abs_tol=float(solve.abs_tol),
                                                 max_iterations=int(_math.max(solve.max_iterations)), x0=x0)
    except (NotEligible, TypeError, ValueError) as why:
        return _fall('diffuse.implicit', why, stock, field, diffusivity, dt, original_solve, gradient, upwind, correct_skew, gradient_for_diffusivity)
    out = field.with_values(values)
    _report(solve, info, out, info.pop('components'))
    return out


def _varying_diffusivity(field, diffusivity):
    """The values of a spatially varying diffusivity (diffuse.py:129-141: a centred Field, or a Tensor with spatial dims), None for
    anything else (plain numbers and per-batch values take the numeric path).  A Field must lie on `field`'s grid: the fast path does
    not resample (amount.at(u), phi/field/_resample.py:56-63, is then the identity apart from the boundary takeover)."""
    if isinstance(diffusivity, _Field):
        if not diffusivity.is_grid or diffusivity.is_staggered:
            raise NotEligible("a diffusivity Field that is not a CenteredGrid (it would need resampling)")
        try:
            same = _grid_info(diffusivity)[:2] == _grid_info(field)[:2] and bool(diffusivity.bounds == field.bounds)
        except (TypeError, ValueError, AttributeError):
            same = False
        if not same:
            raise NotEligible("a diffusivity on a different grid (bounds / resolution; it would need resampling)")
        return diffusivity.values
    if isinstance(diffusivity, _math.Tensor) and diffusivity.shape.spatial.rank:
        return diffusivity
    return None


def _implicit_varying(field, k_values, dt, solve, stock, stock_args):
    """diffuse.implicit with a varying diffusivity, fast path for a scalar CenteredGrid (its values' channel-free shape), Solve('CG')."""
    try:
        if field.is_staggered:
            raise NotEligible("StaggeredGrid with a varying diffusivity (the reference raises NotImplementedError, diffuse.py:137-138)")
        dt = _number(dt)
        solve = solve.with_defaults('solve')
        if solve.method != 'CG' or solve.preconditioner is not None:
            raise NotEligible(f"solver '{solve.method}' / preconditioner {solve.preconditioner} (fast path: Solve('CG'))")
        dims, res, dx = _grid_info(field)
        x0 = solve.x0.values if isinstance(solve.x0, _Field) else None
        if solve.x0 is not None and x0 is None:
            raise NotEligible("x0 that is not a Field")
        values, info = _adapter.diffuse_implicit_varying(field.values, field.extrapolation, dx, dims, res, k_values, dt,
                                                         rel_tol=float(solve.rel_tol), abs_tol=float(solve.abs_tol),
                                                         max_iterations=int(_math.max(solve.max_iterations)), x0=x0)
    except (NotEligible, TypeError, ValueError) as why:
        return _fall('diffuse.implicit', why, stock, *stock_args)
    out = field.with_values(values)
    _report(solve, info, out)
    return out


def _clone(module, **replacements):
    clone = _types.ModuleType(module.__name__, module.__doc__)
    clone.__dict__.update({k: v for k, v in module.__dict__.items() if not k.startswith('__')})
    clone.__dict__.update(replacements)
    return clone


fluid = _clone(_fluid, make_incompressible=make_incompressible)
advect = _clone(_advect, semi_lagrangian=semi_lagrangian, mac_cormack=mac_cormack,
                advect=lambda field, velocity, dt, integrator=_advect.euler: (semi_lagrangian(field, velocity, dt, integrator)
                                                                             if isinstance(field, _Field) and field.is_grid else _advect.advect(field, velocity, dt, integrator)))
field = _clone(_field, laplace=laplace, divergence=divergence)
diffuse = _clone(_diffuse, implicit=implicit)
