"""
`from phiflow_b200.flow import *`  --  the reference's user-facing names for the incompressible-fluid hot path
(the surface `from phi.flow import *` gives a grid-fluid notebook: phi/flow.py:13-28), backed by the CUDA kernels.

Mirrored (same names, argument meaning and error behaviour; reference file:line in each docstring):
    Box, Sphere, union, geom.infinite_cylinder, CenteredGrid, StaggeredGrid, extrapolation (ZERO, ONE, PERIODIC, ZERO_GRADIENT, BOUNDARY, combine_sides),
    Solve, SolveTape, NotConverged, Diverged, field.{divergence, laplace, spatial_gradient}, resample,
    advect.{semi_lagrangian, mac_cormack, advect}, diffuse.{explicit, implicit}, fluid.{make_incompressible, incompressible_step},
    write / read (field.write / field.read: the reference's .npz field files, see field_io.py).
Fields hold device tensors in the library layout (DESIGN.md section 2); `.numpy()` returns the reference's (x, y[, z]) arrays.
Anything outside the fast path raises NotImplementedError (where the reference-side façade would fall through to stock
PhiFlow, INTEGRATION.md section 2).  No CPU fallback.
"""
import numbers
from builtins import range as builtins_range
from types import SimpleNamespace
from typing import Sequence

import numpy as np
import torch

from . import _ops as ops
from . import field_io
from . import scene as _scene

__all__ = ['Scene', 'vec', 'batch', 'iterate', 'jit_compile', 'Box', 'Sphere', 'union', 'geom', 'CenteredGrid', 'StaggeredGrid', 'extrapolation', 'ZERO', 'ONE', 'PERIODIC', 'ZERO_GRADIENT',
           'BOUNDARY', 'combine_sides', 'Solve', 'SolveTape', 'NotConverged', 'Diverged', 'ConvergenceException', 'field',
           'resample', 'advect', 'diffuse', 'fluid', 'math', 'write', 'read']

AXES = 'xyz'


# ----------------------------------------------------------------------------------------------------------------------
# extrapolation  (PhiML/phiml/math/extrapolation.py)
# ----------------------------------------------------------------------------------------------------------------------
class Extrapolation:
    """Per-side boundary: 'periodic', 'zg' or a constant (number, or tuple = one constant per vector component)."""

    def __init__(self, default=None, sides=None):
        self.default, self.sides = default, dict(sides or {})

    def side(self, axis: str, upper: bool):
        return self.sides.get((axis, upper), self.default)

    def spec(self, axes: Sequence[str], component: int = None):
        """ops-level spec for a scalar array (component selects the entry of vector constants)."""
        def conv(s):
            if isinstance(s, (tuple, list)):
                return float(s[component if component is not None else 0])
            return s if isinstance(s, str) else float(s)
        return tuple((conv(self.side(a, False)), conv(self.side(a, True))) for a in axes)

    def vspec(self, axes):
        per = [self.spec(axes, c) for c in range(len(axes))]
        return per[0] if all(p == per[0] for p in per) else per

    def valid_outer_faces(self, axis: str):
        """extrapolation.py:57-62"""
        lo, hi = self.side(axis, False), self.side(axis, True)
        return (lo in ('zg', 'periodic')), (hi == 'zg')

    @property
    def is_flexible(self):
        """extrapolation.py:288, 565, 665, 1288"""
        kinds = [self.default] + list(self.sides.values())
        return any(k == 'zg' for k in kinds)

    def __eq__(self, other):
        return isinstance(other, Extrapolation) and self.default == other.default and self.sides == other.sides

    def __hash__(self):
        return hash((str(self.default), tuple(sorted((k, str(v)) for k, v in self.sides.items()))))

    def __repr__(self):
        return f"Extrapolation({self.default}, {self.sides})"


def vec(**components):
    """phiml.math.vec(x=1, y=0) as this mirror spells vectors: a tuple in axis order (boundary constants, buoyancy factors)."""
    assert tuple(components) == tuple(AXES[:len(components)]), f"components must be {AXES[:len(components)]} in order"
    return tuple(float(v) for v in components.values())


def ConstantExtrapolation(value):
    """extrapolation.py:247"""
    return Extrapolation(tuple(value) if isinstance(value, (tuple, list)) else float(value))


ZERO, ONE = ConstantExtrapolation(0.0), ConstantExtrapolation(1.0)
PERIODIC = Extrapolation('periodic')
ZERO_GRADIENT = BOUNDARY = Extrapolation('zg')


def combine_sides(**by_axis):
    """extrapolation.combine_sides (extrapolation.py:1209): combine_sides(x=BOUNDARY, y=(ZERO, BOUNDARY))."""
    sides = {}
    for axis, ext in by_axis.items():
        lo, hi = ext if isinstance(ext, (tuple, list)) else (ext, ext)
        sides[(axis, False)] = _as_ext(lo).default
        sides[(axis, True)] = _as_ext(hi).default
    return Extrapolation(None, sides)


def _as_ext(b) -> Extrapolation:
    if isinstance(b, Extrapolation):
        return b
    if isinstance(b, dict):                       # {'x': 0, 'y-': 0, 'y+': ZERO_GRADIENT}
        sides = {}
        for k, v in b.items():
            v = _as_ext(v).default
            if k[-1] in '+-':
                sides[(k[:-1], k[-1] == '+')] = v
            else:
                sides[(k, False)] = sides[(k, True)] = v
        return Extrapolation(None, sides)
    return ConstantExtrapolation(b)


extrapolation = SimpleNamespace(ZERO=ZERO, ONE=ONE, PERIODIC=PERIODIC, ZERO_GRADIENT=ZERO_GRADIENT, BOUNDARY=BOUNDARY,
                                combine_sides=combine_sides, ConstantExtrapolation=ConstantExtrapolation, Extrapolation=Extrapolation)


# ----------------------------------------------------------------------------------------------------------------------
# geometry  (phi/geom)
# ----------------------------------------------------------------------------------------------------------------------
class Box:
    """Box(x=100, y=100) or Box(x=(1, 3), y=(0, 1))  (phi/geom/_box.py)."""

    def __init__(self, **dims):
        self.names = tuple(dims)
        self.lower = {k: float(v[0]) if isinstance(v, (tuple, list)) else 0.0 for k, v in dims.items()}
        self.upper = {k: float(v[1]) if isinstance(v, (tuple, list)) else float(v) for k, v in dims.items()}

    def lies_inside(self, pts):
        ok = np.ones(pts.shape[:-1], bool)
        for i, k in enumerate(self.names):
            ok &= (pts[..., i] >= self.lower[k]) & (pts[..., i] <= self.upper[k])
        return ok

    def signed_distance(self, pts):
        """Box.approximate_signed_distance (phi/geom/_box.py:217-236): signed L-infinity distance to the nearest side."""
        d = None
        for i, k in enumerate(self.names):
            c, h = 0.5 * (self.lower[k] + self.upper[k]), 0.5 * (self.upper[k] - self.lower[k])
            di = np.abs(pts[..., i] - np.float32(c)) - np.float32(h)
            d = di if d is None else np.maximum(d, di)
        return d.astype(np.float32)


class Sphere:
    """Sphere(x=50, y=9.5, radius=5)  (phi/geom/_sphere.py)."""

    def __init__(self, radius, **center):
        self.names, self.center, self.radius = tuple(center), tuple(float(v) for v in center.values()), float(radius)

    def lies_inside(self, pts):
        return np.sum((pts - np.asarray(self.center, np.float32)) ** 2, -1) <= self.radius ** 2

    def signed_distance(self, pts):
        """Sphere.approximate_signed_distance (phi/geom/_sphere.py:107-120)."""
        d = np.sqrt(np.maximum(np.sum((pts - np.asarray(self.center, np.float32)) ** 2, -1, dtype=np.float32), np.float32(1e-6)))
        return (d - np.float32(self.radius)).astype(np.float32)

    def soft_mask(self, pts, cell_radius):
        """Geometry.approximate_fraction_inside (phi/geom/_geom.py:278-308) with Sphere.approximate_signed_distance
        (phi/geom/_sphere.py:107-120, vec_length eps=1e-3)."""
        d = np.sqrt(np.maximum(np.sum((pts - np.asarray(self.center, np.float32)) ** 2, -1, dtype=np.float32), np.float32(1e-6)))
        return np.clip(np.float32(0.5) - (d - np.float32(self.radius)) / np.float32(cell_radius), 0, 1).astype(np.float32)


class InfiniteCylinder:
    """geom.infinite_cylinder(x=20, y=50, radius=10, inf_dim='z')  (phi/geom/_embed.py:139-158): a Sphere over the named axes,
    embedded along `inf_dim`.  Points are projected onto the sphere's axes (_EmbeddedGeometry._down_project, _embed.py:41-47)."""

    def __init__(self, sphere: Sphere, inf_dim: str):
        self.sphere, self.inf_dim = sphere, inf_dim

    def _down_project(self, pts):
        return pts[..., [AXES.index(n) for n in self.sphere.names]]

    def lies_inside(self, pts):
        return self.sphere.lies_inside(self._down_project(pts))

    def signed_distance(self, pts):
        return self.sphere.signed_distance(self._down_project(pts))


def infinite_cylinder(center=None, radius=None, inf_dim: str = None, **center_):
    """geom.infinite_cylinder (phi/geom/_embed.py:139-158) with the centre as keyword arguments over the other axes."""
    _require(center is None and isinstance(inf_dim, str) and inf_dim in AXES and inf_dim not in center_ and radius is not None,
             "infinite_cylinder other than infinite_cylinder(x=..., y=..., radius=..., inf_dim='z')")
    _require(all(n in AXES for n in center_), f"cylinder axes {tuple(center_)}")
    return InfiniteCylinder(Sphere(radius, **center_), inf_dim)


class Union:
    """union(Box(...), Box(...))  (phi/geom/_geom_ops.py:297-320): a point lies inside when it lies inside any member."""

    def __init__(self, *geometries):
        self.geometries = tuple(geometries)

    def lies_inside(self, pts):
        ok = np.zeros(pts.shape[:-1], bool)
        for g in self.geometries:
            ok |= g.lies_inside(pts)
        return ok

    def signed_distance(self, pts):
        """Union.approximate_signed_distance (phi/geom/_geom_ops.py:100-102): the minimum over the members, so a union obstacle's face
        factors are 1 - max of the members' fractions (Fluid_Logo.ipynb's eight touching boxes), not the product of separate obstacles."""
        return np.minimum.reduce([g.signed_distance(pts) for g in self.geometries]).astype(np.float32)


def union(*geometries):
    """geom.union (phi/geom/_geom_ops.py:297-320): union(Box(x=(0, 10), y=(2, 3)), Box(x=(4.5, 5.5), y=(1, 4))) as Heat_Flow.ipynb builds its
    bars.  Usable where a hard geometry mask is sampled (CenteredGrid(values=union(...)))."""
    flat = []
    for g in (geometries[0] if len(geometries) == 1 and isinstance(geometries[0], (list, tuple)) else geometries):
        _require(isinstance(g, (Box, Sphere, Union)), f"union of {type(g).__name__}")
        flat += list(g.geometries) if isinstance(g, Union) else [g]
    return Union(*flat)


geom = SimpleNamespace(Box=Box, Sphere=Sphere, union=union, infinite_cylinder=infinite_cylinder)


# ----------------------------------------------------------------------------------------------------------------------
# math: Solve and friends  (PhiML/phiml/math/_optimize.py)
# ----------------------------------------------------------------------------------------------------------------------
class ConvergenceException(RuntimeError):
    def __init__(self, result):
        super().__init__(result.msg)
        self.result = result


class NotConverged(ConvergenceException):
    """_optimize.py: raised when max_iterations is reached"""


class Diverged(ConvergenceException):
    """_optimize.py: raised when the residual grows (stop_on_l2, _linalg.py:29-36)"""


class Solve:
    """phiml.math.Solve (_optimize.py:25-41): method, rel_tol, abs_tol, x0, max_iterations, suppress."""

    def __init__(self, method='auto', rel_tol=None, abs_tol=None, x0=None, max_iterations=1000, suppress=(), matrix_offset=0.0):
        self.method, self.x0, self.max_iterations, self.suppress = method or 'auto', x0, int(max_iterations), tuple(suppress)
        self.rel_tol = 1e-5 if rel_tol is None else float(rel_tol)        # _default_tolerance, fp32 (_optimize.py:130-136)
        self.abs_tol = 1e-5 if abs_tol is None else float(abs_tol)
        self.matrix_offset = matrix_offset                                # see DESIGN.md section 3; 0 = plain CG


class SolveInfo:
    def __init__(self, solve, raw):
        self.solve = solve
        self.iterations, self.converged, self.diverged = raw['iterations'].copy(), raw['converged'].astype(bool), raw['diverged'].astype(bool)
        self.residual_sq, self.tol_sq = raw['residual_sq'].copy(), raw['tol_sq'].copy()
        self.msg = f"CG: iterations={self.iterations.tolist()} converged={self.converged.tolist()} diverged={self.diverged.tolist()}"


_TAPES = []


class SolveTape:
    """with math.SolveTape() as solves: ...; solves[solve].iterations  (_optimize.py:268-334)."""

    def __enter__(self):
        self.records = []
        _TAPES.append(self)
        return self

    def __exit__(self, *exc):
        _TAPES.remove(self)

    def __getitem__(self, solve):
        if isinstance(solve, int):                 # tape[i] / tape[-1]: records in the order the solves ran (_optimize.py:300-318)
            return self.records[solve][1]
        for s, info in self.records:
            if s is solve:
                return info
        raise KeyError(solve)

    def __len__(self):
        return len(self.records)


math = SimpleNamespace(Solve=Solve, SolveTape=SolveTape, NotConverged=NotConverged, Diverged=Diverged,
                       ConvergenceException=ConvergenceException, extrapolation=extrapolation)


def jit_compile(f=None, **_):
    """math.jit_compile (PhiML/phiml/math/_functional.py): the identity here - every call already is a pre-compiled CUDA kernel behind
    the C ABI, and ctypes launches must not be traced (SURVEY.md Appendix C)."""
    return f if f is not None else (lambda g: g)


def batch(**dims):
    """batch(time=300) as `iterate` uses it: the name and length of the trajectory dimension."""
    assert len(dims) == 1, "one trajectory dimension"
    return dict(dims)


def iterate(f, iterations, *x0, f_kwargs: dict = None, range=range, substeps: int = 1, **f_kwargs_):
    """math.iterate (PhiML/phiml/math/_functional.py:1241-1300): calls `x = f(*x, **kwargs)` repeatedly.  `iterations` = int -> the final
    state; = batch(time=N) -> one trajectory per state variable, as a LIST of N + 1 entries starting with the initial state (the
    reference stacks them along the batch dim; stacked device trajectories of 3-D runs do not fit, lists of Fields do the same job).
    `substeps` calls of f separate two recorded entries."""
    kwargs = dict(f_kwargs or {}, **f_kwargs_)
    x = tuple(x0)
    record = isinstance(iterations, dict)
    n = int(next(iter(iterations.values()))) if record else int(iterations)
    trj = [[xi] for xi in x] if record else None
    for _ in range(n):
        for _ in builtins_range(substeps):
            out = f(*x[:len(x0)], **kwargs)
            x = tuple(out) if isinstance(out, (tuple, list)) else (out,)
        if record:
            for t, xi in zip(trj, x):
                t.append(xi)
    result = tuple(trj) if record else x
    return result if len(result) > 1 else result[0]


# ----------------------------------------------------------------------------------------------------------------------
# fields  (phi/field/_field.py, _grid.py)
# ----------------------------------------------------------------------------------------------------------------------
_DOMAINS = {}
_DEVICE = 'cuda'


def set_device(device):
    """Device that newly created fields live on.  'cpu' fields are data containers only (construction, `.numpy()`, file IO);
    every kernel still requires a CUDA device - there is no CPU fallback."""
    global _DEVICE
    _DEVICE = str(device)


def _domain(res, dx, batch, vspec):
    upper = tuple(ops.stored_faces(vspec, a)[1] for a in range(len(res))) if vspec is not None else (False,) * len(res)
    key = (tuple(res), tuple(dx), batch, upper, _DEVICE)
    if key not in _DOMAINS:
        _DOMAINS[key] = ops.Domain(res, dx, batch, vbc=vspec, device=_DEVICE)
    return _DOMAINS[key]


class _Grid:
    def _geometry(self, bounds, resolution, batch):
        self.axes = tuple(resolution)
        assert self.axes == tuple(AXES[:len(self.axes)]), f"spatial dims must be {AXES[:len(self.axes)]} in order, got {self.axes}"
        self.res = tuple(int(resolution[a]) for a in self.axes)
        self.bounds = bounds if bounds is not None else Box(**{a: n for a, n in zip(self.axes, self.res)})
        self.lower = tuple(self.bounds.lower[a] for a in self.axes)
        self.upper = tuple(self.bounds.upper[a] for a in self.axes)
        self.dx = tuple((u - l) / n for l, u, n in zip(self.lower, self.upper, self.res))
        self.batch = batch

    @property
    def extrapolation(self):
        return self.boundary

    def _same_grid(self, other):
        return self.res == other.res and self.lower == other.lower and self.upper == other.upper and self.batch == other.batch


class CenteredGrid(_Grid):
    """CenteredGrid(values, boundary, bounds, x=..., y=...)  (phi/field/_grid.py:21-86).
    values: number, numpy array in (x, y[, z]) order (optional leading batch axis), or a geometry (Box / Sphere: hard mask)."""

    def __init__(self, values=0., boundary=ZERO, bounds=None, batch=1, _data=None, _scale=None, **resolution):
        self._geometry(bounds, resolution, batch)
        self.boundary = _as_ext(boundary)
        self.dom = _domain(self.res, self.dx, batch, None)
        self.vector_scale = _scale                       # s * (0, 0.1): a centred vector field that is a scalar times constants
        if _data is not None:
            self.data = _data
        elif isinstance(values, (Box, Sphere, Union)):
            self.data = self.dom.centered_from_numpy(values.lies_inside(self.points()).astype(np.float32))
        elif np.isscalar(values):
            self.data = self.dom.alloc_centered()
            if values != 0:
                self.data += float(values)
        else:
            self.data = self.dom.centered_from_numpy(np.asarray(values, np.float32))

    def points(self):
        axes = [(np.linspace(0.5 / n, 1 - 0.5 / n, n).astype(np.float32) * np.float32(u - l) + np.float32(l)) for l, u, n in zip(self.lower, self.upper, self.res)]
        return np.stack(np.meshgrid(*axes, indexing='ij'), -1).astype(np.float32)

    @property
    def spec(self):
        return self.boundary.spec(self.axes)

    def with_values(self, data):
        return CenteredGrid(boundary=self.boundary, bounds=self.bounds, batch=self.batch, _data=data, **dict(zip(self.axes, self.res)))

    def with_extrapolation(self, boundary):
        return CenteredGrid(boundary=boundary, bounds=self.bounds, batch=self.batch, _data=self.data, **dict(zip(self.axes, self.res)))

    with_boundary = with_extrapolation

    def numpy(self):
        return self.dom.centered_to_numpy(self.data)

    def _valid(self):
        idx = (slice(None),) + tuple(slice(0, n) for n in reversed(self.res))
        return self.data[idx]

    def __add__(self, other):
        if isinstance(other, CenteredGrid):
            assert self._same_grid(other)
            return self.with_values(self.data + other.data)
        return self.with_values(self.data + float(other))

    __radd__ = __add__

    def __sub__(self, other):
        return self + (other * -1.0)

    def __mul__(self, other):
        if isinstance(other, (tuple, list)):             # scalar field times a constant vector, e.g. s * (0, 0.1)
            g = self.with_values(self.data)
            g.vector_scale = tuple(float(o) for o in other)
            return g
        if isinstance(other, CenteredGrid):
            return self.with_values(self.data * other.data)
        return self.with_values(self.data * float(other))

    __rmul__ = __mul__


class StaggeredGrid(_Grid):
    """StaggeredGrid(values, boundary, bounds, x=..., y=...)  (phi/field/_grid.py:89-176).
    values: number, tuple of per-component constants, list of per-component numpy arrays shaped as the reference stores
    them (n-1 / n / n+1 faces, tests/commit/field/test__grid.py:25-37), or a geometry (hard mask sampled at face centres)."""

    def __init__(self, values=0., boundary=ZERO, bounds=None, batch=1, _data=None, **resolution):
        self._geometry(bounds, resolution, batch)
        self.boundary = _as_ext(boundary)
        self.vspec = self.boundary.vspec(self.axes)
        self.dom = _domain(self.res, self.dx, batch, self.vspec)
        d = len(self.res)
        if _data is not None:
            self.data = _data
            return
        shapes, _ = self.dom.face_shapes(self.vspec)
        if isinstance(values, (Box, Sphere)):
            comps = [values.lies_inside(self.face_points(c)).astype(np.float32) for c in range(d)]
        elif np.isscalar(values):
            comps = [np.full(shapes[c], values, np.float32) for c in range(d)]
        elif isinstance(values, tuple) and all(np.isscalar(v) for v in values):
            comps = [np.full(shapes[c], values[c], np.float32) for c in range(d)]
        else:
            comps = [np.asarray(v, np.float32) for v in values]
        self.data = self.dom.faces_from_numpy(comps, self.vspec)

    def face_points(self, c):
        """Centres of the stored faces of component c (UniformGrid.stagger, phi/geom/_grid.py:204-209)."""
        lo_st, hi_st = self.boundary.valid_outer_faces(self.axes[c])
        axes = []
        for a, (l, u, n) in enumerate(zip(self.lower, self.upper, self.res)):
            if a == c:
                first, count = (0 if lo_st else 1), n - 1 + int(lo_st) + int(hi_st)
                axes.append((np.float32(l) + (np.arange(count, dtype=np.float32) + first) * np.float32((u - l) / n)).astype(np.float32))
            else:
                axes.append(np.linspace(0.5 / n, 1 - 0.5 / n, n).astype(np.float32) * np.float32(u - l) + np.float32(l))
        return np.stack(np.meshgrid(*axes, indexing='ij'), -1).astype(np.float32)

    def with_values(self, data):
        return StaggeredGrid(boundary=self.boundary, bounds=self.bounds, batch=self.batch, _data=data, **dict(zip(self.axes, self.res)))

    def with_extrapolation(self, boundary):
        boundary = _as_ext(boundary)
        if boundary == self.boundary:
            return self
        # different stored faces: go through the reference layout (tests/commit/field/test__grid.py:85-94)
        new = StaggeredGrid(0, boundary, self.bounds, self.batch, **dict(zip(self.axes, self.res)))
        old = self.numpy()
        comps = []
        for c, a in enumerate(self.axes):
            lo0, hi0 = self.boundary.valid_outer_faces(a)
            lo1, hi1 = boundary.valid_outer_faces(a)
            full = np.zeros(old[c].shape[:old[c].ndim - len(self.res)] + tuple(n + (1 if i == c else 0) for i, n in enumerate(self.res)), np.float32)
            sl = [slice(None)] * full.ndim
            ax = full.ndim - len(self.res) + c
            sl[ax] = slice(0 if lo0 else 1, self.res[c] + 1 if hi0 else self.res[c])
            full[tuple(sl)] = old[c]
            sl[ax] = slice(0 if lo1 else 1, self.res[c] + 1 if hi1 else self.res[c])
            comps.append(full[tuple(sl)])
        new.data = new.dom.faces_from_numpy(comps, new.vspec)
        return new

    with_boundary = with_extrapolation

    def numpy(self):
        """List of per-component arrays in the reference's shapes, (x, y[, z]) order."""
        return self.dom.faces_to_numpy(self.data, self.vspec)

    def __getitem__(self, axis):
        c = self.axes.index(axis)
        return SimpleNamespace(numpy=lambda: self.numpy()[c], values=SimpleNamespace(numpy=lambda order=None: self.numpy()[c]))

    def _binary(self, other, fn):
        if isinstance(other, StaggeredGrid):
            assert self._same_grid(other) and other.boundary == self.boundary, "staggered operands must share grid and boundary"
            return self.with_values([fn(a, b) for a, b in zip(self.data, other.data)])
        if isinstance(other, (tuple, list)):
            return self.with_values([fn(a, float(o)) for a, o in zip(self.data, other)])
        return self.with_values([fn(a, float(other)) for a in self.data])

    def __add__(self, other):
        return self._binary(other, lambda a, b: a + b)

    __radd__ = __add__

    def __sub__(self, other):
        return self._binary(other, lambda a, b: a - b)

    def __mul__(self, other):
        return self._binary(other, lambda a, b: a * b)

    __rmul__ = __mul__


# ----------------------------------------------------------------------------------------------------------------------
# field functions  (phi/field/_field_math.py, _resample.py)
# ----------------------------------------------------------------------------------------------------------------------
def _require(cond, what):
    if not cond:
        raise NotImplementedError(f"{what} is outside the phiflow_b200 fast path (use stock PhiFlow)")


def divergence(v: StaggeredGrid, order=2) -> CenteredGrid:
    """field.divergence (phi/field/_field_math.py:589-626); result boundary = spatial gradient of the velocity boundary."""
    _require(isinstance(v, StaggeredGrid) and order == 2, "divergence of non-staggered / higher-order fields")
    out = ops.divergence(v.dom, v.vspec, v.data)
    return CenteredGrid(boundary=_gradient_boundary(v.boundary), bounds=v.bounds, batch=v.batch, _data=out, **dict(zip(v.axes, v.res)))


def _gradient_boundary(b: Extrapolation) -> Extrapolation:
    conv = lambda s: s if isinstance(s, str) else 0.0          # spatial_gradient of a constant is ZERO
    return Extrapolation(conv(b.default) if b.default is not None else None, {k: conv(s) for k, s in b.sides.items()})


def laplace(u: CenteredGrid, order=2) -> CenteredGrid:
    """field.laplace (phi/field/_field_math.py:46-145), ghost cells from u's boundary."""
    _require(isinstance(u, CenteredGrid) and order == 2, "laplace of non-centred / higher-order fields")
    out = ops.laplace(u.dom, u.spec, u.data)
    return CenteredGrid(boundary=_gradient_boundary(_gradient_boundary(u.boundary)), bounds=u.bounds, batch=u.batch, _data=out, **dict(zip(u.axes, u.res)))


def _pressure_boundary(vb: Extrapolation) -> Extrapolation:
    """fluid._pressure_extrapolation (phi/physics/fluid.py:264-274)."""
    conv = lambda s: 'periodic' if s == 'periodic' else (0.0 if s == 'zg' else 'zg')
    return Extrapolation(conv(vb.default) if vb.default is not None else None, {k: conv(s) for k, s in vb.sides.items()})


def spatial_gradient(p: CenteredGrid, boundary=None, at='face', order=2) -> StaggeredGrid:
    """field.spatial_gradient(p, boundary, at='face') (phi/field/_field_math.py:148-236): (upper - lower)/dx on the faces that
    `boundary` stores.  Fast path: p's boundary must be the pressure boundary belonging to `boundary` (what
    make_incompressible uses, fluid.py:158)."""
    boundary = _as_ext(boundary)
    _require(at == 'face' and order == 2, "spatial_gradient other than at='face', order 2")
    _require(_pressure_boundary(boundary) == p.boundary, "spatial_gradient with an unrelated field boundary")
    g = StaggeredGrid(0, boundary, p.bounds, p.batch, **dict(zip(p.axes, p.res)))
    ops.grad_sub(g.dom, g.vspec, g.data, p.data)
    return g * -1.0


def resample(value, to, soft=False, **_):
    """resample(value, to) for the two cases of the notebook step (phi/field/_resample.py:13-63):
    geometry -> CenteredGrid (soft mask, :192-210) and (CenteredGrid * constant vector) -> StaggeredGrid (:272-276)."""
    if isinstance(value, Sphere) and isinstance(to, CenteredGrid):
        if soft:
            cell_r = float(np.sqrt(sum((h * 0.5) ** 2 for h in to.dx)))
            return to.with_values(to.dom.centered_from_numpy(value.soft_mask(to.points(), cell_r)))
        return to.with_values(to.dom.centered_from_numpy(value.lies_inside(to.points()).astype(np.float32)))
    if isinstance(value, CenteredGrid) and isinstance(to, StaggeredGrid) and value.vector_scale is not None:
        _require(value.res == to.res, "resampling between different resolutions")
        out = StaggeredGrid(0, to.boundary, to.bounds, to.batch, **dict(zip(to.axes, to.res)))
        ops.add_buoyancy(out.dom, out.vspec, value.spec, value.data, value.vector_scale, 1.0, out.data)
        return out
    raise NotImplementedError("resample: only Sphere->CenteredGrid and (scalar*vector)->StaggeredGrid are on the fast path")


# ----------------------------------------------------------------------------------------------------------------------
# file IO  (phi/field/_field_io.py)
# ----------------------------------------------------------------------------------------------------------------------
def write(fld, file: str):
    """field.write(field, file) (phi/field/_field_io.py:13-69): one compressed .npz per field with the reference's keys;
    a staggered grid is stored as its uniform `staggered_tensor()` ((n+1) points per axis, trailing `vector` dim)."""
    _require(isinstance(fld, (CenteredGrid, StaggeredGrid)) and isinstance(file, str), "writing anything but one grid to one file")
    d = len(fld.axes)
    ext = field_io.extrapolation_to_dict(fld.boundary.default, fld.boundary.sides, fld.axes)
    lead_names = ('batch',) if fld.batch > 1 else ()
    lead_types = ('batch',) if fld.batch > 1 else ()
    lower, upper = [fld.lower[i] for i in range(d)], [fld.upper[i] for i in range(d)]
    if isinstance(fld, CenteredGrid):
        field_io.write_single_field(file, 'CenteredGrid', fld.numpy(), lead_names + fld.axes, lead_types + ('spatial',) * d,
                                    (None,) * (len(lead_names) + d), lower, upper, fld.axes, ext)
    else:
        data = field_io.staggered_tensor(fld.numpy(), lambda ax: (fld.boundary.side(fld.axes[ax], False), fld.boundary.side(fld.axes[ax], True)), d)
        field_io.write_single_field(file, 'StaggeredGrid', data, lead_names + fld.axes + ('vector',), lead_types + ('spatial',) * d + ('channel',),
                                    (None,) * (len(lead_names) + d) + (fld.axes,), lower, upper, fld.axes, ext)


def read(file: str):
    """field.read(file) (phi/field/_field_io.py:72-127): restores a CenteredGrid / StaggeredGrid written by `write` or by stock
    PhiFlow (scalar centred grids and staggered grids whose vector components match the spatial dims)."""
    st = field_io.read_single_field(file)
    names, types = st['dim_names'], st['dim_types']
    axes = tuple(n for n, t in zip(names, types) if t == 'spatial')
    lead = tuple(n for n, t in zip(names, types) if t == 'batch')
    _require(len(lead) <= 1 and names[:len(lead)] == lead and names[len(lead):len(lead) + len(axes)] == axes, "batch dims after spatial dims")
    default, sides = field_io.extrapolation_from_dict(st['extrapolation'])
    boundary = Extrapolation(default, sides)
    data = np.asarray(st['data'], np.float32)
    batch = data.shape[0] if lead else 1
    bounds = Box(**{a: (st['lower'][a], st['upper'][a]) for a in axes})
    if st['field_type'] == 'CenteredGrid':
        _require(data.ndim == len(lead) + len(axes), "centred grids with channel dims")
        res = dict(zip(axes, data.shape[len(lead):]))
        return CenteredGrid(data, boundary, bounds, batch, **res)
    _require(names[-1] == 'vector' and data.shape[-1] == len(axes), "staggered tensors whose components are not the spatial dims")
    comps = field_io.unstack_staggered_tensor(data, lambda ax: (boundary.side(axes[ax], False), boundary.side(axes[ax], True)), len(axes))
    res = {a: n - 1 for a, n in zip(axes, data.shape[len(lead):len(lead) + len(axes)])}
    return StaggeredGrid(comps, boundary, bounds, batch, **res)


field = SimpleNamespace(divergence=divergence, laplace=laplace, spatial_gradient=spatial_gradient, resample=resample,
                        CenteredGrid=CenteredGrid, StaggeredGrid=StaggeredGrid, write=write, read=read)


# ----------------------------------------------------------------------------------------------------------------------
# advect  (phi/physics/advect.py)
# ----------------------------------------------------------------------------------------------------------------------
class Scene(_scene.Scene):
    """phi.field.Scene for this package's grids (phi/field/_scene.py:52-426): trajectories as sim_xxxxxx/<name>_<frame>.npz."""

    def __init__(self, path, writer=None, reader=None):
        super().__init__(path, writer or write, reader or read)

    @staticmethod
    def create(parent_directory, name='sim', copy_calling_script=False):
        s = _scene.Scene.create(parent_directory, name, copy_calling_script)
        return Scene(s.path)

    @staticmethod
    def at(directory, id=None):
        return Scene(_scene.Scene.at(directory, id).path)

    @staticmethod
    def list(parent_directory, name='sim'):
        return tuple(Scene(s.path) for s in _scene.Scene.list(parent_directory, name))


def _check_velocity(fld, velocity):
    _require(isinstance(velocity, StaggeredGrid), "advection by a non-staggered velocity")
    _require(fld.res == velocity.res and fld.lower == velocity.lower and fld.upper == velocity.upper, "advection across different grids")


def semi_lagrangian(fld, velocity: StaggeredGrid, dt: float, integrator=None):
    """advect.semi_lagrangian (phi/physics/advect.py:156-179) with the euler integrator (:20-24)."""
    _require(integrator is None, "integrators other than euler")
    _check_velocity(fld, velocity)
    if isinstance(fld, CenteredGrid):
        return fld.with_values(ops.advect_centered(velocity.dom, velocity.vspec, velocity.data, fld.spec, fld.data, float(dt)))
    _require(fld.boundary == velocity.boundary or [ops.stored_faces(fld.vspec, a) for a in range(len(fld.res))] ==
             [ops.stored_faces(velocity.vspec, a) for a in range(len(fld.res))], "staggered fields with different stored faces")
    return fld.with_values(ops.advect_staggered(velocity.dom, velocity.vspec, velocity.data, fld.vspec, fld.data, float(dt)))


def mac_cormack(fld, velocity: StaggeredGrid, dt: float, correction_strength=1.0, integrator=None):
    """advect.mac_cormack (phi/physics/advect.py:182-215); centred fields only on the fast path."""
    _require(integrator is None and isinstance(fld, CenteredGrid), "mac_cormack of staggered fields / other integrators")
    _check_velocity(fld, velocity)
    return fld.with_values(ops.mac_cormack_centered(velocity.dom, velocity.vspec, velocity.data, fld.spec, fld.data, float(dt), correction_strength))


advect = SimpleNamespace(semi_lagrangian=semi_lagrangian, mac_cormack=mac_cormack, advect=semi_lagrangian)


# ----------------------------------------------------------------------------------------------------------------------
# diffuse  (phi/physics/diffuse.py)
# ----------------------------------------------------------------------------------------------------------------------
def explicit(fld, diffusivity: float, dt: float, substeps: int = 1):
    """diffuse.explicit (phi/physics/diffuse.py:13-60): substeps of  u += (dt/substeps) * diffusivity * laplace(u); for a
    StaggeredGrid every component is diffused with its own boundary (Lid_Driven_Cavity.ipynb, Variable_Boundaries.ipynb)."""
    amount = float(diffusivity) * float(dt) / substeps
    if isinstance(fld, StaggeredGrid):
        return fld.with_values(ops.laplace_axpy_faces(fld.dom, fld.vspec, fld.data, amount, substeps))
    _require(isinstance(fld, CenteredGrid), "explicit diffusion of this field type")
    data = fld.data
    for _ in range(substeps):
        data = ops.laplace_axpy(fld.dom, fld.spec, data, amount)
    return fld.with_values(data)


def implicit(fld, diffusivity: float, dt: float, solve: Solve = None):
    """diffuse.implicit (phi/physics/diffuse.py:63-95): solves  x - diffusivity * dt * laplace(x) = fld  with CG (Solve('CG'), x0 = fld
    unless solve.x0 is given), the constant boundary values entering as the bias of the affine system (_optimize.py:622, 645).
    A scalar CenteredGrid with any boundary, or a PERIODIC StaggeredGrid whose components are solved as separate systems, as the
    reference does (one record per batch entry and component, entry b * dim + c).  Returns a new field; SolveTape records,
    NotConverged and Diverged as for make_incompressible.
    A CenteredGrid diffusivity on the same grid (batch 1 or the field's) diffuses a scalar CenteredGrid with a spatially varying k
    (diffuse.py:129-141, Heat_Flow.ipynb): see _implicit_varying."""
    solve = solve or Solve('CG')
    plain = lambda v: isinstance(v, numbers.Real) and not isinstance(v, bool)
    if isinstance(diffusivity, CenteredGrid) and isinstance(fld, CenteredGrid):
        return _implicit_varying(fld, diffusivity, dt, solve)
    _require(plain(diffusivity) and plain(dt), "implicit diffusion with a Field / vector / per-batch diffusivity or dt")
    _require(solve.method == 'CG', f"solver '{solve.method}' for implicit diffusion")
    amount = float(diffusivity) * float(dt)
    if isinstance(fld, StaggeredGrid):
        # the reference supports only PERIODIC here; ZERO and BOUNDARY are "not yet supported" (tests/commit/physics/test_diffuse.py:25,28)
        _require(all(s == 'periodic' for a in fld.axes for s in (fld.boundary.side(a, False), fld.boundary.side(a, True))),
                 "implicit diffusion of a non-periodic StaggeredGrid")
        if solve.x0 is not None:
            _require(isinstance(solve.x0, StaggeredGrid) and solve.x0._same_grid(fld), "x0 on a different grid")
        data = ops.diffuse_implicit(fld.dom, fld.vspec, fld.data, amount, solve.rel_tol, solve.abs_tol, solve.max_iterations,
                                    x0=solve.x0.data if solve.x0 is not None else None)
        _finish_solve(fld.dom, solve, ops.read_results(fld.dom, len(fld.data)))
        return fld.with_values(data)
    _require(isinstance(fld, CenteredGrid) and fld.vector_scale is None, "implicit diffusion of this field type")
    if solve.x0 is not None:
        _require(isinstance(solve.x0, CenteredGrid) and solve.x0._same_grid(fld), "x0 on a different grid")
    data = ops.diffuse_implicit(fld.dom, fld.spec, fld.data, amount, solve.rel_tol, solve.abs_tol, solve.max_iterations,
                                x0=solve.x0.data if solve.x0 is not None else None)
    _finish_solve(fld.dom, solve)
    return fld.with_values(data)


def _implicit_varying(fld, k, dt, solve: Solve):
    """diffuse.implicit(fld, k, dt) with a CenteredGrid diffusivity k (phi/physics/diffuse.py:48-59, 90-95, 129-141): solves
    sharpen(x) = explicit(x, k, -dt) = fld with CG.  Every face takes min(-dt k_lo, -dt k_hi) - for dt > 0 the face MAXIMUM of k - and
    the coefficient ghosts follow fld's boundary, not k's own (amount.at(u), phi/field/_resample.py:56-63): a constant side with
    value c gives min(-dt k_edge, c).  k must lie on fld's grid (no resampling) with batch 1 or fld's batch."""
    _require(isinstance(dt, numbers.Real) and not isinstance(dt, bool), "implicit diffusion with a Field / vector / per-batch dt")
    _require(solve.method == 'CG', f"solver '{solve.method}' for implicit diffusion")
    _require(fld.vector_scale is None and k.vector_scale is None, "implicit diffusion of a vector field with a varying diffusivity")
    _require(k.res == fld.res and k.lower == fld.lower and k.upper == fld.upper,
             "a diffusivity on a different grid (it would need resampling)")
    _require(k.batch in (1, fld.batch), f"a diffusivity with batch {k.batch} for a field with batch {fld.batch}")
    if solve.x0 is not None:
        _require(isinstance(solve.x0, CenteredGrid) and solve.x0._same_grid(fld), "x0 on a different grid")
    data = ops.diffuse_implicit_varying(fld.dom, fld.spec, fld.data, k.data, float(dt), solve.rel_tol, solve.abs_tol, solve.max_iterations,
                                        x0=solve.x0.data if solve.x0 is not None else None)
    _finish_solve(fld.dom, solve)
    return fld.with_values(data)


diffuse = SimpleNamespace(explicit=explicit, implicit=implicit)


# ----------------------------------------------------------------------------------------------------------------------
# fluid  (phi/physics/fluid.py)
# ----------------------------------------------------------------------------------------------------------------------
def _cg_params(v: StaggeredGrid, solve: Solve):
    # Solver policy = the reference's: 'CG' is Shewchuk CG (the north-star solver); 'auto' (the default Solve()) and
    # 'CG-adaptive' run the Hestenes-Stiefel variant exactly as the vendored PhiML maps them (backend/_backend.py:1446-1447,
    # _linalg.py:93-128), tolerance relative to |rhs|^2, with and without obstacle masks.  CG-adaptive lives on the TMA ring
    # kernel only: on grids whose lines do not fit it, 'auto' and 'CG-adaptive' raise Unsupported.
    _require(solve.method in ('CG', 'auto', 'CG-adaptive'), f"solver '{solve.method}'")
    adaptive = solve.method in ('CG-adaptive', 'auto')
    return ops.cg_params(v.vspec, rtol=solve.rel_tol, atol=solve.abs_tol, max_iter=solve.max_iterations,
                         matrix_offset=0.0 if adaptive else solve.matrix_offset, method='CG-adaptive' if adaptive else 'CG')


def _finish_solve(dom, solve: Solve, raw=None):
    info = SolveInfo(solve, ops.read_results(dom) if raw is None else raw)
    for tape in _TAPES:
        tape.records.append((solve, info))
    if info.diverged.any() and Diverged not in solve.suppress:           # SolveInfo.convergence_check (_optimize.py:190-204)
        raise Diverged(info)
    if not info.converged.all() and NotConverged not in solve.suppress:
        raise NotConverged(info)
    return info


def _obstacle_masks(velocity: StaggeredGrid, obstacles):
    """Static obstacles (phi/physics/fluid.py:130-137, 212-240): returns (accessible centred mask, per-component face factors
    1 - resample(geometry, velocity, soft=True, balance=1)).  Geometry sampling is set-up work done on the host."""
    geoms = list(obstacles) if isinstance(obstacles, (tuple, list)) else [obstacles]
    _require(all(isinstance(o, (Box, Sphere, InfiniteCylinder, Union)) for o in geoms),
             "obstacles other than stationary Box / Sphere / infinite_cylinder / union geometries")
    centred = CenteredGrid(0, ZERO, velocity.bounds, velocity.batch, **dict(zip(velocity.axes, velocity.res)))
    pts = centred.points()
    inside = np.zeros(pts.shape[:-1], bool)
    for o in geoms:
        inside |= o.lies_inside(pts)
    accessible = velocity.dom.centered_from_numpy((~inside).astype(np.float32))
    radius = np.float32(np.sqrt(sum((h * 0.5) ** 2 for h in velocity.dx)))        # bounding radius of a (staggered) cell
    factors = []
    for c in range(len(velocity.res)):
        fpts = velocity.face_points(c)
        f = np.ones(fpts.shape[:-1], np.float32)
        for o in geoms:                                                          # approximate_fraction_inside, balance = 1
            f *= np.float32(1) - np.clip(np.float32(1) - o.signed_distance(fpts) / radius, 0, 1).astype(np.float32)
        factors.append(f)
    return accessible, velocity.dom.faces_from_numpy(factors, velocity.vspec)


def _geometry_key(o):
    """The parameters that decide a stationary geometry's masks (hashable)."""
    if isinstance(o, Box):
        return ('box', o.names, tuple(o.lower[k] for k in o.names), tuple(o.upper[k] for k in o.names))
    if isinstance(o, Sphere):
        return ('sphere', o.names, o.center, o.radius)
    if isinstance(o, InfiniteCylinder):
        return ('cylinder', _geometry_key(o.sphere), o.inf_dim)
    if isinstance(o, Union):
        return ('union',) + tuple(_geometry_key(g) for g in o.geometries)
    _require(False, "obstacles other than stationary Box / Sphere / infinite_cylinder / union geometries")


_MASKS = {}
_MASKS_KEPT = 8


def _obstacle_masks_cached(velocity: StaggeredGrid, obstacles):
    """_obstacle_masks memoised on the geometry parameters and the grid (resolution, bounds, batch, boundary, device): a step loop and
    make_incompressible with the same stationary obstacle rasterise it on the host once.  The masks are read-only device tensors."""
    geoms = list(obstacles) if isinstance(obstacles, (tuple, list)) else [obstacles]
    key = (tuple(_geometry_key(o) for o in geoms), velocity.res, velocity.lower, velocity.upper, velocity.batch, velocity.boundary,
           str(velocity.dom.device))
    if key not in _MASKS:
        if len(_MASKS) >= _MASKS_KEPT:
            del _MASKS[next(iter(_MASKS))]
        _MASKS[key] = _obstacle_masks(velocity, obstacles)
    return _MASKS[key]


def make_incompressible(velocity: StaggeredGrid, obstacles=(), solve: Solve = None, active=None, order=2):
    """fluid.make_incompressible (phi/physics/fluid.py:94-162): returns (divergence-free velocity, pressure).
    obstacles: stationary Box / Sphere / infinite_cylinder geometries (row N4)."""
    solve = solve or Solve()
    _require(isinstance(velocity, StaggeredGrid), "CenteredGrid velocities")
    _require(active is None and order == 2, "active masks / higher order")
    if solve.x0 is not None:
        _require(isinstance(solve.x0, CenteredGrid) and solve.x0.res == velocity.res and solve.x0.batch == velocity.batch, "x0 on a different grid")
    if obstacles:
        accessible, factors = _obstacle_masks_cached(velocity, obstacles)
        res = dict(zip(velocity.axes, velocity.res))
        p_data = solve.x0.data.clone() if solve.x0 is not None else velocity.dom.alloc_centered()
        v_data = [c.clone() for c in velocity.data]
        ops.mul_faces(velocity.dom, velocity.vspec, v_data, factors)             # apply_boundary_conditions
        ops.make_incompressible(velocity.dom, velocity.vspec, v_data, p_data, _cg_params(velocity, solve), accessible=accessible)
        _finish_solve(velocity.dom, solve)
        pressure = CenteredGrid(boundary=_pressure_boundary(velocity.boundary), bounds=velocity.bounds, batch=velocity.batch, _data=p_data, **res)
        return velocity.with_values(v_data), pressure
    res = dict(zip(velocity.axes, velocity.res))
    if solve.x0 is not None:
        p_data = solve.x0.data.clone()
    else:
        p_data = velocity.dom.alloc_centered()
    v_data = [c.clone() for c in velocity.data]
    ops.make_incompressible(velocity.dom, velocity.vspec, v_data, p_data, _cg_params(velocity, solve))
    _finish_solve(velocity.dom, solve)
    pressure = CenteredGrid(boundary=_pressure_boundary(velocity.boundary), bounds=velocity.bounds, batch=velocity.batch, _data=p_data, **res)
    return velocity.with_values(v_data), pressure


def incompressible_step(v: StaggeredGrid, s: CenteredGrid, p, dt: float, inflow: CenteredGrid = None, inflow_rate: float = 0.0,
                        buoyancy=(0, 0.1), solve: Solve = None, smoke_advection='semi_lagrangian', obstacles=()):
    """The notebook step (examples/grids/Smoke_Plume.ipynb:58-68) as ONE library call:
        s = advect(s, v, dt) + inflow_rate * inflow ;  v = semi_lagrangian(v, v, dt) + resample(s * buoyancy, to=v) * dt ;
        v, p = make_incompressible(v, obstacles, Solve('CG', ..., x0=p))
    obstacles: the stationary geometries make_incompressible takes (Box, Sphere, infinite_cylinder, union; Batched_Smoke.ipynb,
    Fluid_Logo.ipynb); their masks are rasterised once per geometry and grid.
    Returns new (v, s, p); inputs are not modified."""
    solve = solve or Solve('CG', 1e-3)
    _check_velocity(s, v)
    kw = {}
    if obstacles:
        kw['accessible'], kw['factors'] = _obstacle_masks_cached(v, obstacles)
    prm = _cg_params(v, solve)
    v_data = [c.clone() for c in v.data]
    s_data = s.data.clone()
    p_data = p.data.clone() if p is not None else v.dom.alloc_centered()
    infl = inflow.data if inflow is not None else None
    ops.plume_step(v.dom, v.vspec, s.spec, v_data, s_data, p_data, infl, float(dt), float(inflow_rate), tuple(buoyancy),
                   prm, mac_cormack=(smoke_advection == 'mac_cormack'), **kw)
    _finish_solve(v.dom, solve)
    pressure = CenteredGrid(boundary=_pressure_boundary(v.boundary), bounds=v.bounds, batch=v.batch, _data=p_data, **dict(zip(v.axes, v.res)))
    return v.with_values(v_data), s.with_values(s_data), pressure


fluid = SimpleNamespace(make_incompressible=make_incompressible, incompressible_step=incompressible_step)
