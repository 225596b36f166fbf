"""
`from phiflow_b200.flow import *`  --  the reference's user-facing names for the incompressible-fluid hot path
(the surface `from phi.flow import *` gives a grid-fluid notebook: phi/flow.py:13-28), backed by the CUDA kernels.

Mirrored (same names, argument meaning and error behaviour; reference file:line in each docstring):
    Box, Sphere, union, geom.infinite_cylinder, CenteredGrid, StaggeredGrid, extrapolation (ZERO, ONE, PERIODIC, ZERO_GRADIENT, BOUNDARY, combine_sides),
    Solve, SolveTape, NotConverged, Diverged, math.{sin, exp, linspace, PI, rotate_vector}, PI, field.{divergence, laplace, spatial_gradient, where}, resample,
    advect.{semi_lagrangian, mac_cormack, advect, points, euler, rk4}, geom.Point, spatial, diffuse.{explicit, implicit}, fluid.{make_incompressible, incompressible_step},
    write / read (field.write / field.read: the reference's .npz field files, see field_io.py).
Fused notebook steps (one kernel launch for all substeps of a call): reaction_diffusion (Reaction_Diffusion), wave_step (Waves).
Streamlines: streamlines(x0, v, step_size, iterations) returns every position of an advect.points trajectory from one kernel launch.
SPH: sph_step(x, v, domain, smoothing_length, particle_mass, dt, gravity, substeps=) runs the SPH notebook's substeps in one kernel launch.
Julia_Set: julia_set(c, iter_count, bounds, x=..., y=...) returns the escape counts as an int32 CenteredGrid in one kernel launch; an
int32 grid is a result only, which every operator refuses.
Precision: math.set_global_precision(64) / math.precision(64) make new grids float64 (the Taylor-Green notebook); laplace,
diffuse.explicit, divergence, spatial_gradient, semi_lagrangian and make_incompressible with Solve('CG') then run the fp64 kernels.
Fields hold device tensors in the library layout (DESIGN.md section 2); `.numpy()` returns the reference's (x, y[, z]) arrays.
Anything outside the fast path raises NotImplementedError (where the reference-side façade would fall through to stock
PhiFlow, INTEGRATION.md section 2).  No CPU fallback.
"""
import contextlib
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
           'resample', 'advect', 'diffuse', 'fluid', 'math', 'write', 'read', 'wave_step', 'julia_set', 'PI', 'spatial', 'streamlines', 'sph_step']

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

    @property
    def center(self):
        """Box.center (phi/geom/_box.py:109): (lower + upper) / 2 as a float32 NumPy vector, so that `bounds.center + vector` adds
        element by element (a `vec` is a tuple here, and tuple + tuple would concatenate)."""
        return np.array([(self.lower[k] + self.upper[k]) * 0.5 for k in self.names], np.float32)

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
    """Sphere(x=50, y=9.5, radius=5) or Sphere(center=vector, radius=1.)  (phi/geom/_sphere.py)."""

    def __init__(self, radius=None, center=None, **center_):
        _require(radius is not None and (center is None) != (not center_), "Sphere without a radius, or with both `center` and axis keywords")
        if center is not None:
            center = np.asarray(center, np.float32).reshape(-1)
            _require(len(center) in (2, 3), f"Sphere centre of {len(center)} components")
            center_ = dict(zip(AXES, center))
        self.names, self.center, self.radius = tuple(center_), tuple(float(v) for v in center_.values()), float(radius)

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


class Point:
    """geom.Point(center) (phi/geom/_geom.py): zero-volume points at `center`, a vec, a float32 NumPy array or a float32 CUDA tensor
    (..., dim) of world positions - what advect.points moves."""

    def __init__(self, center):
        self.center = center


geom = SimpleNamespace(Box=Box, Sphere=Sphere, union=union, infinite_cylinder=infinite_cylinder, Point=Point)


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


_PRECISION = [32]


def set_global_precision(bits: int):
    """math.set_global_precision (PhiML/phiml/backend/_dtype.py): 32 or 64 bits for the grids created from now on."""
    _require(bits in (32, 64), f"precision {bits}")
    _PRECISION[0] = int(bits)


def get_precision() -> int:
    return _PRECISION[0]


@contextlib.contextmanager
def precision(bits: int):
    """with math.precision(64): ... (PhiML/phiml/backend/_dtype.py)."""
    old = _PRECISION[0]
    set_global_precision(bits)
    try:
        yield
    finally:
        _PRECISION[0] = old


def _default_tolerance() -> float:
    """_optimize.py:130-136: 1e-12 in precision 64, 1e-5 in precision 32, taken when the solve runs."""
    return 1e-12 if _PRECISION[0] == 64 else 1e-5


class Solve:
    """phiml.math.Solve (_optimize.py:25-41): method, rel_tol, abs_tol, x0, max_iterations, suppress.  rel_tol / abs_tol left at None
    take _default_tolerance() of the precision in force when they are read (_optimize.py:108-111)."""

    def __init__(self, method='auto', rel_tol=None, abs_tol=None, x0=None, max_iterations=1000, suppress=(), matrix_offset=0.0):
        self.method, self.x0, self.max_iterations, self.suppress = method or 'auto', x0, int(max_iterations), tuple(suppress)
        self._rel_tol = None if rel_tol is None else float(rel_tol)
        self._abs_tol = None if abs_tol is None else float(abs_tol)
        self.matrix_offset = matrix_offset                                # see DESIGN.md section 3; 0 = plain CG

    @property
    def rel_tol(self) -> float:
        return _default_tolerance() if self._rel_tol is None else self._rel_tol

    @property
    def abs_tol(self) -> float:
        return _default_tolerance() if self._abs_tol is None else self._abs_tol


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


def _sin(x):
    """math.sin of a plain number: float32, as PhiML's NumPy backend returns it."""
    _require(isinstance(x, numbers.Real) and not isinstance(x, bool), "math.sin of anything but a plain number")
    return np.sin(np.float32(x))


def rotate_vector(vector, angle):
    """math.rotate_vector (PhiML/phiml/math/_nd.py:195-215) of a 2-D vector by a plain-number angle: (cos v_x - sin v_y,
    sin v_x + cos v_y) with sin and cos of the float32 angle, every operation in float32.  Returns a float32 NumPy vector."""
    v = np.asarray(vector, np.float32).reshape(-1)
    _require(len(v) == 2 and isinstance(angle, numbers.Real) and not isinstance(angle, bool), "rotate_vector other than 2-D by a plain number")
    s, c = np.sin(np.float32(angle)), np.cos(np.float32(angle))
    return np.array([c * v[0] + (-s) * v[1], s * v[0] + c * v[1]], np.float32)


def _linspace(start, stop, dim):
    """math.linspace(start, stop, batch(time=N)) (PhiML/phiml/math/_ops.py:648): N float32 numbers from start to stop, as a NumPy
    array along the one dimension (the notebooks' constants); bit for bit PhiML's, whose limits arrive as float32 numbers."""
    plain = lambda v: isinstance(v, numbers.Real) and not isinstance(v, bool)
    _require(plain(start) and plain(stop) and isinstance(dim, dict) and len(dim) == 1, "linspace other than between two numbers along one dim")
    return np.linspace(np.float32(start), np.float32(stop), int(next(iter(dim.values()))), dtype=np.float32)


def _exp(x):
    """math.exp of a plain number or of a float32 / complex64 NumPy array (what math.linspace and arithmetic on it make): float32 or
    complex64, as PhiML's NumPy backend computes it in precision 32."""
    if isinstance(x, numbers.Number) and not isinstance(x, bool):
        x = np.complex64(x) if isinstance(x, complex) else np.float32(x)
    x = np.asarray(x)
    _require(x.dtype in (np.float32, np.complex64), f"math.exp of {x.dtype} values")
    return np.exp(x)


PI = np.pi
math = SimpleNamespace(Solve=Solve, SolveTape=SolveTape, NotConverged=NotConverged, Diverged=Diverged,
                       ConvergenceException=ConvergenceException, extrapolation=extrapolation, sin=_sin, exp=_exp, linspace=_linspace, PI=PI,
                       rotate_vector=rotate_vector,
                       set_global_precision=set_global_precision, get_precision=get_precision, precision=precision)


def jit_compile(f=None, **_):
    """math.jit_compile (PhiML/phiml/math/_functional.py): the identity here - every call already is a pre-compiled CUDA kernel behind
    the C ABI, and ctypes launches must not be traced (SURVEY.md Appendix C)."""
    return f if f is not None else (lambda g: g)


def batch(**dims):
    """batch(time=300) as `iterate` uses it: the name and length of the trajectory dimension."""
    assert len(dims) == 1, "one trajectory dimension"
    return dict(dims)


def spatial(**dims):
    """spatial(iter=50) as `iterate` uses it (the Streamlines notebook): the name and length of the trajectory dimension, as `batch`."""
    return batch(**dims)


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


def _domain(res, dx, batch, vspec, dtype):
    upper = tuple(ops.stored_faces(vspec, a)[1] for a in range(len(res))) if vspec is not None else (False,) * len(res)
    key = (tuple(res), tuple(dx), batch, upper, _DEVICE, dtype)
    if key not in _DOMAINS:
        _DOMAINS[key] = ops.Domain(res, dx, batch, vbc=vspec, device=_DEVICE, dtype=dtype)
    return _DOMAINS[key]


def _grid_dtype(data):
    """dtype of a new grid's domain: that of the float data it wraps (int32 counts share the float32 layout), else the global
    precision's."""
    if data is not None:
        return torch.float64 if (data[0] if isinstance(data, (list, tuple)) else data).dtype == torch.float64 else torch.float32
    return torch.float64 if _PRECISION[0] == 64 else torch.float32


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

    @property
    def dtype(self) -> torch.dtype:
        data = self.__dict__.get('data')                 # not yet set while a geometry's mask is being sampled: the domain's
        if data is None:
            return self.dom.dtype
        return (data[0] if isinstance(data, (list, tuple)) else data).dtype

    @property
    def precision(self):
        """32 or 64 for float32 / float64 values; None for an int32 grid (julia_set's counts), which no operator takes."""
        return {torch.float32: 32, torch.float64: 64}.get(self.dtype)


class CenteredGrid(_Grid):
    """CenteredGrid(values, boundary, bounds, x=..., y=...)  (phi/field/_grid.py:21-86).
    values: number, numpy array in (x, y[, z]) order (optional leading batch axis), or a geometry (Box / Sphere: hard mask)."""

    def __init__(self, values=0., boundary=ZERO, bounds=None, batch=1, _data=None, _scale=None, **resolution):
        self._geometry(bounds, resolution, batch)
        self.boundary = _as_ext(boundary)
        self.dom = _domain(self.res, self.dx, batch, None, _grid_dtype(_data))
        self.vector_scale = _scale                       # s * (0, 0.1): a centred vector field that is a scalar times constants
        if _data is not None:
            self.data = _data
        elif isinstance(values, (Box, Sphere, Union)):
            _require_f32("a geometry as grid values (its mask is sampled at float32 cell centres)", self)
            self.data = self.dom.centered_from_numpy(values.lies_inside(self.points()).astype(self.dom.np_dtype))
        elif np.isscalar(values):
            self.data = self.dom.alloc_centered()
            if values != 0:
                self.data += float(values)
        else:
            self.data = self.dom.centered_from_numpy(np.asarray(values, self.dom.np_dtype))

    def points(self):
        axes = [(np.linspace(0.5 / n, 1 - 0.5 / n, n).astype(np.float32) * np.float32(u - l) + np.float32(l)) for l, u, n in zip(self.lower, self.upper, self.res)]
        return np.stack(np.meshgrid(*axes, indexing='ij'), -1).astype(np.float32)

    def axis_centres(self):
        """The reference's float32 cell centres along each axis, bit for bit (UniformGrid.center, phi/geom/_grid.py:60-63):
        PhiML's linspace runs in float32 (its limits arrive as float32 numbers), then lower + local * size.  `points()` forms the
        linspace in float64 and can differ by one ulp; the disc masks of field.where and wave_step use these."""
        return [np.linspace(np.float32(0.5 / n), np.float32(1 - 0.5 / n), n, dtype=np.float32) * np.float32(u - l) + np.float32(l)
                for l, u, n in zip(self.lower, self.upper, self.res)]

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
        _require_float("arithmetic", self)
        if isinstance(other, CenteredGrid):
            assert self._same_grid(other)
            _same_precision(self, other)
            return self.with_values(self.data + other.data)
        return self.with_values(self.data + float(other))

    __radd__ = __add__

    def __sub__(self, other):
        return self + (other * -1.0)

    def __mul__(self, other):
        _require_float("arithmetic", self)
        if isinstance(other, (tuple, list)):             # scalar field times a constant vector, e.g. s * (0, 0.1)
            g = self.with_values(self.data)
            g.vector_scale = tuple(float(o) for o in other)
            return g
        if isinstance(other, CenteredGrid):
            _same_precision(self, other)
            return self.with_values(self.data * other.data)
        return self.with_values(self.data * float(other))

    __rmul__ = __mul__

    def __rsub__(self, other):
        """number - field keeps the field's extrapolation (phi/field/_field.py:788-813)."""
        return (self * -1.0) + other

    def __neg__(self):
        return self * -1.0

    def __pow__(self, power):
        _require(isinstance(power, numbers.Real) and not isinstance(power, bool), "a power other than a plain number")
        _require_float("arithmetic", self)
        return self.with_values(self.data ** float(power))

    def laplace(self, order=2):
        """Field.laplace (phi/field/_field.py:563-573) = field.laplace(self)."""
        return laplace(self, order)


class StaggeredGrid(_Grid):
    """StaggeredGrid(values, boundary, bounds, x=..., y=...)  (phi/field/_grid.py:89-176).
    values: number, tuple of per-component constants, list of per-component numpy arrays shaped as the reference stores
    them (n-1 / n / n+1 faces, tests/commit/field/test__grid.py:25-37), or a geometry (hard mask sampled at face centres)."""

    def __init__(self, values=0., boundary=ZERO, bounds=None, batch=1, _data=None, **resolution):
        self._geometry(bounds, resolution, batch)
        self.boundary = _as_ext(boundary)
        self.vspec = self.boundary.vspec(self.axes)
        self.dom = _domain(self.res, self.dx, batch, self.vspec, _grid_dtype(_data))
        d = len(self.res)
        if _data is not None:
            self.data = _data
            return
        shapes, _ = self.dom.face_shapes(self.vspec)
        dt = self.dom.np_dtype
        if isinstance(values, (Box, Sphere)):
            _require_f32("a geometry as grid values (its mask is sampled at float32 face centres)", self)
            comps = [values.lies_inside(self.face_points(c)).astype(dt) for c in range(d)]
        elif np.isscalar(values):
            comps = [np.full(shapes[c], values, dt) for c in range(d)]
        elif isinstance(values, tuple) and all(np.isscalar(v) for v in values):
            comps = [np.full(shapes[c], values[c], dt) for c in range(d)]
        else:
            comps = [np.asarray(v, dt) for v in values]
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
        with precision(self.precision):
            new = StaggeredGrid(0, boundary, self.bounds, self.batch, **dict(zip(self.axes, self.res)))
        old = self.numpy()
        comps = []
        for c, a in enumerate(self.axes):
            lo0, hi0 = self.boundary.valid_outer_faces(a)
            lo1, hi1 = boundary.valid_outer_faces(a)
            full = np.zeros(old[c].shape[:old[c].ndim - len(self.res)] + tuple(n + (1 if i == c else 0) for i, n in enumerate(self.res)), old[c].dtype)
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
            _same_precision(self, other)
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


def _same_precision(*fields):
    """Fields of one operation share their precision: nothing is converted silently."""
    _require_float("an operation", *fields)
    bits = {f.precision for f in fields if isinstance(f, _Grid)}
    _require(len(bits) <= 1, "mixing float32 and float64 fields in one operation")


def _require_f32(what, *fields):
    _require_float(what, *fields)
    _require(all(f.precision == 32 for f in fields if isinstance(f, _Grid)), f"{what} in precision 64 (fp32 only)")


def _require_float(what, *fields):
    """Operators take float32 or float64 grids; an int32 grid (julia_set's counts) is refused instead of being read as float32."""
    bad = sorted({str(f.dtype) for f in fields if isinstance(f, _Grid) and f.precision is None})
    _require(not bad, f"{what} of {', '.join(bad)} grids")


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
    _require_float("laplace", u)
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
    _require_float("spatial_gradient", p)
    _require(_pressure_boundary(boundary) == p.boundary, "spatial_gradient with an unrelated field boundary")
    with precision(p.precision):
        g = StaggeredGrid(0, boundary, p.bounds, p.batch, **dict(zip(p.axes, p.res)))
    ops.grad_sub(g.dom, g.vspec, g.data, p.data)
    return g * -1.0


def resample(value, to, soft=False, **_):
    """resample(value, to) for the two cases of the notebook step (phi/field/_resample.py:13-63):
    geometry -> CenteredGrid (soft mask, :192-210) and (CenteredGrid * constant vector) -> StaggeredGrid (:272-276)."""
    if isinstance(value, Sphere) and isinstance(to, CenteredGrid):
        _require_f32("resample(geometry, to=CenteredGrid) (the mask is sampled at float32 cell centres)", to)
        if soft:
            cell_r = float(np.sqrt(sum((h * 0.5) ** 2 for h in to.dx)))
            return to.with_values(to.dom.centered_from_numpy(value.soft_mask(to.points(), cell_r)))
        return to.with_values(to.dom.centered_from_numpy(value.lies_inside(to.points()).astype(np.float32)))
    if isinstance(value, CenteredGrid) and isinstance(to, StaggeredGrid) and value.vector_scale is not None:
        _require(value.res == to.res, "resampling between different resolutions")
        _require_f32("resample(CenteredGrid * vector, to=StaggeredGrid)", value, to)
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
    bits = 64 if np.asarray(st['data']).dtype == np.float64 else 32          # float64 files stay float64
    data = np.asarray(st['data'], np.float64 if bits == 64 else np.float32)
    batch = data.shape[0] if lead else 1
    bounds = Box(**{a: (st['lower'][a], st['upper'][a]) for a in axes})
    if st['field_type'] == 'CenteredGrid':
        _require(data.ndim == len(lead) + len(axes), "centred grids with channel dims")
        res = dict(zip(axes, data.shape[len(lead):]))
        with precision(bits):
            return CenteredGrid(data, boundary, bounds, batch, **res)
    _require(names[-1] == 'vector' and data.shape[-1] == len(axes), "staggered tensors whose components are not the spatial dims")
    comps = field_io.unstack_staggered_tensor(data, lambda ax: (boundary.side(axes[ax], False), boundary.side(axes[ax], True)), len(axes))
    res = {a: n - 1 for a, n in zip(axes, data.shape[len(lead):len(lead) + len(axes)])}
    with precision(bits):
        return StaggeredGrid(comps, boundary, bounds, batch, **res)


def where(mask, field_true, field_false):
    """field.where (phi/field/_field_math.py:997-1015) on CenteredGrids with a hard mask: mask is a geometry (Box / Sphere / union,
    sampled at the cell centres: _resample.py:192-210, Sphere.lies_inside, phi/geom/_sphere.py:103-105) or a CenteredGrid (non-zero
    = True); field_true / field_false are CenteredGrids or plain numbers.  The result carries the extrapolation of the first field
    among (field_true, field_false, mask), as _auto_resample resamples everything onto it."""
    fields = [f for f in (field_true, field_false, mask) if isinstance(f, CenteredGrid)]
    _require(bool(fields), "field.where without a CenteredGrid")
    ref = fields[0]
    _require(all(f._same_grid(ref) and f.vector_scale is None for f in fields), "field.where of vector fields or fields on different grids")
    plain = lambda x: isinstance(x, numbers.Real) and not isinstance(x, bool)
    _require(all(isinstance(x, CenteredGrid) or plain(x) for x in (field_true, field_false)), "field.where with non-number values")
    _require_f32("field.where", *fields)
    if isinstance(mask, CenteredGrid):
        m = mask.data != 0
    else:
        _require(isinstance(mask, (Box, Sphere, Union)), f"field.where with a {type(mask).__name__} mask")
        pts = np.stack(np.meshgrid(*ref.axis_centres(), indexing='ij'), -1)
        m = ref.dom.centered_from_numpy(mask.lies_inside(pts).astype(np.float32)) != 0
    val = lambda x: x.data if isinstance(x, CenteredGrid) else torch.tensor(np.float32(x), device=ref.data.device)
    return ref.with_values(torch.where(m, val(field_true), val(field_false)))


field = SimpleNamespace(divergence=divergence, laplace=laplace, spatial_gradient=spatial_gradient, resample=resample, where=where,
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
    _same_precision(fld, velocity)


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
    _require_f32("advect.mac_cormack", fld, velocity)
    return fld.with_values(ops.mac_cormack_centered(velocity.dom, velocity.vspec, velocity.data, fld.spec, fld.data, float(dt), correction_strength))


def euler(data, velocity, dt: float, v0=None):
    """advect.euler (phi/physics/advect.py:20-24) on points: the positions after one Euler step (what advect.points computes with it)."""
    _require(v0 is None, "integrators with a given v0")
    return points(data, velocity, dt, integrator=euler)


def rk4(data, velocity, dt: float, v0=None):
    """advect.rk4 (phi/physics/advect.py:27-35) on points: the positions after one Runge-Kutta-4 step."""
    _require(v0 is None, "integrators with a given v0")
    return points(data, velocity, dt, integrator=rk4)


def finite_rk4(data, velocity, dt: float, v0=None):
    """advect.finite_rk4 (phi/physics/advect.py:38-50): not on the fast path."""
    _require(False, "advect.finite_rk4")


_INTEGRATOR_NAMES = {euler: 'euler', rk4: 'rk4'}


def _as_points(x, dim):
    """(kind, float32 tensor (N, dim), shape of x) of a Point centre, vec, float32 NumPy array or float32 CUDA tensor.  A vec comes
    back as a float32 NumPy vector, the kind `iterate` carries as ONE state variable (a tuple would be several)."""
    if isinstance(x, torch.Tensor):
        _require(x.dtype == torch.float32 and x.is_cuda, f"points as a {x.dtype} tensor on {x.device} (float32 CUDA tensors)")
        kind, t = 'tensor', x
    elif isinstance(x, tuple) and all(isinstance(v, numbers.Real) and not isinstance(v, bool) for v in x):
        kind, t = 'vec', torch.tensor(np.array(x, np.float32))
    else:
        _require(isinstance(x, np.ndarray) and x.dtype == np.float32, f"points of type {type(x).__name__} "
                 f"{getattr(x, 'dtype', '')} (a vec, float32 NumPy arrays or float32 CUDA tensors)")
        kind, t = 'numpy', torch.from_numpy(np.ascontiguousarray(x))
    _require(t.dim() >= 1 and t.shape[-1] == dim, f"points of shape {tuple(t.shape)} in a {dim}-D velocity")
    return kind, t, tuple(t.shape)


def _from_points(kind, t, shape):
    if kind == 'tensor':
        return t.reshape(shape)
    return t.cpu().numpy().reshape(shape)


def _advect_points(x, velocity, dt, integrator, steps, trajectory):
    """steps of advect.points in one launch; x: the points of any supported kind.  Returns (kind, result tensor, shape of x)."""
    _require(isinstance(velocity, StaggeredGrid), "advect.points by a non-staggered velocity")
    _require_f32("advect.points", velocity)
    _require(integrator in _INTEGRATOR_NAMES, f"advect.points with integrator {getattr(integrator, '__name__', integrator)!r} (euler, rk4)")
    kind, t, shape = _as_points(x, len(velocity.res))
    d = len(velocity.res)
    pts = t.reshape(1, -1, d).to(velocity.dom.device).contiguous()
    if pts.data_ptr() == t.data_ptr():
        pts = pts.clone()                                # the kernel writes its own output; the caller's points stay as they are
    res = ops.advect_points(velocity.dom, velocity.vspec, velocity.data, velocity.lower, velocity.upper, pts, float(dt),
                            _INTEGRATOR_NAMES[integrator], steps, out=None if trajectory or velocity.batch > 1 else pts,
                            trajectory=trajectory)
    return kind, (res[1] if trajectory else res), shape


def points(points, velocity: StaggeredGrid, dt: float, integrator=euler):
    """advect.points (phi/physics/advect.py:136-153): moves the points by `integrator` (advect.euler or advect.rk4) through the float32
    StaggeredGrid `velocity`, in one kernel launch, bit for bit as PhiML computes it (DESIGN.md row N11).  points: a geom.Point, a
    vec, a float32 NumPy array or a float32 CUDA tensor (..., dim); the result has the same kind and shape (a Point for a Point; a
    float32 NumPy vector for a vec).
    A velocity of batch B > 1 moves the same points in every batch entry; the result then gains a leading axis of length B."""
    x = points.center if isinstance(points, Point) else points
    kind, t, shape = _advect_points(x, velocity, dt, integrator, 1, False)
    out = _from_points(kind, t, (t.shape[0],) + shape if t.shape[0] > 1 else shape)
    return Point(out) if isinstance(points, Point) else out


def streamlines(x0, velocity: StaggeredGrid, step_size: float, iterations: int, integrator=rk4):
    """The Streamlines notebook's trajectory  iterate(lambda x: advect.points(geom.Point(x), v, step_size, integrator).center,
    spatial(iter=iterations), x0)  from ONE kernel launch: the positions (iterations + 1, [B,] ..., dim), entry 0 = x0, as a NumPy array
    (a CUDA tensor for a tensor x0), bit for bit the same as the iterate form."""
    _require(isinstance(iterations, int) and not isinstance(iterations, bool) and iterations >= 1, f"iterations = {iterations!r}")
    x = x0.center if isinstance(x0, Point) else x0
    kind, t, shape = _advect_points(x, velocity, step_size, integrator, iterations, True)
    shape = (iterations + 1,) + ((t.shape[1],) if t.shape[1] > 1 else ()) + shape
    return t.reshape(shape) if kind == 'tensor' else t.cpu().numpy().reshape(shape)


def sph_step(x, v, domain: Box, smoothing_length: float, particle_mass: float, dt: float, gravity, dynamic_visc: float = 0.025,
             isotropic_exp: float = 20., base_density: float = 1., damping_coef: float = -0.95, substeps: int = 1):
    """The SPH notebook's substep apply_bounds(sph_step(v)) (examples/particles/SPH.ipynb, phi/physics/sph.py) with the poly6 kernel,
    `substeps` times in one kernel launch (DESIGN.md row N12).  x, v: particle positions and velocities, float32 NumPy arrays or
    float32 CUDA tensors of one kind and shape (N, d), d = 2 or 3 = the axes of `domain`; gravity: a vec / d numbers.  The support
    radius comes from smoothing_length as the notebook's desired_neighbors gives it; particle_mass is the notebook's
    0.01 * mean(volume).  Returns (x, v) of the same kind.  iterate(lambda x, v: sph_step(x, v, ...), batch(t=480), x, v, substeps=40)
    runs the notebook's loop one substep per call; sph_step(..., substeps=40) runs a frame in one launch."""
    kx, tx, sx = _as_points(x, len(domain.names))
    kv, tv, sv = _as_points(v, len(domain.names))
    d = len(domain.names)
    _require(kx == kv and kx in ('numpy', 'tensor'), f"sph_step of {kx} positions and {kv} velocities (both float32 NumPy arrays or both "
                                                     f"float32 CUDA tensors)")
    _require(len(sx) == 2 and sx == sv and d in (2, 3), f"sph_step of positions {sx} and velocities {sv} in a {d}-D domain ((N, d), d = 2 or 3)")
    _require(isinstance(gravity, (tuple, list, np.ndarray)) and len(gravity) == d, f"sph_step with gravity {gravity!r} ({d} numbers)")
    _require(isinstance(substeps, int) and not isinstance(substeps, bool) and substeps >= 1, f"sph_step with substeps = {substeps!r}")
    prm = ops.sph_params([domain.lower[k] for k in domain.names], [domain.upper[k] for k in domain.names], smoothing_length,
                         particle_mass, dt, gravity, dynamic_visc, isotropic_exp, base_density, damping_coef)
    dev = _DEVICE if kx == 'numpy' else tx.device
    xo, vo = ops.sph(tx.to(dev).contiguous(), tv.to(dev).contiguous(), prm, substeps)
    return _from_points(kx, xo, sx), _from_points(kv, vo, sv)


def _advect(fld, velocity, dt: float, integrator=euler):
    """advect.advect (phi/physics/advect.py:53-74): points (a Point, vec, array or tensor) go to advect.points, grids to
    semi_lagrangian (Euler only)."""
    if isinstance(fld, (Point, np.ndarray, torch.Tensor, tuple)):
        return points(fld, velocity, dt, integrator)
    _require(integrator is euler or integrator is None, "grid advection with integrators other than euler")
    return semi_lagrangian(fld, velocity, dt)


advect = SimpleNamespace(semi_lagrangian=semi_lagrangian, mac_cormack=mac_cormack, advect=_advect, points=points, euler=euler, rk4=rk4,
                         finite_rk4=finite_rk4)


# ----------------------------------------------------------------------------------------------------------------------
# diffuse  (phi/physics/diffuse.py)
# ----------------------------------------------------------------------------------------------------------------------
def explicit(fld, diffusivity: float, dt: float, substeps: int = 1):
    """diffuse.explicit (phi/physics/diffuse.py:13-60): substeps of  u += (dt/substeps) * diffusivity * laplace(u); for a
    StaggeredGrid every component is diffused with its own boundary (Lid_Driven_Cavity.ipynb, Variable_Boundaries.ipynb)."""
    amount = float(diffusivity) * float(dt) / substeps
    _require_float("diffuse.explicit", fld)
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
    _require_f32("diffuse.implicit", fld, diffusivity)
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
# reaction-diffusion  (examples/grids/Reaction_Diffusion.ipynb)
# ----------------------------------------------------------------------------------------------------------------------
def _fixed_point_side(s):
    """Sides whose extrapolation the step maps to itself: PhiML's field arithmetic keeps a field's own extrapolation when it is
    combined with a number, so a constant c turns into 2c - c**2 after one step; only c = 0 stays."""
    return s in ('periodic', 'zg') or (isinstance(s, float) and s == 0.0)


def reaction_diffusion(u: CenteredGrid, v: CenteredGrid, du: float, dv: float, f: float, k: float, dt: float, substeps: int = 1):
    """The Reaction_Diffusion notebook's Gray-Scott step, `substeps` times in one kernel launch:
        uvv = u * v**2;  su = du * field.laplace(u) - uvv + f * (1 - u);  sv = dv * field.laplace(v) + uvv - (f + k) * v
        return u + dt * su, v + dt * sv
    with the rounding of the reference's float32 field arithmetic.  Returns new fields (u', v'); u and v are not modified and may be
    the same field (the notebook passes u0, u0).  Boundaries: PERIODIC, ZERO_GRADIENT and ZERO per side, the same kinds for u and
    v; a non-zero constant drifts under the reference's step and raises NotImplementedError."""
    plain = lambda x: isinstance(x, numbers.Real) and not isinstance(x, bool)
    _require(isinstance(u, CenteredGrid) and isinstance(v, CenteredGrid), "reaction-diffusion of non-centred fields")
    _require(u.vector_scale is None and v.vector_scale is None, "reaction-diffusion of vector fields")
    _require(u._same_grid(v), "reaction-diffusion of fields on different grids")
    _require_f32("reaction_diffusion", u, v)
    _require(all(plain(x) for x in (du, dv, f, k, dt)), "reaction-diffusion with Field / per-batch parameters")
    _require(isinstance(substeps, int) and substeps >= 0, f"substeps = {substeps!r}")
    su, sv = u.spec, v.spec
    _require(all(_fixed_point_side(s) for spec in (su, sv) for ax in spec for s in ax),
             f"reaction-diffusion with a non-zero constant boundary ({u.boundary}, {v.boundary}): the reference's step moves it to 2c - c**2")
    _require(all(a == b or (not isinstance(a, str) and not isinstance(b, str)) for ax_u, ax_v in zip(su, sv) for a, b in zip(ax_u, ax_v)),
             "reaction-diffusion with different boundary kinds for u and v")
    un, vn = ops.reaction_diffusion(u.dom, [su, sv], u.data, v.data, float(du), float(dv), float(f), float(k), float(dt), substeps)
    return u.with_values(un), v.with_values(vn)


# ----------------------------------------------------------------------------------------------------------------------
# waves  (examples/grids/Waves.ipynb)
# ----------------------------------------------------------------------------------------------------------------------
def wave_step(h_c: CenteredGrid, h_p: CenteredGrid, time, dt: float, k_speed: float = 1.0, k_damp: float = 0.0, substeps: int = 1,
              source=None):
    """The Waves notebook's step, `substeps` times in one kernel launch.  Per substep, at the substep's time:
        sphere, value = source(time);  h_c, h_p = [field.where(sphere, value, f) for f in (h_c, h_p)]
        h_n = 2.0 * h_c - h_p + dt * dt * (k_speed * h_c.laplace() - k_damp * (h_c - h_p));  h_c, h_p, time = h_n, h_c, time + dt
    with the rounding of the reference's float32 field arithmetic.  `source`: None (no disc) or a callable time -> (Sphere, value),
    evaluated on the host for every substep; one disc per substep for every batch entry, one radius per call.  Returns (h_n, h_c,
    time): the newest state, the previous (stamped) one and the advanced time.  h_c and h_p are not modified and may be the same field
    (the notebook passes h0, h0).  Boundaries: PERIODIC, ZERO_GRADIENT and ZERO per side; a non-zero constant c drifts to 0 under
    the reference's step (2.0 * h_c keeps h_c's extrapolation) and raises NotImplementedError."""
    plain = lambda x: isinstance(x, numbers.Real) and not isinstance(x, bool)
    _require(isinstance(h_c, CenteredGrid) and isinstance(h_p, CenteredGrid), "the wave step of non-centred fields")
    _require(h_c.vector_scale is None and h_p.vector_scale is None, "the wave step of vector fields")
    _require(h_c._same_grid(h_p) and h_c.boundary == h_p.boundary, "the wave step of fields on different grids or with different boundaries")
    _require_f32("wave_step", h_c, h_p)
    _require(all(plain(x) for x in (time, dt, k_speed, k_damp)), "the wave step with Field / per-batch parameters")
    _require(isinstance(substeps, int) and substeps >= 0, f"substeps = {substeps!r}")
    _require(all(_fixed_point_side(s) for ax in h_c.spec for s in ax),
             f"the wave step with a non-zero constant boundary ({h_c.boundary}): the reference's step moves it to c - c = 0")
    discs, radius = [], None
    for _ in builtins_range(substeps):
        if source is None:
            discs.append(None)
        else:
            sphere, value = source(time)
            _require(isinstance(sphere, Sphere) and sphere.names == h_c.axes, f"a {type(sphere).__name__} source (a Sphere over the grid's axes is on the fast path)")
            _require(plain(value), "a source value that is not a plain number")
            _require(radius is None or sphere.radius == radius, "sources of different radii in one call")
            radius = sphere.radius
            discs.append((np.asarray(sphere.center, np.float32), np.float32(value)))
        time = time + dt
    r2 = np.float32((radius if radius is not None else 0.0) ** 2)
    hn, hc = ops.wave(h_c.dom, h_c.spec, h_c.data, h_p.data, np.float32(dt * dt), float(k_speed), float(k_damp), discs, r2,
                      np.concatenate(h_c.axis_centres()), substeps)
    return h_c.with_values(hn), h_c.with_values(hc), time


# ----------------------------------------------------------------------------------------------------------------------
# Julia sets  (examples/grids/Julia_Set.ipynb)
# ----------------------------------------------------------------------------------------------------------------------
def julia_set(c, iter_count: int, bounds: Box = None, **resolution) -> CenteredGrid:
    """The Julia_Set notebook's sampled grid in one kernel launch:
        CenteredGrid(lambda x, y: iterate(julia_map, iter_count, x + y * 1j, 0, c=c)[1], x=..., y=..., bounds=bounds)
        julia_map(z, counter, c) = z ** 2 + c, counter + (abs(z) < 2)
    with PhiML's complex64 rounding.  c: one complex constant or a 1-D array of them (the notebook's
    0.7885 * math.exp(1j * math.linspace(0, 2 * PI, batch(time=100)))), one batch entry each.  Returns an int32 CenteredGrid of batch
    len(c) whose .numpy() is (batch, x, y) (batch 1: (x, y)); the axes x and y stand for the real and imaginary parts."""
    cc = np.atleast_1d(np.asarray(c))
    _require(cc.ndim == 1 and cc.size >= 1 and np.issubdtype(cc.dtype, np.number), "Julia constants other than a 1-D array of numbers")
    _require(tuple(resolution) == ('x', 'y'), f"a Julia set on axes {tuple(resolution)} (2-D x, y)")
    _require(isinstance(iter_count, int) and not isinstance(iter_count, bool) and iter_count >= 0, f"iter_count = {iter_count!r}")
    out = CenteredGrid(bounds=bounds, batch=cc.size, _data=torch.empty(0, dtype=torch.int32), **resolution)
    out.data = ops.julia(out.dom, np.concatenate(out.axis_centres()), cc.astype(np.complex64), iter_count)
    return out


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
    _require(not adaptive or v.precision == 32, f"Solve('{solve.method}') in precision 64 (CG-adaptive runs on the fp32 ring kernel only; "
                                                f"use Solve('CG'))")
    return ops.cg_params(v.vspec, rtol=solve.rel_tol, atol=solve.abs_tol, max_iter=solve.max_iterations,
                         matrix_offset=0.0 if adaptive else solve.matrix_offset, method='CG-adaptive' if adaptive else 'CG', dtype=v.dom.dtype)


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
        _same_precision(velocity, solve.x0)
    if obstacles:
        _require_f32("make_incompressible with obstacles", velocity)
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
    _require_f32("incompressible_step", v, s, p, inflow)
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
