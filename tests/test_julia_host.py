"""
Julia sets without a GPU: the oracle against PhiML 1.7.2 (tests/golden/phiml_julia.npz), the kernel's band shortcut against the exact
abs, the mirror's constants and cell centres, argument validation of phicuda_julia_f32, and the refusal of int32 grids by every
operator of the mirror.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import phiflow_b200.flow as flow
from oracle_julia import F32, JULIA_HI, JULIA_LO, JuliaOracleEngine, abs32, band_decision, julia_counts, square_plus
from phiflow_b200 import _lib
from test_gpu_julia import CASES, GOLD, golden_case


def simd_found():
    from numpy._core._multiarray_umath import __cpu_dispatch__, __cpu_features__
    return ' '.join(f for f in __cpu_dispatch__ if __cpu_features__[f])


def require_recorded_dispatch():
    """NumPy's complex64 loops round as recorded only where NumPy dispatches to the same SIMD targets."""
    recorded = str(np.load(GOLD)['numpy/simd_found'])
    if simd_found() != recorded:
        pytest.skip(f"NumPy dispatches to [{simd_found()}] here, the fixture was recorded with [{recorded}]")


# ---- oracle vs PhiML -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_phiml(name):
    """Every case, every count: the oracle's float32 operations are PhiML's complex64 arithmetic bit for bit."""
    c, centres, res, iterations, counts = golden_case(np.load(GOLD), name)
    assert np.array_equal(julia_counts(centres[:res[0]], centres[res[0]:], c, iterations), counts)


def test_band_cases_need_numpys_abs():
    """The thin boxes around |z0| = 2 separate NumPy's abs from a correctly rounded hypot."""
    g = np.load(GOLD)
    assert all(int(g[f'{n}/hypot_differs']) > 0 for n in ('band_x', 'band_y', 'band_diag'))


def test_numpy_rounds_as_the_oracle():
    """Live NumPy complex64 on this CPU: np.power(z, 2) + c (PhiML's z ** 2) and abs(z) as the oracle restates them (2 M seeded
    points)."""
    require_recorded_dispatch()
    rng = np.random.default_rng(7)
    a, b, cr, ci = (rng.uniform(-3, 3, 1 << 21).astype(F32) for _ in range(4))
    z = (a + 1j * b).astype(np.complex64)
    w = np.power(z, 2) + (cr + 1j * ci).astype(np.complex64)
    re, im = square_plus(a, b, cr, ci)
    assert np.array_equal(w.real, re) and np.array_equal(w.imag, im)
    assert np.array_equal(np.abs(z), abs32(a, b))


def test_band_shortcut_equals_exact_abs():
    """The kernel's test of fma(a, a, b*b) against [JULIA_LO, JULIA_HI] decides abs(z) < 2 as the exact formula does: on points
    spread around the circle within 1e-5 of it, and on points whose s lies on either side of each band edge."""
    rng = np.random.default_rng(11)
    t = rng.uniform(0, 2 * np.pi, 1 << 20)
    r = 2 + rng.uniform(-1e-5, 1e-5, t.size)
    a, b = (r * np.cos(t)).astype(F32), (r * np.sin(t)).astype(F32)
    assert np.array_equal(band_decision(a, b), abs32(a, b) < F32(2))
    for edge in (JULIA_LO, JULIA_HI):
        for ulps in range(-4, 5):
            s = np.float64(edge) + ulps * np.float64(np.spacing(edge))
            rr = np.sqrt(s)
            a, b = (rr * np.cos(t[:4096])).astype(F32), (rr * np.sin(t[:4096])).astype(F32)
            assert np.array_equal(band_decision(a, b), abs32(a, b) < F32(2))
    assert abs32(F32(np.nan), F32(1.0)) != abs32(F32(np.nan), F32(1.0)) and not band_decision(F32(np.nan), F32(1.0))


# ---- the mirror's constants and centres ---------------------------------------------------------------------------------------------
@pytest.fixture()
def oracle_mirror():
    saved = flow.ops, flow._DEVICE
    flow.ops = JuliaOracleEngine
    flow.set_device('cpu')
    try:
        yield
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])


def test_mirror_constants_match_phiml():
    """The notebook's cell `c = 0.7885 * math.exp(1j*math.linspace(0, 2*PI, batch(time=100)))`, run unmodified on the mirror."""
    require_recorded_dispatch()
    math, PI, batch = flow.math, flow.PI, flow.batch
    c = 0.7885 * math.exp(1j*math.linspace(0, 2*PI, batch(time=100)))
    assert c.dtype == np.complex64 and c.shape == (100,)
    assert np.array_equal(c.view(F32).reshape(-1, 2).view(np.uint32), np.load(GOLD)['notebook/c_all'].view(np.uint32))


@pytest.mark.parametrize('name', CASES)
def test_mirror_centres_match_phiml(name, oracle_mirror):
    g = np.load(GOLD)
    c, centres, res, iterations, counts = golden_case(g, name)
    box = g[f'{name}/box']
    grid = flow.CenteredGrid(0, bounds=flow.Box(x=tuple(box[0]), y=tuple(box[1])), x=res[0], y=res[1])
    assert np.array_equal(np.concatenate(grid.axis_centres()), centres)


def test_mirror_julia_set(oracle_mirror):
    """flow.julia_set: an int32 CenteredGrid of batch len(c), (batch, x, y) from .numpy(), the fixture's counts."""
    g = np.load(GOLD)
    c, centres, res, iterations, counts = golden_case(g, 'iter50')
    box = g['iter50/box']
    out = flow.julia_set(c, iterations, flow.Box(x=tuple(box[0]), y=tuple(box[1])), x=res[0], y=res[1])
    assert isinstance(out, flow.CenteredGrid) and out.batch == len(c) and out.data.dtype == torch.int32
    assert out.numpy().dtype == np.int32 and np.array_equal(out.numpy(), counts)
    one = flow.julia_set(complex(c[1]), iterations, flow.Box(x=tuple(box[0]), y=tuple(box[1])), x=res[0], y=res[1])
    assert one.batch == 1 and np.array_equal(one.numpy(), counts[1])
    for bad in (lambda: flow.julia_set(c, 50, x=8, y=8, z=8), lambda: flow.julia_set(c, -1, x=8, y=8),
                lambda: flow.julia_set(c, 2.5, x=8, y=8), lambda: flow.julia_set(np.ones((2, 2)), 5, x=8, y=8)):
        with pytest.raises(NotImplementedError):
            bad()


class _NoKernels:
    """An engine that fails on use: an int32 grid must be refused by the mirror before any kernel is chosen."""

    def __getattr__(self, name):
        raise AssertionError(f"ops.{name} reached with an int32 grid")


def test_int32_grids_are_refused_by_every_operator(oracle_mirror):
    counts = flow.julia_set([0.3 + 0.5j], 5, flow.Box(x=(-2, 2), y=(-2, 2)), x=8, y=8)
    assert counts.precision is None and counts.dtype == torch.int32
    v = flow.StaggeredGrid(0.1, flow.PERIODIC, flow.Box(x=(-2, 2), y=(-2, 2)), x=8, y=8)
    s = flow.CenteredGrid(0.2, flow.PERIODIC, flow.Box(x=(-2, 2), y=(-2, 2)), x=8, y=8)
    cases = [
        lambda: flow.field.laplace(counts), lambda: counts.laplace(),
        lambda: flow.spatial_gradient(counts, flow.PERIODIC),
        lambda: flow.diffuse.explicit(counts, 0.1, 0.1), lambda: flow.diffuse.implicit(counts, 0.1, 0.1),
        lambda: flow.diffuse.implicit(s, counts, 0.1),
        lambda: flow.advect.semi_lagrangian(counts, v, 0.1), lambda: flow.advect.mac_cormack(counts, v, 0.1),
        lambda: flow.field.where(flow.Sphere(x=0, y=0, radius=1), 1.0, counts), lambda: flow.field.where(counts, 1.0, s),
        lambda: flow.resample(counts * (0, 0.1), to=v), lambda: flow.resample(flow.Sphere(x=0, y=0, radius=1), to=counts),
        lambda: flow.reaction_diffusion(counts, counts, 0.1, 0.1, 0.01, 0.05, 1.0),
        lambda: flow.wave_step(counts, counts, 0.0, 0.1),
        lambda: flow.fluid.make_incompressible(v, (), flow.Solve('CG', x0=counts)),
        lambda: flow.fluid.incompressible_step(v, counts, None, 0.1),
        lambda: flow.fluid.incompressible_step(v, s, counts, 0.1),
        lambda: flow.fluid.incompressible_step(v, s, None, 0.1, inflow=counts),
        lambda: counts + 1, lambda: counts * 2.0, lambda: counts ** 2, lambda: 1 - counts, lambda: -counts, lambda: counts + s,
    ]
    flow.ops = _NoKernels()
    for i, case in enumerate(cases):
        with pytest.raises(NotImplementedError, match='int32'):
            case()


def test_ops_refuse_int32_arrays(monkeypatch):
    """Below the mirror: entry points without an fp64 kernel test the dtype itself, the others take only the domain's float dtype."""
    from phiflow_b200 import _ops
    monkeypatch.setattr(_ops, 'require_cuda', lambda: None)
    spec = ((P, P), (P, P))
    dom = _ops.Domain((8, 8), (1.0, 1.0), 1, vbc=spec, device='cpu')
    i32 = torch.zeros(dom._shape(dom.cext), dtype=torch.int32)
    with pytest.raises(_lib.Unsupported, match='int32'):
        _ops.reaction_diffusion(dom, spec, i32, i32, 0.1, 0.1, 0.01, 0.05, 1.0)
    with pytest.raises(_lib.Unsupported, match='int32'):
        _ops.diffuse_implicit(dom, spec, i32, 0.1)
    with pytest.raises(_lib.Unsupported, match='int32'):
        _ops.axpy_centered(dom, 1.0, i32, dom.alloc_centered())
    with pytest.raises(AssertionError, match='domain'):
        _ops.laplace(dom, spec, i32, out=i32.clone())


# ---- C ABI validation (no CUDA call is reached) -------------------------------------------------------------------------------------
P = 'periodic'


def _grid(dim=2, n=(16, 8, 4), batch=2):
    g = _lib.PhiGrid()
    g.dim, g.batch, g.halo = dim, batch, 0
    for a in range(dim):
        g.n[a] = n[a]
        g.cext[a] = g.fext[a] = (n[a] + 3) // 4 * 4 if a == 0 else n[a]
        g.dx[a] = 1.0
    return g


def _call(g=None, counts=16 << 20, scratch=48 << 20, iterations=5, short=0, centres=None, c=True, null_centres=False):
    lib = _lib.load()
    g = g or _grid()
    need = lib.phicuda_julia_scratch_bytes(C.byref(g))
    nax = sum(g.n[a] for a in range(g.dim))
    cs = np.ascontiguousarray(np.linspace(-2, 2, nax, dtype=F32) if centres is None else centres, F32)
    cc = np.zeros(2 * g.batch, F32)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    # addresses are never dereferenced: validation fails first
    return lib.phicuda_julia_f32(C.byref(g), None if null_centres else fp(cs), fp(cc) if c else None, iterations, C.c_void_p(counts),
                                 C.c_void_p(scratch), C.c_size_t(need - short), None)


@pytest.mark.parametrize('kw,code,word', [
    ({'counts': 0}, _lib.ERR_INVALID, 'NULL'),
    ({'scratch': 0}, _lib.ERR_INVALID, 'NULL'),
    ({'c': False}, _lib.ERR_INVALID, 'NULL'),
    ({'null_centres': True}, _lib.ERR_INVALID, 'NULL'),
    ({'short': 4}, _lib.ERR_INVALID, 'scratch'),
    ({'scratch': (16 << 20) + 64}, _lib.ERR_INVALID, 'overlaps'),
    ({'scratch': (16 << 20) - 64}, _lib.ERR_INVALID, 'overlaps'),
    ({'iterations': -1}, _lib.ERR_INVALID, 'iterations'),
    ({'centres': np.full(24, np.inf, np.float32)}, _lib.ERR_INVALID, 'cell centre'),
    ({'g': _grid(3)}, _lib.ERR_UNSUPPORTED, '2-D'),
    ({'g': _grid(batch=0)}, _lib.ERR_INVALID, 'batch'),
])
def test_argument_validation_without_gpu(kw, code, word):
    assert _call(**kw) == code
    assert word in _lib.last_error()


def test_scratch_bytes():
    g = _grid(n=(37, 23), batch=3)
    assert _lib.load().phicuda_julia_scratch_bytes(C.byref(g)) == 4 * (2 * 3 + 37 + 23)
    assert _lib.load().phicuda_julia_scratch_bytes(None) == 0


def test_kernel_id():
    assert _lib.KERNEL_JULIA == 8
