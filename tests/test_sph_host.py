"""
SPH (DESIGN.md row N12) without a GPU: the kernel's restatement (tests/oracle_sph.py) against PhiML's SPH substep
(tests/golden/phiml_sph.npz, tests/golden/make_sph_golden.py), the constants of _ops.sph_params, the C declaration, every argument
check of phicuda_sph_f32 (all of them run before the first CUDA call), every refusal of flow.sph_step, and examples/sph.py over the
oracle.
"""
import ctypes as C
import importlib.util
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import oracle_sph as O
import phiflow_b200.flow as flow
from phiflow_b200 import _lib, _ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'phiml_sph.npz')
F = np.float32


def cases():
    return json.loads(str(np.load(GOLD)['meta']))['cases']


def golden_params(g, name):
    x0 = g[f'{name}/x0']
    return O.notebook_params(x0.shape[1], lower=tuple(g[f'{name}/lower']), upper=tuple(g[f'{name}/upper']))


def ulps(a, b):
    return int(np.max(np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)))) if a.size else 0


@pytest.mark.parametrize('name', cases())
def test_constants_match_phiml(name):
    """s, m, P, V and the poly6 normalisation of the oracle and of _ops.sph_params equal PhiML's float32 values; s is 0.79999995, not
    h, in 3-D."""
    g = np.load(GOLD)
    prm = golden_params(g, name)
    s, m, P, V, norm = g[f'{name}/const']
    assert (prm['s'], prm['m'], prm['P'], prm['V'], prm['norm']) == (s, m, P, V, norm)
    d = g[f'{name}/x0'].shape[1]
    assert (s == F(0.79999995)) if d == 3 else (s == F(0.8))
    p = _ops.sph_params(prm['lower'], prm['upper'], 0.8, m, 0.01 * 0.8, prm['gravity'])
    assert (F(p.support), F(p.mass), F(p.pressure_norm), F(p.viscous_norm), F(p.kernel_norm)) == (s, m, P, V, norm)
    assert (F(p.dt), F(p.damping), F(p.isotropic_exp), F(p.base_density)) == (prm['dt'], prm['damping'], F(20), F(1))


@pytest.mark.parametrize('name', cases())
def test_pairs_match_phiml(name):
    """The oracle's pairs are the pairs with sqrt(r2) < s of PhiML's dense search, in the fixture's stored order; PhiML's own sparse
    search (1.7.2) finds all of them except those in the (-1, ..., -1) neighbour cell, and stores duplicates instead."""
    g = np.load(GOLD)
    prm = golden_params(g, name)
    x0 = g[f'{name}/x0']
    d = x0.shape[1]
    I, J = O.pairs(x0, prm['lower'], prm['upper'], prm['s'])
    assert np.array_equal(I, g[f'{name}/rows']) and np.array_equal(J, g[f'{name}/cols'])
    assert np.all(np.diff(I) >= 0) and set(range(len(x0))) <= set(I.tolist())     # every particle has its self pair
    res, edge = O.hash_grid(prm['lower'], prm['upper'], prm['s'], d)
    c = O.cells(x0, prm['lower'], res, edge)
    ours = set(zip(I.tolist(), J.tolist()))
    searched = set(zip(g[f'{name}/search_rows'].tolist(), g[f'{name}/search_cols'].tolist()))
    assert searched <= ours
    assert ours - searched == {(i, j) for i, j in ours if np.all(c[j] - c[i] == -1)}


def test_fixture_covers_the_edge_cases():
    """Pairs at distance exactly s (not stored: the test is <), a pair closer than sqrt(1e-5), an isolated particle, particles above
    the upper corner (the top-cell clamp) and particles leaving the box on one axis and on several."""
    g = np.load(GOLD)
    for d in (2, 3):
        name = f'special{d}_1'
        prm = golden_params(g, name)
        x0 = g[f'{name}/x0']
        I, J = O.pairs(x0, prm['lower'], prm['upper'], prm['s'])
        dist = np.sqrt(((x0[:, None] - x0[None]) ** 2).sum(-1))
        exact = np.argwhere(dist == prm['s'])
        assert len(exact) and not ({tuple(p) for p in exact.tolist()} & set(zip(I.tolist(), J.tolist())))
        close = [(i, j) for i, j in zip(I, J) if i != j and dist[i, j] < np.sqrt(1e-5)]
        assert close
        counts = np.bincount(I, minlength=len(x0))
        assert np.any(counts == 1)
        res, edge = O.hash_grid(prm['lower'], prm['upper'], prm['s'], d)
        raw = np.trunc((x0 - np.asarray(prm['lower'], F)) / edge)
        assert np.any(raw >= res)
        lo, up = np.asarray(prm['lower'], F), np.asarray(prm['upper'], F)
        x1 = g[f'{name}/x']
        left = (((x1 == lo) | (x1 == up)) & (x0 > lo) & (x0 < up)).sum(1)        # components clipped in the substep
        assert np.any(left == 1) and np.any(left >= 2)


# The reference rounds the cube of the poly6 kernel with np.power(diff, 3), the oracle (and the kernel) as (diff diff) diff:
# they differ in the last bit for about a third of all arguments on this NumPy (SIMD pow).  On the jittered lattices the results
# nevertheless agree bit for bit; on the edge-case boxes rho differs by at most 2 ulp and everything downstream accordingly.
RHO_ULPS = 4
REL = 1e-6


@pytest.mark.parametrize('name', cases())
def test_oracle_matches_phiml(name):
    g = np.load(GOLD)
    prm = golden_params(g, name)
    x0, v0 = g[f'{name}/x0'], g[f'{name}/v0']
    _, _, rho, f = O.sph_substep(x0, v0, prm)
    x, v, _ = O.sph(x0, v0, prm, int(g[f'{name}/substeps']))
    exact = name.startswith('lattice')
    if exact:
        assert np.array_equal(rho, g[f'{name}/rho']) and np.array_equal(f, g[f'{name}/force'])
        assert np.array_equal(x, g[f'{name}/x']) and np.array_equal(v, g[f'{name}/v'])
        return
    assert ulps(rho, g[f'{name}/rho']) <= RHO_ULPS
    for got, want in ((f, g[f'{name}/force']), (x, g[f'{name}/x']), (v, g[f'{name}/v'])):
        assert np.max(np.abs(got - want)) <= REL * max(1.0, float(np.abs(want).max()))


def test_oracle_rows_subset_equals_full_step():
    g = np.load(GOLD)
    name = 'special3_1'
    prm = golden_params(g, name)
    x0, v0 = g[f'{name}/x0'], g[f'{name}/v0']
    full = O.sph_substep(x0, v0, prm)
    rows = np.array([0, 5, 24, 26, 30])
    part = O.sph_substep(x0, v0, prm, rows)
    for a, b in zip(part, full):
        assert np.array_equal(a, b[rows])


def test_cells_clamp_unsafe_positions():
    """NaN, +-inf and positions far outside land in a cell of the grid (the reference would index out of range below lower)."""
    res, edge = O.hash_grid((0., 0.), (4., 4.), F(0.8), 2)
    x = np.array([[np.nan, 1.], [np.inf, -np.inf], [-1e30, 1e30], [-0.5, 3.99], [-0.9, 4.]], F)
    c = O.cells(x, (0., 0.), res, edge)
    assert np.all((c >= 0) & (c < res))
    assert c.tolist() == [[0, 1], [4, 0], [0, 4], [0, 4], [0, 4]]


# ---- the C declaration and the ABI's argument checks (no CUDA call is reached) ------------------------------------------------------
def test_declaration_matches_c():
    src = r'''#include <stdio.h>
    #include "phicuda.h"
    typedef int (*fn_t)(const float*, const float*, int64_t, int32_t, const PhiSphParams*, int32_t, float*, float*, float*, void*, size_t,
                        void*);
    typedef size_t (*bytes_t)(int64_t, int32_t, const PhiSphParams*);
    fn_t declared(void) { return phicuda_sph_f32; }     /* -Werror: the declarations have exactly these types */
    bytes_t declared_bytes(void) { return phicuda_sph_scratch_bytes; }
    #ifndef CHECK_ONLY
    int main(void) { printf("%zu %d\n", sizeof(PhiSphParams), PHI_KERNEL_SPH); return 0; }
    #endif'''
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, 'p.c'), os.path.join(d, 'p')
        open(c, 'w').write(src)
        subprocess.check_call(['gcc', '-Werror', '-DCHECK_ONLY', '-I', os.path.join(ROOT, 'include'), '-c', c, '-o', exe + '.o'])
        open(c, 'w').write(src.replace('fn_t declared(void) { return phicuda_sph_f32; }', '')
                           .replace('bytes_t declared_bytes(void) { return phicuda_sph_scratch_bytes; }', ''))
        subprocess.check_call(['gcc', '-Werror', '-I', os.path.join(ROOT, 'include'), c, '-o', exe])
        vals = [int(v) for v in subprocess.check_output([exe]).split()]
    assert vals == [C.sizeof(_lib.PhiSphParams), _lib.KERNEL_SPH]
    assert _lib.KERNEL_SPH == 10


def _prm(d=3, **kw):
    prm = O.notebook_params(d, upper=(8.,) * d)
    p = _ops.sph_params(prm['lower'], prm['upper'], 0.8, prm['m'], 0.008, prm['gravity'])
    for k, v in kw.items():
        if isinstance(v, tuple):
            getattr(p, k)[v[0]] = v[1]
        else:
            setattr(p, k, v)
    return p


def _call(n=6, dim=3, substeps=2, prm=None, null=None, alias=None, scratch_bytes=None):
    """phicuda_sph_f32 on host arrays: a refused call must return before touching them (or any device)."""
    lib = _lib.load()
    prm = _prm(dim if dim in (2, 3) else 3) if prm is None else prm
    rows = min(max(n, 1), 16)            # a refused call reads none of them
    x, v = np.zeros((rows, 3), F), np.zeros((rows, 3), F)
    xo, vo, ro = np.full_like(x, 7.0), np.full_like(v, 7.0), np.full(rows, 7.0, F)
    need = lib.phicuda_sph_scratch_bytes(min(max(n, 0), 16), dim, C.byref(prm))
    scratch = np.zeros(max(need, 1) + 64, np.uint8)
    args = dict(x=x.ctypes.data, v=v.ctypes.data, xo=xo.ctypes.data, vo=vo.ctypes.data, ro=ro.ctypes.data, scratch=scratch.ctypes.data,
                prm=C.byref(prm))
    if alias == 'xo=x':
        args['xo'] = args['x']
    if alias == 'vo=xo':
        args['vo'] = args['xo']
    if alias == 'ro=v':
        args['ro'] = args['v']
    if alias == 'scratch=vo':
        args['scratch'] = args['vo']
    if null:
        args[null] = None
    code = lib.phicuda_sph_f32(C.c_void_p(args['x']), C.c_void_p(args['v']), n, dim, args['prm'], substeps, C.c_void_p(args['xo']),
                               C.c_void_p(args['vo']), C.c_void_p(args['ro']), C.c_void_p(args['scratch']),
                               need if scratch_bytes is None else scratch_bytes, None)
    untouched = np.all(xo == 7.0) and np.all(vo == 7.0) and np.all(ro == 7.0)
    return code, untouched


NAN, INF = float('nan'), float('inf')


@pytest.mark.parametrize('kw,word', [
    ({'null': 'x'}, 'NULL'),
    ({'null': 'v'}, 'NULL'),
    ({'null': 'xo'}, 'NULL'),
    ({'null': 'vo'}, 'NULL'),
    ({'null': 'scratch'}, 'NULL'),
    ({'null': 'prm'}, 'NULL'),
    ({'dim': 1}, 'dim'),
    ({'dim': 4}, 'dim'),
    ({'n': -1}, 'n must'),
    ({'n': (1 << 30) + 1}, 'n must'),
    ({'substeps': 0}, 'substeps'),
    ({'substeps': -3}, 'substeps'),
    ({'scratch_bytes': 16}, 'scratch'),
    ({'prm': _prm(support=0.0)}, 'support'),
    ({'prm': _prm(support=-0.8)}, 'support'),
    ({'prm': _prm(support=NAN)}, 'finite'),
    ({'prm': _prm(smoothing_length=INF)}, 'finite'),
    ({'prm': _prm(kernel_norm=NAN)}, 'finite'),
    ({'prm': _prm(mass=INF)}, 'finite'),
    ({'prm': _prm(pressure_norm=NAN)}, 'finite'),
    ({'prm': _prm(viscous_norm=NAN)}, 'finite'),
    ({'prm': _prm(isotropic_exp=INF)}, 'finite'),
    ({'prm': _prm(base_density=NAN)}, 'finite'),
    ({'prm': _prm(dt=NAN)}, 'finite'),
    ({'prm': _prm(damping=-INF)}, 'finite'),
    ({'prm': _prm(lower=(0, NAN))}, 'lower'),
    ({'prm': _prm(upper=(2, INF))}, 'lower'),
    ({'prm': _prm(upper=(1, 0.0))}, 'lower'),
    ({'prm': _prm(upper=(1, -1.0))}, 'lower'),
    ({'prm': _prm(gravity=(2, NAN))}, 'gravity'),
    ({'prm': _prm(support=1e-4)}, 'hash cells'),
    ({'prm': _prm(upper=(0, 1e38), support=1.0)}, 'hash cells'),
    ({'alias': 'xo=x'}, 'overlaps'),
    ({'alias': 'vo=xo'}, 'overlap'),
    ({'alias': 'ro=v'}, 'overlaps'),
    ({'alias': 'scratch=vo'}, 'overlap'),
])
def test_argument_validation_without_gpu(kw, word):
    got, untouched = _call(**kw)
    assert got == _lib.ERR_INVALID, _lib.last_error()
    assert word in _lib.last_error()
    assert untouched


def test_no_particles_returns_before_cuda():
    got, untouched = _call(n=0)
    assert got == 0 and untouched


def test_scratch_bytes():
    lib = _lib.load()
    assert lib.phicuda_sph_scratch_bytes(10, 3, None) == 0
    assert lib.phicuda_sph_scratch_bytes(10, 5, C.byref(_prm())) == 0
    small = lib.phicuda_sph_scratch_bytes(1000, 3, C.byref(_prm()))
    assert small > 1000 * (3 * 4 + 6 * 4 + 4) and lib.phicuda_sph_scratch_bytes(2000, 3, C.byref(_prm())) > small


# ---- the mirror ---------------------------------------------------------------------------------------------------------------------
class SphOracleEngine:
    """flow.ops for sph_step on the CPU: _ops.sph_params and the oracle's substeps."""
    sph_params = staticmethod(_ops.sph_params)

    @staticmethod
    def sph(x, v, p, substeps=1):
        d = x.shape[1]
        prm = dict(lower=tuple(p.lower[:d]), upper=tuple(p.upper[:d]), s=F(p.support), h=F(p.smoothing_length), norm=F(p.kernel_norm),
                   m=F(p.mass), P=F(p.pressure_norm), V=F(p.viscous_norm), iso=F(p.isotropic_exp), base=F(p.base_density), dt=F(p.dt),
                   gravity=tuple(F(c) for c in p.gravity[:d]), damping=F(p.damping))
        xo, vo, _ = O.sph(x.numpy(), v.numpy(), prm, substeps)
        return torch.from_numpy(xo), torch.from_numpy(vo)


class _NoKernels:
    def __getattr__(self, name):
        raise AssertionError(f"ops.{name} reached by a refused call")


@pytest.fixture()
def engine():
    saved = flow.ops, flow._DEVICE
    flow.set_device('cpu')
    flow.ops = SphOracleEngine
    try:
        yield flow
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])


def load_example():
    spec = importlib.util.spec_from_file_location('sph_example', os.path.join(ROOT, 'examples', 'sph.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_example_over_the_oracle(engine):
    """examples/sph.py at a small lattice: the fused frames and the notebook's iterate loop give the oracle's bits."""
    ex = load_example()
    x0, v0 = ex.initial_state(4, 6, 4)
    assert x0.shape == (96, 3)
    prm = O.notebook_params(3)
    assert F(F(0.01) * ex.particle_volume(0.8)) == prm['m']
    want = O.sph(x0, v0, prm, 2 * 40)[:2]
    for cell in (False, True):
        x, v = ex.run(4, 6, 4, frames=2, cell=cell)
        assert np.array_equal(x, want[0]) and np.array_equal(v, want[1])
    ex.main(['--nx', '3', '--ny', '3', '--nz', '3', '--frames', '1'])


def test_mirror_returns_the_oracle(engine):
    g = np.load(GOLD)
    for name in ('special2_5', 'lattice3_1'):
        x0, v0 = g[f'{name}/x0'], g[f'{name}/v0']
        d = x0.shape[1]
        prm = golden_params(g, name)
        box = flow.Box(**{a: (float(lo), float(up)) for a, lo, up in zip('xyz', g[f'{name}/lower'], g[f'{name}/upper'])})
        x, v = flow.sph_step(x0, v0, box, 0.8, prm['m'], 0.01 * 0.8, (0., 0., -0.1) if d == 3 else (0., -0.1),
                             substeps=int(g[f'{name}/substeps']))
        want = O.sph(x0, v0, prm, int(g[f'{name}/substeps']))
        assert isinstance(x, np.ndarray) and np.array_equal(x, want[0]) and np.array_equal(v, want[1])


def test_mirror_refusals():
    saved = flow.ops
    flow.ops = _NoKernels()
    try:
        box3, box2 = flow.Box(x=8, y=8, z=8), flow.Box(x=8, y=8)
        x3 = np.zeros((5, 3), F)
        g3 = (0., 0., -0.1)
        cases = [
            lambda: flow.sph_step(x3.astype(np.float64), x3, box3, 0.8, 0.005, 0.008, g3),
            lambda: flow.sph_step(x3, x3.astype(np.float64), box3, 0.8, 0.005, 0.008, g3),
            lambda: flow.sph_step(torch.zeros(5, 3), x3, box3, 0.8, 0.005, 0.008, g3),            # a CPU tensor
            lambda: flow.sph_step(torch.zeros(5, 3, dtype=torch.float64), x3, box3, 0.8, 0.005, 0.008, g3),
            lambda: flow.sph_step((1., 2., 3.), (0., 0., 0.), box3, 0.8, 0.005, 0.008, g3),         # a vec is one point, not (N, d)
            lambda: flow.sph_step(x3, np.zeros((4, 3), F), box3, 0.8, 0.005, 0.008, g3),
            lambda: flow.sph_step(np.zeros((2, 5, 3), F), np.zeros((2, 5, 3), F), box3, 0.8, 0.005, 0.008, g3),
            lambda: flow.sph_step(x3, x3, box2, 0.8, 0.005, 0.008, (0., -0.1)),
            lambda: flow.sph_step(np.zeros((5, 1), F), np.zeros((5, 1), F), flow.Box(x=8), 0.8, 0.005, 0.008, (0.,)),
            lambda: flow.sph_step(x3, x3, box3, 0.8, 0.005, 0.008, (0., -0.1)),
            lambda: flow.sph_step(x3, x3, box3, 0.8, 0.005, 0.008, 0.1),
            lambda: flow.sph_step(x3, x3, box3, 0.8, 0.005, 0.008, g3, substeps=0),
            lambda: flow.sph_step(x3, x3, box3, 0.8, 0.005, 0.008, g3, substeps=2.0),
            lambda: flow.sph_step(x3, x3, box3, 0.8, 0.005, 0.008, g3, substeps=True),
        ]
        for i, case in enumerate(cases):
            with pytest.raises(NotImplementedError):
                case()
    finally:
        flow.ops = saved


def test_ops_refuse_float64(monkeypatch):
    monkeypatch.setattr(_ops, 'require_cuda', lambda: None)
    x = torch.zeros(4, 3)
    with pytest.raises(_lib.Unsupported, match='fp32'):
        _ops.sph(x.double(), x, _prm())
    with pytest.raises(_lib.Unsupported, match='fp32'):
        _ops.sph(x, x.double(), _prm())
