"""
Reaction-diffusion without a GPU: the oracle against PhiML 1.7.2 (tests/golden/phiml_reaction_diffusion.npz), the boundary records,
argument validation of phicuda_reaction_diffusion_f32, and the mirror, the notebook's own cell and examples/reaction_diffusion.py
over the oracle-backed engine.
"""
import ctypes as C

import numpy as np
import pytest

import phiflow_b200.flow as flow
import test_gpu_reaction_diffusion as G
from oracle_reaction_diffusion import ReactionDiffusionOracleEngine, reaction_diffusion
from phiflow_b200 import _lib

P, Z = 'periodic', 'zg'


# ---- oracle vs PhiML ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', G.CASES)
@pytest.mark.parametrize('steps', [1, 20])
def test_oracle_matches_phiml(name, steps):
    """PhiML forms f + k in float64 and casts it once; the oracle (and the library) add the float32 numbers.  That is the one
    difference in the operations: 1 ulp of f + k, far below the bound of one substep; after 20 substeps 20x that bound."""
    g = np.load(G.GOLD)
    u0, v0, bc, dx, prm, dt = G.golden_case(g, name)
    for b in range(u0.shape[0]):
        u, v = reaction_diffusion(u0[b], v0[b], bc, dx, dt=dt, substeps=steps, **prm)
        ru, rv = g[f'{name}/s{steps}/u'][b], g[f'{name}/s{steps}/v'][b]
        bu, bv = G.step_bound(ru, rv, bc, dx, prm, dt)
        assert np.all(np.abs(u - ru) <= steps * bu) and np.all(np.abs(v - rv) <= steps * bv)


def test_boundary_records():
    """The reference's extrapolation after one step: ZERO, ZERO_GRADIENT and PERIODIC are fixed points, a constant 0.3 drifts
    (u: 2c - c^2 = 0.51, v: c^2 = 0.09)."""
    g = np.load(G.GOLD)
    assert str(g['ext/zero/u']) == '0' and str(g['ext/zero/v']) == '0'
    assert str(g['ext/zg/u']) == 'zero-gradient' and str(g['ext/zg/v']) == 'zero-gradient'
    assert str(g['ext/periodic/u']) == 'periodic' and str(g['ext/periodic/v']) == 'periodic'
    assert float(str(g['ext/c0.3/u'])) == pytest.approx(0.51) and float(str(g['ext/c0.3/v'])) == pytest.approx(0.09)


# ---- C ABI validation (no CUDA call is reached) -----------------------------------------------------------------------------------
def _grid(dim=2, n=(16, 8, 4), halo=0):
    g = _lib.PhiGrid()
    g.dim, g.batch, g.halo = dim, 2, halo
    for a in range(dim):
        g.n[a] = n[a]
        g.cext[a] = g.fext[a] = n[a] + (2 * halo if a == 2 else 0)
        g.dx[a] = 1.0
    return g


def _vbc(spec_u, spec_v):
    from phiflow_b200 import _ops
    return _ops.make_vbc([spec_u, spec_v], 2)


def _call(g=None, spec_u=((P, P), (P, P)), spec_v=None, u=16 << 20, v=32 << 20, scratch=48 << 20, substeps=3, short=0, null_bc=False):
    lib = _lib.load()
    g = g or _grid()
    need = lib.phicuda_reaction_diffusion_scratch_bytes(C.byref(g))
    vbc = None if null_bc else C.byref(_vbc(spec_u, spec_v or spec_u))
    # addresses are never dereferenced: validation fails first (or substeps == 0 returns before any CUDA call)
    return lib.phicuda_reaction_diffusion_f32(C.byref(g), vbc, C.c_void_p(u), C.c_void_p(v), 0.19, 0.05, 0.06, 0.062, 0.5, substeps,
                                              C.c_void_p(scratch), C.c_size_t(need - short), None)


@pytest.mark.parametrize('kw,code,word', [
    ({'u': 0}, _lib.ERR_INVALID, 'NULL'),
    ({'scratch': 0}, _lib.ERR_INVALID, 'NULL'),
    ({'null_bc': True}, _lib.ERR_INVALID, 'NULL'),
    ({'short': 4}, _lib.ERR_INVALID, 'scratch'),
    ({'v': 16 << 20}, _lib.ERR_INVALID, 'distinct'),
    ({'v': (16 << 20) + 64}, _lib.ERR_INVALID, 'distinct'),
    ({'scratch': (32 << 20) - 64}, _lib.ERR_INVALID, 'overlaps'),
    ({'substeps': -1}, _lib.ERR_INVALID, 'substeps'),
    ({'spec_v': ((Z, Z), (P, P))}, _lib.ERR_UNSUPPORTED, 'agree'),
    ({'spec_u': ((0.3, 0.0), (P, P)), 'spec_v': ((0.0, 0.0), (P, P))}, _lib.ERR_UNSUPPORTED, '2c - c^2'),
    ({'spec_u': ((0.0, 0.0), (P, P)), 'spec_v': ((0.0, 0.0), (P, -1.0))}, _lib.ERR_INVALID, 'PERIODIC'),
    ({'spec_u': ((0.0, 0.0), (Z, 0.0)), 'spec_v': ((0.0, 0.0), (Z, 0.5))}, _lib.ERR_UNSUPPORTED, 'of v'),
    ({'g': _grid(3, halo=1), 'spec_u': ((P, P), (P, P), (P, P))}, _lib.ERR_UNSUPPORTED, 'z-slab'),
])
def test_argument_validation_without_gpu(kw, code, word):
    assert _call(**kw) == code
    assert word in _lib.last_error()


def test_zero_substeps_returns_before_any_cuda_call():
    assert _call(substeps=0) == 0


@pytest.mark.parametrize('dim,widest', [(2, 4096), (3, 2420)])
def test_ring_width_limit_is_named(dim, widest):
    n = (widest, 4, 4)
    assert _call(_grid(dim, n), spec_u=((P, P),) * dim, substeps=0) == 0
    g = _grid(dim, (widest + 4, 4, 4))
    assert _call(g, spec_u=((P, P),) * dim) == _lib.ERR_UNSUPPORTED
    assert f'at most {widest} cells' in _lib.last_error()


# ---- the mirror, the notebook's cell and the example over the oracle engine ------------------------------------------------------
@pytest.fixture()
def oracle_mirror():
    saved = flow.ops, flow._DEVICE
    flow.ops = ReactionDiffusionOracleEngine
    flow.set_device('cpu')
    try:
        yield
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])


def test_mirror(oracle_mirror):
    G.check_mirror(flow)


def test_example(oracle_mirror):
    G.check_example()
