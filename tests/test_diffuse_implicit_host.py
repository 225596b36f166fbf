"""
diffuse.implicit without a GPU: the oracle against PhiML 1.7.2 (tests/golden/phiml_diffuse_implicit.npz), argument validation of
phicuda_diffuse_implicit_f32, the mirror (phiflow_b200/flow.py) over the oracle-backed engine, and the facade over the test double.
"""
import ctypes as C
import os

import numpy as np
import pytest

import phiflow_b200.flow as flow
from oracle_diffuse import DiffuseOracleEngine, diffuse_implicit
from phiflow_b200 import _lib

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'phiml_diffuse_implicit.npz')
CASES = ['zero', 'periodic', 'mixed', 'heat', 'aniso', 'mixed3']


def _spec(arr):
    return tuple(tuple('periodic' if np.isnan(s) else ('zg' if np.isinf(s) else float(s)) for s in ax) for ax in arr)


# ---- oracle vs PhiML ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', CASES)
@pytest.mark.parametrize('k', ['0.1', '5'])
@pytest.mark.parametrize('tag,rtol', [('r3', 1e-3), ('r5', 1e-5)])
def test_oracle_matches_phiml(name, k, tag, rtol):
    g = np.load(GOLD)
    u, bc, dx = g[f'{name}/u'], _spec(g[f'{name}/bc']), tuple(g[f'{name}/dx'])
    x, info = diffuse_implicit(u, bc, dx, float(g[f'{name}/k{k}/amount']), rtol, 1e-5, 1000)
    ref = g[f'{name}/k{k}/{tag}/x']
    assert info['iterations'] == int(g[f'{name}/k{k}/{tag}/iterations'])
    assert np.abs(x - ref).max() <= 8 * np.finfo(np.float32).eps * np.abs(ref).max()


@pytest.mark.parametrize('tag,rtol', [('r3', 1e-3), ('r5', 1e-5)])
def test_oracle_vector_components_are_separate_systems(tag, rtol):
    g = np.load(GOLD)
    u = g['vec2/u']
    per = (('periodic', 'periodic'),) * 2
    xs, infos = diffuse_implicit([u[..., 0], u[..., 1]], per, (1.0, 1.0), 2.0, rtol, 1e-5, 1000)
    assert [i['iterations'] for i in infos] == g[f'vec2/{tag}/iterations'].tolist()
    ref = g[f'vec2/{tag}/x']
    for c in range(2):
        assert np.abs(xs[c] - ref[..., c]).max() <= 8 * np.finfo(np.float32).eps * np.abs(ref).max()


def test_bias_only_next_to_non_zero_constants():
    u = np.zeros((6, 5), np.float32)
    x, info = diffuse_implicit(u, ((1.0, 'zg'), ('periodic', 'periodic')), (1.0, 1.0), 0.0, 1e-5, 1e-5, 1000)
    assert info['iterations'] == 0 and (x == 0).all()                  # a = 0: nothing to solve
    x, _ = diffuse_implicit(u, ((1.0, 'zg'), ('periodic', 'periodic')), (1.0, 1.0), 0.5, 1e-6, 1e-7, 1000)
    assert (x[0] > x[1]).all() and (x[1] > 0).all() and np.allclose(x, x[:, :1])    # heat flows in from x-, uniform in periodic y


# ---- C ABI validation (no CUDA call is reached) -----------------------------------------------------------------------------------
def _grid(batch=2):
    g = _lib.PhiGrid()
    g.dim, g.batch = 2, batch
    g.n[0], g.n[1], g.cext[0], g.cext[1], g.fext[0], g.fext[1] = 16, 8, 16, 8, 16, 8
    g.dx[0] = g.dx[1] = 1.0
    return g


def _call(g, components=1, **prm_kw):
    lib = _lib.load()
    prm = _lib.PhiCgParams()
    prm.rtol, prm.atol, prm.max_iter = 1e-5, 1e-5, 100
    for k, v in prm_kw.items():
        setattr(prm, k, v)
    vbc = _lib.PhiVBC()
    for c in range(3):
        for a in range(2):
            vbc.comp[c].lo[a] = vbc.comp[c].hi[a] = _lib.BC_PERIODIC
    n = lib.phicuda_cg_workspace_bytes(C.byref(g))
    dummy = C.c_void_p(16)          # never dereferenced: validation fails first
    return lib.phicuda_diffuse_implicit_f32(C.byref(g), C.byref(vbc), components, C.c_float(0.5), dummy, dummy, C.byref(prm), dummy,
                                            dummy, C.c_size_t(n), None)


@pytest.mark.parametrize('components,batch,kw,code,word', [
    (0, 2, {}, _lib.ERR_INVALID, 'components'),
    (4, 4, {}, _lib.ERR_INVALID, 'components'),
    (2, 3, {}, _lib.ERR_INVALID, 'multiple'),
    (1, 2, {'balance_rhs': 1}, _lib.ERR_INVALID, 'balance_rhs'),
    (1, 2, {'project_mean': 1}, _lib.ERR_INVALID, 'project_mean'),
    (1, 2, {'matrix_offset': 0.5}, _lib.ERR_INVALID, 'matrix_offset'),
    (1, 2, {'method': 1}, _lib.ERR_UNSUPPORTED, 'PHI_SOLVER_CG'),
])
def test_argument_validation_without_gpu(components, batch, kw, code, word):
    assert _call(_grid(batch), components, **kw) == code
    assert word in _lib.last_error()


def test_grids_outside_the_ring_are_unsupported():
    g = _grid(1)
    g.n[0], g.cext[0], g.fext[0] = 65536, 65536, 65536          # a line longer than the ring's shared-memory stages
    assert _call(g) == _lib.ERR_UNSUPPORTED and 'ring' in _lib.last_error()
    g = _grid(1)
    g.dim, g.n[2], g.cext[2], g.fext[2], g.dx[2], g.halo = 3, 4, 6, 6, 1.0, 1
    assert _call(g) == _lib.ERR_UNSUPPORTED and 'z-slab' in _lib.last_error()


# ---- the mirror over the oracle engine --------------------------------------------------------------------------------------------
@pytest.fixture()
def oracle_mirror():
    saved = flow.ops, flow._DEVICE
    flow.ops = DiffuseOracleEngine
    flow.set_device('cpu')
    try:
        yield
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])


def test_mirror_implicit_heat_flow(oracle_mirror):
    import test_gpu_diffuse_implicit as G
    G.check_mirror_heat_flow(flow)


def test_mirror_implicit_staggered_and_errors(oracle_mirror):
    import test_gpu_diffuse_implicit as G
    G.check_mirror_staggered_and_errors(flow)


def test_mirror_implicit_reference_identities(oracle_mirror):
    import test_gpu_diffuse_implicit as G
    G.check_mirror_reference_identities(flow)


# ---- the facade over the test double --------------------------------------------------------------------------------------------
def test_facade_implicit():
    import test_gpu_diffuse_implicit as G
    with G.facade(DiffuseOracleEngine, 'cpu') as module:
        G.check_facade(module)
