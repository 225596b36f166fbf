"""
diffuse.implicit with a varying diffusivity without a GPU: the oracle against PhiML 1.7.2 (tests/golden/phiml_diffuse_varying.npz),
argument validation of phicuda_diffuse_implicit_varying_f32, and the mirror, examples/heat_flow.py and the facade over the
oracle-backed engine.
"""
import ctypes as C
import os

import numpy as np
import pytest

import phiflow_b200.flow as flow
from oracle_diffuse_varying import VaryingDiffuseOracleEngine, diffuse_implicit_varying, sharpen_varying, varying_system
from phiflow_b200 import _lib

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'phiml_diffuse_varying.npz')
CASES = ['zero', 'periodic', 'zg', 'mixed', 'heat', 'aniso', 'mixed3', 'back']
ULP8 = 8 * np.finfo(np.float32).eps


def _spec(arr):
    return tuple(tuple('periodic' if np.isnan(s) else ('zg' if np.isinf(s) else float(s)) for s in ax) for ax in arr)


def _case(g, name):
    return g[f'{name}/u'], g[f'{name}/k'], _spec(g[f'{name}/bc']), tuple(g[f'{name}/dx']), float(g[f'{name}/dt'])


# ---- oracle vs PhiML ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', CASES)
@pytest.mark.parametrize('tag,rtol', [('r3', 1e-3), ('r5', 1e-5)])
def test_oracle_matches_phiml(name, tag, rtol):
    g = np.load(GOLD)
    u, k, bc, dx, dt = _case(g, name)
    x, info = diffuse_implicit_varying(u, k, bc, dx, dt, rtol, 1e-5, 1000)
    ref = g[f'{name}/{tag}/x']
    assert info['iterations'] == int(g[f'{name}/{tag}/iterations'])
    assert np.abs(x - ref).max() <= ULP8 * np.abs(ref).max()


@pytest.mark.parametrize('name', [c for c in CASES if c != 'back'])
def test_golden_data_pins_the_face_rule(name):
    """Faces built as -dt * min(k) instead of the reference's min(-dt k) (for dt > 0: the face minimum of k instead of the maximum)
    miss PhiML's solution by more than 100x the tolerance above.  (For dt < 0 both rules give the same faces.)"""
    g = np.load(GOLD)
    u, k, bc, dx, dt = _case(g, name)
    x, _ = diffuse_implicit_varying(u, k, bc, dx, dt, 1e-5, 1e-5, 1000, face='k')
    ref = g[f'{name}/r5/x']
    assert np.abs(x - ref).max() > 100 * ULP8 * np.abs(ref).max()


def test_golden_data_pins_the_constant_side_coefficient():
    """Back-diffusion with c = 0.01 below w_edge: a constant side's face takes min(w_edge, c) = c.  Taking w_edge there (as if k kept
    its own ZERO_GRADIENT boundary) misses PhiML's solution by more than 100x the tolerance."""
    g = np.load(GOLD)
    u, k, bc, dx, dt = _case(g, 'back')
    assert bc[0][0] == 0.01 and float(-dt * k[0].min()) > 0.01
    coef_bc = tuple(tuple('zg' if not isinstance(s, str) else s for s in ax) for ax in bc)
    x, _ = diffuse_implicit_varying(u, k, bc, dx, dt, 1e-5, 1e-5, 1000, coef_bc=coef_bc)
    ref = g['back/r5/x']
    assert np.abs(x - ref).max() > 100 * ULP8 * np.abs(ref).max()


@pytest.mark.parametrize('name', CASES)
def test_matrix_and_bias_restate_sharpen(name):
    g = np.load(GOLD)
    u, k, bc, dx, dt = _case(g, name)
    M, y = varying_system(u, k, bc, dx, dt)
    x = np.random.default_rng(0).standard_normal(u.shape).astype(np.float32)
    bias = (u.ravel() - y).reshape(u.shape)
    np.testing.assert_allclose((M @ x.ravel()).reshape(u.shape) + bias, sharpen_varying(x, k, bc, dx, dt), atol=1e-5)
    assert abs(M - M.T).max() == 0                                             # one coefficient per face: symmetric


@pytest.mark.parametrize('tag,rtol', [('r3', 1e-3), ('r5', 1e-5)])
def test_batch_entries(tag, rtol):
    """Each entry alone is what the library computes.  PhiML runs a batch-dependent matrix as one block-diagonal CG with one stopping
    rule; that joint solve agrees with the per-entry solves to the solver tolerance."""
    g = np.load(GOLD)
    u, k, bc, dx, dt = g['batch/u'], g['batch/k'], _spec(g['batch/bc']), tuple(g['batch/dx']), float(g['batch/dt'])
    for b in range(2):
        x, info = diffuse_implicit_varying(u[b], k[b], bc, dx, dt, rtol, 1e-5, 1000)
        ref = g[f'batch/{b}/{tag}/x']
        assert info['iterations'] == int(g[f'batch/{b}/{tag}/iterations'])
        assert np.abs(x - ref).max() <= ULP8 * np.abs(ref).max()
        joint = g[f'batch/joint/{tag}/x'][b]
        assert np.abs(x - joint).max() <= 20 * rtol * np.abs(joint).max()


def test_zero_dt_and_negative_constants():
    u = np.random.default_rng(1).standard_normal((12, 8)).astype(np.float32)
    k = np.random.default_rng(2).uniform(0.01, 1.0, (12, 8)).astype(np.float32)
    x, info = diffuse_implicit_varying(u, k, ((1.0, 'zg'), ('periodic', 'periodic')), (1.0, 1.0), 0.0)
    assert info['iterations'] == 0 and np.array_equal(x, u)
    x, info = diffuse_implicit_varying(u, k, ((-0.5, 'zg'), ('periodic', 'periodic')), (1.0, 1.0), 0.0)
    assert info['iterations'] > 0 and not np.array_equal(x, u)                  # f_b = min(-0, c) = c < 0


# ---- C ABI validation (no CUDA call is reached) -----------------------------------------------------------------------------------
def _grid(batch=2):
    g = _lib.PhiGrid()
    g.dim, g.batch = 2, batch
    g.n[0], g.n[1], g.cext[0], g.cext[1], g.fext[0], g.fext[1] = 16, 8, 16, 8, 16, 8
    g.dx[0] = g.dx[1] = 1.0
    return g


def _call(g, kbatch=1, dt=0.5, null_k=False, **prm_kw):
    lib = _lib.load()
    prm = _lib.PhiCgParams()
    prm.rtol, prm.atol, prm.max_iter = 1e-5, 1e-5, 100
    for key, v in prm_kw.items():
        setattr(prm, key, v)
    bc = _lib.PhiBC()
    for a in range(2):
        bc.lo[a] = bc.hi[a] = _lib.BC_PERIODIC
    n = lib.phicuda_cg_workspace_bytes(C.byref(g))
    dummy = C.c_void_p(16)          # never dereferenced: validation fails first
    return lib.phicuda_diffuse_implicit_varying_f32(C.byref(g), C.byref(bc), None if null_k else dummy, kbatch, C.c_float(dt), dummy, dummy,
                                                    C.byref(prm), dummy, dummy, C.c_size_t(n), None)


@pytest.mark.parametrize('batch,kw,code,word', [
    (2, {'null_k': True}, _lib.ERR_INVALID, 'NULL'),
    (2, {'kbatch': 0}, _lib.ERR_INVALID, 'diffusivity_batch'),
    (3, {'kbatch': 2}, _lib.ERR_INVALID, 'diffusivity_batch'),
    (2, {'dt': float('nan')}, _lib.ERR_INVALID, 'dt'),
    (2, {'balance_rhs': 1}, _lib.ERR_INVALID, 'balance_rhs'),
    (2, {'project_mean': 1}, _lib.ERR_INVALID, 'project_mean'),
    (2, {'matrix_offset': 0.5}, _lib.ERR_INVALID, 'matrix_offset'),
    (2, {'method': 1}, _lib.ERR_UNSUPPORTED, 'PHI_SOLVER_CG'),
])
def test_argument_validation_without_gpu(batch, kw, code, word):
    assert _call(_grid(batch), **kw) == code
    assert word in _lib.last_error()


def test_grids_outside_the_ring_are_unsupported():
    g = _grid(1)
    g.n[0], g.cext[0], g.fext[0] = 65536, 65536, 65536          # a line longer than the ring's shared-memory stages
    assert _call(g) == _lib.ERR_UNSUPPORTED and 'ring' in _lib.last_error()
    g = _grid(1)
    g.dim, g.n[2], g.cext[2], g.fext[2], g.dx[2], g.halo = 3, 4, 6, 6, 1.0, 1
    assert _call(g) == _lib.ERR_UNSUPPORTED and 'z-slab' in _lib.last_error()


def test_no_cg_operator_before_a_launch():
    from phiflow_b200 import _ops
    assert _lib.load().phicuda_last_cg_operator() in (0, 1, 2, 3) and _ops.CG_OPERATORS[0] is None


# ---- the mirror and the example over the oracle engine ----------------------------------------------------------------------------
@pytest.fixture()
def oracle_mirror():
    saved = flow.ops, flow._DEVICE
    flow.ops = VaryingDiffuseOracleEngine
    flow.set_device('cpu')
    try:
        yield
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])


def test_mirror_varying(oracle_mirror):
    import test_gpu_diffuse_varying as G
    G.check_mirror_varying(flow)


def test_heat_flow_example(oracle_mirror):
    import test_gpu_diffuse_varying as G
    out = G.run_heat_flow_example()
    t, its = out['t'], out['iterations']
    assert t.shape == (100, 50) and len(its) == 100 and all(i > 0 for i in its)
    assert 0.0 <= t.min() and t.max() <= 1.0 + 1e-4 and t[0].mean() > t[-1].mean()
    assert np.allclose(np.unique(out['conductivity']), [0.01, 1.01])


# ---- the facade over the test double --------------------------------------------------------------------------------------------
def test_facade_varying():
    import test_gpu_diffuse_implicit as G
    import test_gpu_diffuse_varying as V
    with G.facade(VaryingDiffuseOracleEngine, 'cpu') as module:
        V.check_facade_varying(module)
