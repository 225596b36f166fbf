"""
diffuse.implicit on the GPU: phicuda_diffuse_implicit_f32 (two-sweep TMA-ring CG on M = I - a L0 with the constant boundary values
as bias) against the oracle (tests/oracle_diffuse.py, pinned to PhiML 1.7.2), then the mirror and the facade on the real engine.
The check_* functions are shared with tests/test_diffuse_implicit_host.py, which runs them over the oracle-backed engine.
"""
import contextlib
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from oracle import oracle_np as O
from oracle_diffuse import diffuse_implicit as oracle_implicit
from phiflow_b200 import _lib

STUBS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'stubs')

BCS_2D = {
    'zero': ((0.0, 0.0), (0.0, 0.0)),
    'periodic': (('periodic', 'periodic'), ('periodic', 'periodic')),
    'zg': (('zg', 'zg'), ('zg', 'zg')),
    'heat': ((1.0, 'zg'), ('periodic', 'periodic')),
    'mixed': (('zg', -0.5), (2.0, 'zg')),
}
BCS_3D = {
    'mixed3': (('periodic', 'periodic'), (0.0, 'zg'), ('zg', 0.5)),
    'const3': ((1.0, -1.0), ('zg', 'zg'), (0.25, 'zg')),
    'periodic3': (('periodic', 'periodic'),) * 3,
}


def _ops():
    from phiflow_b200 import _ops
    return _ops


def _field(res, batch=1, seed=0):
    return np.random.default_rng(seed).standard_normal((batch,) + tuple(res)).astype(np.float32)


def _gpu_solve(res, dx, spec, u, amount, rtol=1e-5, atol=1e-5, max_iter=1000):
    """u: (batch, *res) or a list of such per component.  Returns (x in the same form, records, launch info)."""
    ops = _ops()
    comps = u if isinstance(u, list) else [u]
    dom = ops.Domain(res, dx, comps[0].shape[0])
    dev = [dom.centered_from_numpy(c) for c in comps]
    out = ops.diffuse_implicit(dom, spec, dev if isinstance(u, list) else dev[0], amount, rtol, atol, max_iter)
    info = ops.last_launch_info()
    rec = ops.read_results(dom, len(comps)) if isinstance(u, list) and len(comps) > 1 else ops.read_results(dom)
    xs = [dom.centered_to_numpy(t, squeeze=False) for t in (out if isinstance(out, list) else [out])]
    for c, t in zip(comps, dev):                                   # inputs untouched
        assert np.array_equal(dom.centered_to_numpy(t, squeeze=False), c)
    return (xs if isinstance(u, list) else xs[0]), rec, info


# ---- truncated iterates: M, the bias and the update order per iteration ----------------------------------------------------------
TRUNC = [((21, 13), (1.0, 1.0), n, 1.0) for n in BCS_2D] + [((19, 7, 6), (1.0, 1.0, 1.0), n, 1.0) for n in BCS_3D] + [
    ((256, 16), (1.0, 1.0), 'periodic', 1.0),                       # branch-free variant
    ((256, 8, 8), (1.0, 1.0, 1.0), 'periodic3', 1.0),
    ((24, 16), (0.5, 0.25), 'mixed', 0.05),                        # anisotropic dx, a/dx^2 = 0.05 .. 50
    ((24, 16), (0.5, 0.25), 'heat', 1.0),
    ((24, 16), (0.5, 0.25), 'zero', 50.0),
]


@pytest.mark.gpu
@pytest.mark.parametrize('res,dx,name,k', TRUNC)
def test_truncated_iterates_match_oracle(res, dx, name, k):
    spec = {**BCS_2D, **BCS_3D}[name]
    amount = k * min(dx) ** 2
    u = _field(res, 1, seed=len(res) * 7 + int(k))
    for its in (1, 2, 3, 4, 7):
        x, rec, info = _gpu_solve(res, dx, spec, u, amount, rtol=0.0, atol=0.0, max_iter=its)
        ref, oinfo = oracle_implicit(u[0], spec, dx, amount, 0.0, 0.0, its)
        assert info['kernel'] == _lib.KERNEL_CG_RING and info['passes'] == 2
        if res[0] % 256 == 0:
            assert info['generic'] == 0
        assert rec['iterations'][0] == oinfo['iterations'] == its
        scale = np.abs(ref).max()
        assert np.abs(x[0] - ref).max() <= 2e-5 * scale, (its, np.abs(x[0] - ref).max(), scale)


# ---- full solves ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('rtol', [1e-3, 1e-5])
@pytest.mark.parametrize('res,dx,name,k', [((40, 24), (1.0, 1.0), 'heat', 4.0), ((40, 24), (1.0, 1.0), 'zero', 0.3),
                                            ((24, 16, 20), (1.0, 1.0, 1.0), 'mixed3', 2.0), ((256, 32), (1.0, 1.0), 'periodic', 8.0)])
def test_full_solve_matches_oracle(res, dx, name, k, rtol):
    spec = {**BCS_2D, **BCS_3D}[name]
    u = _field(res, 1, seed=3)
    x, rec, _ = _gpu_solve(res, dx, spec, u, k, rtol=rtol)
    ref, oinfo = oracle_implicit(u[0], spec, dx, k, rtol, 1e-5, 1000)
    assert rec['converged'][0] == 1 and oinfo['converged']
    assert rec['residual_sq'][0] <= rec['tol_sq'][0]
    assert abs(int(rec['iterations'][0]) - oinfo['iterations']) <= max(2, 0.1 * oinfo['iterations'])
    assert np.abs(x[0] - ref).max() <= 20 * rtol * np.abs(ref).max()


@pytest.mark.gpu
def test_batch_entries_stop_independently():
    res, dx, spec = (48, 32), (1.0, 1.0), BCS_2D['mixed']
    u = _field(res, 3, seed=5)
    u[0] = 0.01 * u[0] + 1.0                                        # almost converged at x0 = u
    u[1] = np.cumsum(np.cumsum(u[1], 0), 1) * 0.01                  # smooth
    x, rec, _ = _gpu_solve(res, dx, spec, u, 3.0, rtol=1e-5)
    its = []
    for b in range(3):
        ref, oinfo = oracle_implicit(u[b], spec, dx, 3.0, 1e-5, 1e-5, 1000)
        assert rec['converged'][b] == 1 and abs(int(rec['iterations'][b]) - oinfo['iterations']) <= max(2, 0.1 * oinfo['iterations'])
        assert np.abs(x[b] - ref).max() <= 2e-4 * np.abs(ref).max()
        its.append(int(rec['iterations'][b]))
    assert len(set(its)) > 1, its


@pytest.mark.gpu
@pytest.mark.parametrize('C_', [2, 3])
def test_components_are_separate_systems_with_their_constants(C_):
    res, dx = (32, 20, 12), (1.0, 0.5, 1.0)
    base = BCS_3D['const3']
    specs = [tuple(tuple(s if isinstance(s, str) else s + c for s in ax) for ax in base) for c in range(C_)]
    comps = [_field(res, 2, seed=10 + c) * (1 + 3 * c) for c in range(C_)]
    xs, rec, info = _gpu_solve(res, dx, specs, comps, 2.0, rtol=1e-5)
    assert info['passes'] == 2 and len(rec) == 2 * C_
    for b in range(2):
        for c in range(C_):
            ref, oinfo = oracle_implicit(comps[c][b], specs[c], dx, 2.0, 1e-5, 1e-5, 1000)
            r = rec[b * C_ + c]
            assert r['converged'] == 1 and r['residual_sq'] <= r['tol_sq']
            assert abs(int(r['iterations']) - oinfo['iterations']) <= max(2, 0.1 * oinfo['iterations'])
            assert np.abs(xs[c][b] - ref).max() <= 2e-4 * np.abs(ref).max()
    # truncated: every component follows its own CG, iteration by iteration
    xs, rec, _ = _gpu_solve(res, dx, specs, comps, 2.0, rtol=0.0, atol=0.0, max_iter=3)
    for c in range(C_):
        ref, _ = oracle_implicit(comps[c][1], specs[c], dx, 2.0, 0.0, 0.0, 3)
        assert np.abs(xs[c][1] - ref).max() <= 2e-5 * np.abs(ref).max()


# ---- edge cases ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_aliased_x_and_y_and_zero_amount():
    ops = _ops()
    res, dx, spec = (40, 24), (1.0, 1.0), BCS_2D['heat']
    u = _field(res, 2, seed=8)
    dom = ops.Domain(res, dx, 2)
    t = dom.centered_from_numpy(u)
    ws, _ = dom.workspace()
    prm = _lib.PhiCgParams()
    prm.rtol, prm.atol, prm.max_iter = 1e-5, 1e-5, 1000
    code = _lib.load().phicuda_diffuse_implicit_f32(C.byref(dom.grid), C.byref(ops.make_vbc(spec, 1)), 1, C.c_float(2.0), ops._ptr(t), ops._ptr(t),
                                                    C.byref(prm), ops._ptr(dom.results()), ops._ptr(ws), C.c_size_t(ws.numel()), ops._stream())
    _lib.check(code)
    got = dom.centered_to_numpy(t, squeeze=False)
    for b in range(2):
        ref, _ = oracle_implicit(u[b], spec, dx, 2.0, 1e-5, 1e-5, 1000)
        assert np.abs(got[b] - ref).max() <= 2e-4 * np.abs(ref).max()
    x, rec, _ = _gpu_solve(res, dx, spec, u, 0.0)
    assert (rec['iterations'] == 0).all() and np.array_equal(x, u)


def check_mirror_reference_identities(flow):
    """tests/commit/physics/test_diffuse.py:32-66 on 2-D embeddings (one periodic y line, or constant along y)."""
    grid = flow.CenteredGrid(1, flow.PERIODIC, x=5, y=5)                                  # test_constant_diffusion
    np.testing.assert_allclose(flow.diffuse.implicit(grid, 1, 1).numpy(), 1.0, atol=1e-5)
    line = np.array([1.0] * 100 + [0.0] * 100, np.float32)                              # test_equality_1d_periodic
    grid = flow.CenteredGrid(line[:, None], flow.PERIODIC, x=200, y=1)
    explicit = flow.diffuse.explicit(grid, 0.5, 1, substeps=10)
    implicit = flow.diffuse.implicit(grid, 0.5, 1)
    # implicit Euler vs 10 explicit substeps differ by O(dt^2) at the unit step (0.064 here, the same in the oracle): 0.1 as the
    # reference's bound against the Fourier solution
    assert np.abs(explicit.numpy() - implicit.numpy()).max() <= 0.1
    # back-diffusion (negative dt, M indefinite) runs the same CG: it converges here, to what the oracle's CG reaches
    back = flow.diffuse.implicit(implicit, 0.5, -1)
    ref, oinfo = oracle_implicit(implicit.numpy(), (('periodic', 'periodic'),) * 2, (1.0, 1.0), -0.5)
    assert oinfo['converged'] and np.abs(back.numpy() - ref).max() <= 1e-3
    step = np.array([1.0] * 3 + [0.0] * 18, np.float32)                                 # test_implicit_stability
    grid = flow.CenteredGrid(np.repeat(step[:, None], 4, 1), flow.PERIODIC, x=21, y=4)
    try:
        out = flow.diffuse.implicit(grid, 10, 1).numpy()
        assert out.min() >= 0 and out.max() <= 1.0001
    except flow.NotConverged:
        pass


def check_mirror_heat_flow(flow):
    """Heat_Flow.ipynb's boundary {'x-': 1, 'x+': ZERO_GRADIENT, 'y': PERIODIC}: the constant enters as the bias."""
    u = _field((32, 16), 2, seed=21)[:, :, :]
    bnd = {'x-': 1, 'x+': flow.ZERO_GRADIENT, 'y': flow.PERIODIC}
    grid = flow.CenteredGrid(u, bnd, flow.Box(x=8, y=4), batch=2, x=32, y=16)
    before = grid.numpy().copy()
    with flow.SolveTape() as tape:
        out = flow.diffuse.implicit(grid, 0.3, 0.5, flow.Solve('CG', 1e-5, 1e-5))
    assert isinstance(out, flow.CenteredGrid) and out.boundary == grid.boundary and np.array_equal(grid.numpy(), before)
    spec = grid.spec
    for b in range(2):
        ref, oinfo = oracle_implicit(u[b], spec, grid.dx, 0.15, 1e-5, 1e-5, 1000)
        assert np.abs(out.numpy()[b] - ref).max() <= 2e-4 * np.abs(ref).max()
        assert abs(int(tape[0].iterations[b]) - oinfo['iterations']) <= 2
    assert tape[0].converged.all()
    with pytest.raises(flow.NotConverged):
        flow.diffuse.implicit(grid, 0.3, 0.5, flow.Solve('CG', 1e-7, 1e-9, max_iterations=2))
    out = flow.diffuse.implicit(grid, 0.3, 0.5, flow.Solve('CG', 1e-7, 1e-9, max_iterations=2, suppress=[flow.NotConverged]))
    assert np.isfinite(out.numpy()).all()
    x0 = grid * 0.0
    out = flow.diffuse.implicit(grid, 0.3, 0.5, flow.Solve('CG', 1e-5, 1e-5, x0=x0))
    ref, _ = oracle_implicit(u[0], spec, grid.dx, 0.15, 1e-5, 1e-5, 1000, x0=np.zeros((32, 16), np.float32))
    assert np.abs(out.numpy()[0] - ref).max() <= 2e-4 * np.abs(ref).max()


def check_mirror_staggered_and_errors(flow):
    res = (16, 12)
    comps = [_field(res, 2, seed=30 + c) for c in range(2)]
    v = flow.StaggeredGrid(comps, flow.PERIODIC, batch=2, x=16, y=12)
    with flow.SolveTape() as tape:
        out = flow.diffuse.implicit(v, 1.5, 1.0, flow.Solve('CG', 1e-5, 1e-5))
    assert isinstance(out, flow.StaggeredGrid) and len(tape[0].iterations) == 4           # (batch entry, component)
    got = out.numpy()
    per = ((('periodic', 'periodic'),) * 2)
    for b in range(2):
        for c in range(2):
            ref, oinfo = oracle_implicit(comps[c][b], per, (1.0, 1.0), 1.5, 1e-5, 1e-5, 1000)
            assert np.abs(got[c][b] - ref).max() <= 2e-4 * np.abs(ref).max()
            assert abs(int(tape[0].iterations[b * 2 + c]) - oinfo['iterations']) <= 2
    walls = flow.StaggeredGrid(0, flow.ZERO, x=16, y=12)
    for call in (lambda: flow.diffuse.implicit(walls, 1, 1),                                 # test_diffuse.py:25,28
                 lambda: flow.diffuse.implicit(v, (1.0, 0.5), 1),
                 lambda: flow.diffuse.implicit(v, flow.CenteredGrid(1, x=16, y=12), 1),
                 lambda: flow.diffuse.implicit(v, 1, 1, flow.Solve('biCG-stab(2)'))):
        with pytest.raises(NotImplementedError, match='fast path'):
            call()


# ---- facade --------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def facade(engine, device):
    """The facade imported over the test double with `engine` under the adapter; undoes every global side effect."""
    from _phiml import ensure_phiml
    if not ensure_phiml():
        pytest.skip('PhiML not available (neither installed nor in oracle/_ref)')
    try:
        import phi  # noqa: F401
        if 'test-double' not in getattr(phi, '__version__', ''):
            pytest.skip('a real PhiFlow is importable here; the facade tests run on the test double')
    except ImportError:
        pass
    from phiml import backend as phiml_backend
    from phiflow_b200.phi_cuda import _adapter as A
    previous_default = phiml_backend.default_backend()
    saved = A.ENGINE, A.DEVICE
    A.ENGINE, A.DEVICE = engine, device
    sys.path.insert(0, STUBS)
    try:
        import importlib
        module = importlib.import_module('phiflow_b200.phi_cuda.flow')
        # the double's phi.physics.diffuse has no stock implicit: give the imported module one that only records the call, as the
        # double's other stock functions do (the facade looks the stock function up when it falls through)
        stub = sys.modules['phi.physics.diffuse']
        calls = sys.modules['phi'].STOCK_CALLS

        def stock_implicit(field, diffusivity, dt, solve=None, gradient=None, upwind=None, correct_skew=True, gradient_for_diffusivity=True):
            calls.append(('diffuse.implicit', (field, diffusivity, dt, solve)))
            return 'stock implicit'
        stub.implicit = stock_implicit
        yield module
    finally:
        phiml_backend.set_global_default_backend(previous_default)
        A.ENGINE, A.DEVICE = saved
        sys.path.remove(STUBS)
        for name in [m for m in sys.modules if m == 'phi' or m.startswith('phi.') or m == 'phiflow_b200.phi_cuda.flow']:
            del sys.modules[name]


def check_facade(flow):
    import phi
    from phiml import math
    from phiml.math import extrapolation as E, spatial, batch, channel, dual
    assert flow.diffuse.implicit is flow.implicit and phi.physics.diffuse.implicit is not flow.implicit
    rng = np.random.default_rng(40)
    box = flow.Box(x=32, y=16)
    # scalar CenteredGrid, Heat_Flow boundary (bias)
    a = rng.standard_normal((2, 32, 16)).astype(np.float32)
    ext = E.combine_sides(x=(E.ConstantExtrapolation(1.0), E.ZERO_GRADIENT), y=E.PERIODIC)
    u = flow.CenteredGrid(math.tensor(a, batch(b=2) & spatial(x=32, y=16)), ext, box, x=32, y=16)
    del flow.FALLTHROUGH_LOG[:]
    with math.SolveTape() as tape:
        out = flow.diffuse.implicit(u, 0.5, 1.0, flow.Solve('CG', 1e-5, 1e-5))
    assert not flow.FALLTHROUGH_LOG and out.extrapolation is ext and not out.is_staggered
    spec = ((1.0, 'zg'), ('periodic', 'periodic'))
    for b in range(2):
        ref, _ = oracle_implicit(a[b], spec, (1.0, 1.0), 0.5, 1e-5, 1e-5, 1000)
        np.testing.assert_allclose(out.values.b[b].numpy('x,y'), ref, atol=2e-4 * np.abs(ref).max())
    assert tape[0].method == 'phicuda' and tape[0].iterations.shape.names == ('b',) and bool(tape[0].converged.all)
    # CenteredGrid with a vector channel (Burgers): one system per component
    av = rng.standard_normal((32, 16, 2)).astype(np.float32)
    uv = flow.CenteredGrid(math.tensor(av, spatial(x=32, y=16) & channel(vector='x,y')), E.PERIODIC, box, x=32, y=16)
    with math.SolveTape() as tape:
        out = flow.diffuse.implicit(uv, 2.0, 1.0, flow.Solve('CG', 1e-5, 1e-5))
    assert not flow.FALLTHROUGH_LOG and out.values.shape.get_item_names('vector') == ('x', 'y')
    assert tape[0].iterations.shape.names == ('vector',)
    for c, d in enumerate('xy'):
        ref, _ = oracle_implicit(av[..., c], (('periodic', 'periodic'),) * 2, (1.0, 1.0), 2.0, 1e-5, 1e-5, 1000)
        np.testing.assert_allclose(out.values.vector[d].numpy('x,y'), ref, atol=2e-4 * np.abs(ref).max())
    # periodic StaggeredGrid
    comps = [rng.standard_normal((32, 16)).astype(np.float32) for _ in range(2)]
    vals = math.stack([math.tensor(c, spatial(x=32, y=16)) for c in comps], dual(vector='x,y'))
    st = flow.StaggeredGrid(vals, E.PERIODIC, box, x=32, y=16)
    out = flow.diffuse.implicit(st, 1.0, 1.0, flow.Solve('CG', 1e-5, 1e-5))
    assert not flow.FALLTHROUGH_LOG and out.is_staggered
    for c, d in enumerate('xy'):
        ref, _ = oracle_implicit(comps[c], (('periodic', 'periodic'),) * 2, (1.0, 1.0), 1.0, 1e-5, 1e-5, 1000)
        np.testing.assert_allclose(out.values[{'~vector': d}].numpy('x,y'), ref, atol=2e-4 * np.abs(ref).max())
    # NotConverged / suppress
    with pytest.raises(math.NotConverged):
        flow.diffuse.implicit(u, 0.5, 1.0, flow.Solve('CG', 1e-7, 1e-9, max_iterations=2))
    out = flow.diffuse.implicit(u, 0.5, 1.0, flow.Solve('CG', 1e-7, 1e-9, max_iterations=2, suppress=[math.NotConverged]))
    assert np.isfinite(out.values.numpy('b,x,y')).all()
    # ineligible -> stock, with a reason
    walls = flow.StaggeredGrid(vals, E.ZERO, box, x=32, y=16)
    cases = [((walls, 1.0, 1.0), 'non-periodic'),
             ((u, 1.0, 1.0, flow.Solve('biCG-stab(2)', 1e-5, 1e-5)), 'solver'),
             ((u, math.wrap([1.0, 0.5], batch('b')), 1.0), 'plain number'),
             ((u, 1.0, 1.0, flow.Solve('CG', 1e-5, 1e-5, preconditioner='ilu')), 'preconditioner')]
    for args, word in cases:
        del flow.FALLTHROUGH_LOG[:], phi.STOCK_CALLS[:]
        assert flow.diffuse.implicit(*args) == 'stock implicit' and phi.STOCK_CALLS[0][0] == 'diffuse.implicit'
        assert flow.FALLTHROUGH_LOG[0][0] == 'diffuse.implicit' and word in flow.FALLTHROUGH_LOG[0][1], flow.FALLTHROUGH_LOG
    with math.precision(64):
        assert flow.diffuse.implicit(u, 1.0, 1.0) == 'stock implicit' and 'precision 64' in flow.FALLTHROUGH_LOG[-1][1]


@pytest.mark.gpu
def test_mirror_on_the_gpu():
    import phiflow_b200.flow as flow
    check_mirror_heat_flow(flow)
    check_mirror_staggered_and_errors(flow)
    check_mirror_reference_identities(flow)


@pytest.mark.gpu
def test_facade_on_the_gpu():
    from phiflow_b200 import _ops
    with facade(_ops, 'cuda') as module:
        check_facade(module)
