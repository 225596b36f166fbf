"""
diffuse.implicit with a spatially varying diffusivity on the GPU: phicuda_diffuse_implicit_varying_f32 (two-sweep TMA-ring CG on
M = I + D0 with face coefficients min(-dt k), the constant boundary values as bias and as coefficient ghosts) against the oracle
(tests/oracle_diffuse_varying.py varying_system, pinned to PhiML 1.7.2 by tests/golden/phiml_diffuse_varying.npz), then the mirror, the
facade and examples/heat_flow.py on the real engine.  The check_* functions are shared with tests/test_diffuse_varying_host.py, which
runs them over the oracle-backed engine.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oracle_diffuse_varying import diffuse_implicit_varying as oracle_varying
from phiflow_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BCS_2D = {
    'zero': ((0.0, 0.0), (0.0, 0.0)),
    'periodic': (('periodic', 'periodic'), ('periodic', 'periodic')),
    'zg': (('zg', 'zg'), ('zg', 'zg')),
    'heat': ((1.0, 'zg'), ('periodic', 'periodic')),
    'mixed': (('zg', -0.5), (2.0, 'zg')),
    'consts': ((0.75, -0.02), (-0.3, 0.4)),
}
BCS_3D = {
    'mixed3': (('periodic', 'periodic'), (0.5, 'zg'), ('zg', -0.05)),
    'const3': ((1.0, -1.0), ('zg', 'zg'), (0.25, 'zg')),
    'periodic3': (('periodic', 'periodic'),) * 3,
}


def _ops():
    from phiflow_b200 import _ops
    return _ops


def _field(res, batch=1, seed=0):
    return np.random.default_rng(seed).standard_normal((batch,) + tuple(res)).astype(np.float32)


def blocky_k(res, batch=1, seed=0, contrast=100.0, base=0.01):
    """Background `base` with a few axis-aligned blocks of base * contrast (Heat_Flow's bars)."""
    rng = np.random.default_rng(seed)
    k = np.full((batch,) + tuple(res), base, np.float32)
    for b in range(batch):
        for _ in range(3):
            lo = [int(rng.integers(0, n)) for n in res]
            hi = [int(min(n, l + rng.integers(1, max(2, n // 2) + 1))) for l, n in zip(lo, res)]
            k[(b,) + tuple(slice(l, h) for l, h in zip(lo, hi))] = base * contrast
    return k


def gpu_solve(res, dx, spec, u, k, dt, rtol=1e-5, atol=1e-5, max_iter=1000, x0=None):
    """u: (batch, *res), k: (1 or batch, *res).  Returns (x, records, launch info, operator)."""
    ops = _ops()
    dom = ops.Domain(res, dx, u.shape[0])
    du = dom.centered_from_numpy(u)
    kdom = ops.Domain(res, dx, k.shape[0])
    dk = kdom.centered_from_numpy(k)
    dx0 = None if x0 is None else dom.centered_from_numpy(x0)
    out = ops.diffuse_implicit_varying(dom, spec, du, dk, dt, rtol, atol, max_iter, x0=dx0)
    info, op = ops.last_launch_info(), ops.last_cg_operator()
    rec = ops.read_results(dom)
    assert np.array_equal(dom.centered_to_numpy(du, squeeze=False), u)                # inputs untouched
    assert np.array_equal(kdom.centered_to_numpy(dk, squeeze=False), k)
    if x0 is not None:
        assert np.array_equal(dom.centered_to_numpy(dx0, squeeze=False), x0)
    return dom.centered_to_numpy(out, squeeze=False), rec, info, op


def _check_launch(info, op):
    assert info['kernel'] == _lib.KERNEL_CG_RING and info['passes'] == 2 and info['generic'] == 1
    assert op == 'helmholtz_varying'


# ---- truncated iterates: the operator, the bias and the update order per iteration ----------------------------------------------
TRUNC = [((21, 13), (1.0, 1.0), n, 1.0) for n in BCS_2D] + [((19, 7, 6), (1.0, 1.0, 1.0), n, 0.5) for n in BCS_3D] + [
    ((256, 16), (1.0, 1.0), 'periodic', 1.0),                      # full-width lines (branch-free tiling for the other operators)
    ((256, 8, 8), (1.0, 1.0, 1.0), 'periodic3', 1.0),
    ((24, 16), (0.5, 0.25), 'mixed', 0.01),                         # anisotropic dx: dt k / dx^2 = 0.0016 .. 1.6
    ((24, 16), (0.5, 0.25), 'consts', 0.05),
    ((37, 5, 9), (0.5, 1.0, 0.25), 'const3', 0.02),
]


@pytest.mark.gpu
@pytest.mark.parametrize('res,dx,name,dt', TRUNC)
def test_truncated_iterates_match_oracle(res, dx, name, dt):
    spec = {**BCS_2D, **BCS_3D}[name]
    u = _field(res, 1, seed=len(res) * 7 + res[0])
    k = blocky_k(res, 1, seed=res[1])
    for its in (1, 2, 3, 4, 7):
        x, rec, info, op = gpu_solve(res, dx, spec, u, k, dt, rtol=0.0, atol=0.0, max_iter=its)
        ref, oinfo = oracle_varying(u[0], k[0], spec, dx, dt, 0.0, 0.0, its)
        _check_launch(info, op)
        assert rec['iterations'][0] == oinfo['iterations'] == its
        scale = np.abs(ref).max()
        assert np.abs(x[0] - ref).max() <= 2e-5 * scale, (its, np.abs(x[0] - ref).max(), scale)


# ---- full solves ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('rtol', [1e-3, 1e-5])
@pytest.mark.parametrize('res,dx,name,dt', [((40, 24), (1.0, 1.0), 'heat', 1.0), ((40, 24), (1.0, 1.0), 'consts', 0.3),
                                             ((24, 16, 20), (1.0, 1.0, 1.0), 'mixed3', 2.0), ((256, 32), (1.0, 1.0), 'periodic', 8.0)])
def test_full_solve_matches_oracle(res, dx, name, dt, rtol):
    spec = {**BCS_2D, **BCS_3D}[name]
    u = _field(res, 1, seed=3)
    k = blocky_k(res, 1, seed=4)
    x, rec, info, op = gpu_solve(res, dx, spec, u, k, dt, rtol=rtol)
    _check_launch(info, op)
    ref, oinfo = oracle_varying(u[0], k[0], spec, dx, dt, rtol, 1e-5, 1000)
    assert rec['converged'][0] == 1 and oinfo['converged']
    assert rec['residual_sq'][0] <= rec['tol_sq'][0]
    assert abs(int(rec['iterations'][0]) - oinfo['iterations']) <= max(2, 0.1 * oinfo['iterations'])
    assert np.abs(x[0] - ref).max() <= 20 * rtol * np.abs(ref).max()


@pytest.mark.gpu
@pytest.mark.parametrize('shared', [False, True])
def test_batch_entries_with_own_and_broadcast_k(shared):
    res, dx, spec = (48, 32), (1.0, 1.0), BCS_2D['mixed']
    u = _field(res, 3, seed=5)
    u[1] = np.cumsum(np.cumsum(u[1], 0), 1) * 0.01                  # smooth: stops at another iteration
    k = blocky_k(res, 1 if shared else 3, seed=6)
    x, rec, info, op = gpu_solve(res, dx, spec, u, k, 2.0, rtol=1e-5)
    _check_launch(info, op)
    its = []
    for b in range(3):
        ref, oinfo = oracle_varying(u[b], k[0 if shared else b], spec, dx, 2.0, 1e-5, 1e-5, 1000)
        assert rec['converged'][b] == 1 and abs(int(rec['iterations'][b]) - oinfo['iterations']) <= max(2, 0.1 * oinfo['iterations'])
        assert np.abs(x[b] - ref).max() <= 2e-4 * np.abs(ref).max()
        its.append(int(rec['iterations'][b]))
    assert len(set(its)) > 1, its
    x, rec, _, _ = gpu_solve(res, dx, spec, u, k, 2.0, rtol=0.0, atol=0.0, max_iter=3)      # truncated: each entry its own CG
    for b in range(3):
        ref, _ = oracle_varying(u[b], k[0 if shared else b], spec, dx, 2.0, 0.0, 0.0, 3)
        assert np.abs(x[b] - ref).max() <= 2e-5 * np.abs(ref).max()


@pytest.mark.gpu
def test_back_diffusion_with_constant_below_the_edge_coefficient():
    """dt < 0: w = -dt k > 0, and the constant side x- = 0.01 lies below w_edge, so its face takes min(w_edge, c) = c."""
    res, dx, spec, dt = (32, 20), (1.0, 1.0), ((0.01, 'zg'), ('zg', 0.0)), -0.05
    u = _field(res, 1, seed=12)
    k = np.random.default_rng(13).uniform(0.5, 1.0, (1,) + res).astype(np.float32)
    for its in (1, 3):
        x, rec, info, op = gpu_solve(res, dx, spec, u, k, dt, rtol=0.0, atol=0.0, max_iter=its)
        ref, _ = oracle_varying(u[0], k[0], spec, dx, dt, 0.0, 0.0, its)
        assert np.abs(x[0] - ref).max() <= 2e-5 * np.abs(ref).max()
    x, rec, info, op = gpu_solve(res, dx, spec, u, k, dt, rtol=1e-5)
    ref, oinfo = oracle_varying(u[0], k[0], spec, dx, dt, 1e-5, 1e-5, 1000)
    _check_launch(info, op)
    assert rec['converged'][0] == 1 and abs(int(rec['iterations'][0]) - oinfo['iterations']) <= 2
    assert np.abs(x[0] - ref).max() <= 2e-4 * np.abs(ref).max()


# ---- edge cases and identities ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_aliased_x_and_y():
    ops = _ops()
    res, dx, spec = (40, 24), (1.0, 1.0), BCS_2D['heat']
    u = _field(res, 2, seed=8)
    k = blocky_k(res, 2, seed=9)
    dom = ops.Domain(res, dx, 2)
    t, dk = dom.centered_from_numpy(u), dom.centered_from_numpy(k)
    ws, _ = dom.workspace()
    prm = _lib.PhiCgParams()
    prm.rtol, prm.atol, prm.max_iter = 1e-5, 1e-5, 1000
    code = _lib.load().phicuda_diffuse_implicit_varying_f32(C.byref(dom.grid), C.byref(ops.make_bc(spec)), ops._ptr(dk), 2, C.c_float(1.5),
                                                            ops._ptr(t), ops._ptr(t), C.byref(prm), ops._ptr(dom.results()), ops._ptr(ws),
                                                            C.c_size_t(ws.numel()), ops._stream())
    _lib.check(code)
    got = dom.centered_to_numpy(t, squeeze=False)
    for b in range(2):
        ref, _ = oracle_varying(u[b], k[b], spec, dx, 1.5, 1e-5, 1e-5, 1000)
        assert np.abs(got[b] - ref).max() <= 2e-4 * np.abs(ref).max()


@pytest.mark.gpu
def test_zero_dt():
    res, dx = (40, 24), (1.0, 1.0)
    u = _field(res, 2, seed=14)
    k = blocky_k(res, 1, seed=15)
    for spec in (BCS_2D['heat'], BCS_2D['zero'], ((0.5, 'zg'), (0.0, 2.0))):         # constants >= 0: sharpen = identity
        x, rec, _, _ = gpu_solve(res, dx, spec, u, k, 0.0)
        assert (rec['iterations'] == 0).all() and np.array_equal(x, u)
    # a negative constant c: f_b = min(-0, c) = c, so the operator is not the identity (the oracle agrees)
    spec = ((-0.5, 'zg'), ('periodic', 'periodic'))
    x, rec, info, op = gpu_solve(res, dx, spec, u, k, 0.0)
    ref, oinfo = oracle_varying(u[0], k[0], spec, dx, 0.0, 1e-5, 1e-5, 1000)
    assert oinfo['iterations'] > 0 and rec['iterations'][0] > 0 and not np.array_equal(x, u)
    assert np.abs(x[0] - ref).max() <= 2e-4 * np.abs(ref).max()


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['heat', 'periodic', 'zg', 'mixed3'])
def test_constant_k_agrees_with_the_scalar_solve(name):
    """k = const: min(-dt k, -dt k) = -dt k on every face, and every constant c >= -dt k keeps f_b = -dt k."""
    spec = {**BCS_2D, **BCS_3D}[name]
    res = (40, 24) if len(spec) == 2 else (24, 16, 20)
    dx = (1.0,) * len(res)
    u = _field(res, 1, seed=16)
    kval, dt = 0.7, 1.5
    x, rec, _, _ = gpu_solve(res, dx, spec, u, np.full((1,) + res, kval, np.float32), dt, rtol=1e-5)
    ops = _ops()
    dom = ops.Domain(res, dx, 1)
    xs = dom.centered_to_numpy(ops.diffuse_implicit(dom, spec, dom.centered_from_numpy(u), kval * dt, 1e-5, 1e-5, 1000), squeeze=False)
    rs = ops.read_results(dom)
    assert ops.last_cg_operator() == 'helmholtz'
    assert abs(int(rec['iterations'][0]) - int(rs['iterations'][0])) <= 2
    assert np.abs(x - xs).max() <= 2e-4 * np.abs(xs).max()


@pytest.mark.gpu
@pytest.mark.parametrize('spec', [BCS_2D['periodic'], BCS_2D['zg'], BCS_3D['periodic3'], (('periodic', 'periodic'), ('zg', 'zg'))])
def test_conservation(spec):
    res = (48, 32) if len(spec) == 2 else (32, 16, 12)
    u = _field(res, 1, seed=17) + 1.0
    k = blocky_k(res, 1, seed=18)
    x, rec, _, _ = gpu_solve(res, (1.0,) * len(res), spec, u, k, 3.0, rtol=1e-6, atol=1e-7)
    assert abs(float(x.sum(dtype=np.float64)) - float(u.sum(dtype=np.float64))) <= 1e-4 * np.abs(u).sum()


@pytest.mark.gpu
@pytest.mark.parametrize('spec', [BCS_2D['heat'], BCS_2D['consts'], BCS_3D['const3']])
def test_maximum_principle(spec):
    res = (40, 24) if len(spec) == 2 else (24, 16, 12)
    u = np.random.default_rng(19).uniform(-1.0, 2.0, (1,) + res).astype(np.float32)
    k = blocky_k(res, 1, seed=20)
    x, rec, _, _ = gpu_solve(res, (1.0,) * len(res), spec, u, k, 2.0, rtol=1e-6, atol=1e-7)
    consts = [s for ax in spec for s in ax if not isinstance(s, str)]
    lo, hi = min([u.min()] + consts), max([u.max()] + consts)
    assert x.min() >= lo - 1e-4 and x.max() <= hi + 1e-4


# ---- the mirror, the facade and the example ------------------------------------------------------------------------------------
def check_mirror_varying(flow):
    """Heat_Flow's boundary with a bars-like conductivity, per-entry and shared k, x0, NotConverged, and what stays unsupported."""
    res, box = (32, 16), flow.Box(x=8, y=4)
    u = _field(res, 2, seed=21)
    bnd = {'x-': 1, 'x+': flow.ZERO_GRADIENT, 'y': flow.PERIODIC}
    grid = flow.CenteredGrid(u, bnd, box, batch=2, x=32, y=16)
    bars = flow.union(flow.Box(x=(0, 8), y=(1.5, 2)), flow.Box(x=(3.5, 4.5), y=(0.5, 3.5)))
    cond = flow.CenteredGrid(bars, flow.ZERO_GRADIENT, box, x=32, y=16) + .01
    kn = cond.numpy()
    assert np.allclose(np.unique(kn), [0.01, 1.01])
    before = grid.numpy().copy()
    spec = grid.spec
    with flow.SolveTape() as tape:
        out = flow.diffuse.implicit(grid, cond, 0.5, flow.Solve('CG', 1e-5, 1e-5))
    assert isinstance(out, flow.CenteredGrid) and out.boundary == grid.boundary and np.array_equal(grid.numpy(), before)
    for b in range(2):
        ref, oinfo = oracle_varying(u[b], kn, spec, grid.dx, 0.5, 1e-5, 1e-5, 1000)
        assert np.abs(out.numpy()[b] - ref).max() <= 2e-4 * np.abs(ref).max()
        assert abs(int(tape[0].iterations[b]) - oinfo['iterations']) <= 2
    assert tape[0].converged.all()
    kb = np.stack([kn, 2 * kn])                                                          # one k per entry
    condb = flow.CenteredGrid(kb, flow.ZERO, box, batch=2, x=32, y=16)
    out = flow.diffuse.implicit(grid, condb, 0.5)
    for b in range(2):
        ref, _ = oracle_varying(u[b], kb[b], spec, grid.dx, 0.5, 1e-5, 1e-5, 1000)
        assert np.abs(out.numpy()[b] - ref).max() <= 2e-4 * np.abs(ref).max()
    out = flow.diffuse.implicit(grid, cond, 0.5, flow.Solve('CG', 1e-5, 1e-5, x0=grid * 0.0))
    ref, _ = oracle_varying(u[0], kn, spec, grid.dx, 0.5, 1e-5, 1e-5, 1000, x0=np.zeros(res, np.float32))
    assert np.abs(out.numpy()[0] - ref).max() <= 2e-4 * np.abs(ref).max()
    with pytest.raises(flow.NotConverged):
        flow.diffuse.implicit(grid, cond, 0.5, flow.Solve('CG', 1e-7, 1e-9, max_iterations=2))
    v = flow.StaggeredGrid(0, flow.PERIODIC, box, x=32, y=16)
    for call in (lambda: flow.diffuse.implicit(grid, flow.CenteredGrid(1, x=16, y=8), 0.5),                  # other grid
                 lambda: flow.diffuse.implicit(grid, flow.CenteredGrid(kn[None].repeat(3, 0), bounds=box, batch=3, x=32, y=16), 0.5),
                 lambda: flow.diffuse.implicit(v, cond, 0.5),
                 lambda: flow.diffuse.implicit(grid, cond, 0.5, flow.Solve('biCG-stab(2)'))):
        with pytest.raises(NotImplementedError, match='fast path'):
            call()


def run_heat_flow_example():
    """examples/heat_flow.py: returns (final temperature, per-step iteration counts, conductivity, boundary spec, dx)."""
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    try:
        import importlib
        import heat_flow
        importlib.reload(heat_flow)
        return heat_flow.run()
    finally:
        sys.path.remove(os.path.join(ROOT, 'examples'))


def check_heat_flow_example():
    """The example's 100 steps against the oracle stepping its own trajectory: max |dt| <= 1e-3 at the end; CG iteration counts per
    step within max(2, 15 %) and in total within 8 %.  These solves take 70-90 iterations at a condition number of about 10^3 and
    stop at rtol 1e-5, near fp32's floor.  On one H100 the kernel took 8780 iterations over the 100 steps against the oracle's 9240
    (worst step 11.8 % apart, final max |dt| 1.7e-6); the kernel accumulates its dot products in fp64 partial sums, the oracle in
    fp32, which is the likely reason it stops a few iterations earlier."""
    out = run_heat_flow_example()
    t, its, k, spec, dx = out['t'], out['iterations'], out['conductivity'], out['spec'], out['dx']
    ref = np.zeros_like(k)
    oits = []
    for s in range(len(its)):
        ref, oinfo = oracle_varying(ref, k, spec, dx, 1.0, 1e-5, 1e-5, 1000, x0=ref)
        oits.append(oinfo['iterations'])
    dev = [abs(a - b) / b for a, b in zip(its, oits)]
    print(f"heat flow: iterations gpu {sum(its)} oracle {sum(oits)}, worst step {max(dev):.3f}, max|dt| {np.abs(t - ref).max():.2e}")
    assert all(abs(a - b) <= max(2, 0.15 * b) for a, b in zip(its, oits)), list(zip(its, oits))
    assert abs(sum(its) - sum(oits)) <= 0.08 * sum(oits)
    assert np.abs(t - ref).max() <= 1e-3
    assert 0.0 <= t.min() and t.max() <= 1.0 + 1e-4 and t[0].mean() > t[-1].mean()       # heat flows in from x- = 1


def check_facade_varying(flow):
    import phi
    from phiml import math
    from phiml.math import extrapolation as E, spatial, batch, channel
    rng = np.random.default_rng(41)
    box = flow.Box(x=32, y=16)
    a = rng.standard_normal((2, 32, 16)).astype(np.float32)
    kn = blocky_k((32, 16), 1, seed=42)[0]
    ext = E.combine_sides(x=(E.ConstantExtrapolation(1.0), E.ZERO_GRADIENT), y=E.PERIODIC)
    u = flow.CenteredGrid(math.tensor(a, batch(b=2) & spatial(x=32, y=16)), ext, box, x=32, y=16)
    kf = flow.CenteredGrid(math.tensor(kn, spatial(x=32, y=16)), E.ZERO_GRADIENT, box, x=32, y=16)
    spec = ((1.0, 'zg'), ('periodic', 'periodic'))
    for diffusivity in (kf, math.tensor(kn, spatial(x=32, y=16))):                     # a centred Field and a spatial Tensor
        del flow.FALLTHROUGH_LOG[:]
        with math.SolveTape() as tape:
            out = flow.diffuse.implicit(u, diffusivity, 1.0, flow.Solve('CG', 1e-5, 1e-5))
        assert not flow.FALLTHROUGH_LOG and out.extrapolation is ext and not out.is_staggered
        for b in range(2):
            ref, _ = oracle_varying(a[b], kn, spec, (1.0, 1.0), 1.0, 1e-5, 1e-5, 1000)
            np.testing.assert_allclose(out.values.b[b].numpy('x,y'), ref, atol=2e-4 * np.abs(ref).max())
        assert tape[0].method == 'phicuda' and tape[0].iterations.shape.names == ('b',) and bool(tape[0].converged.all)
    kb = np.stack([kn, 3 * kn])                                                        # per-entry k (batch dims of the field)
    out = flow.diffuse.implicit(u, math.tensor(kb, batch(b=2) & spatial(x=32, y=16)), 1.0, flow.Solve('CG', 1e-5, 1e-5))
    assert not flow.FALLTHROUGH_LOG
    for b in range(2):
        ref, _ = oracle_varying(a[b], kb[b], spec, (1.0, 1.0), 1.0, 1e-5, 1e-5, 1000)
        np.testing.assert_allclose(out.values.b[b].numpy('x,y'), ref, atol=2e-4 * np.abs(ref).max())
    with pytest.raises(math.NotConverged):
        flow.diffuse.implicit(u, kf, 1.0, flow.Solve('CG', 1e-7, 1e-9, max_iterations=2))
    # ineligible -> stock, with a reason
    uv = flow.CenteredGrid(math.tensor(rng.standard_normal((32, 16, 2)).astype(np.float32), spatial(x=32, y=16) & channel(vector='x,y')),
                           E.PERIODIC, box, x=32, y=16)
    st = flow.StaggeredGrid(math.stack([math.tensor(a[0], spatial(x=32, y=16))] * 2, math.dual(vector='x,y')), E.PERIODIC, box, x=32, y=16)
    other = flow.CenteredGrid(math.tensor(kn[:16], spatial(x=16, y=16)), E.ZERO_GRADIENT, flow.Box(x=16, y=16), x=16, y=16)
    cases = [((uv, kf, 1.0), 'channel'),
             ((st, kf, 1.0), 'StaggeredGrid'),
             ((u, other, 1.0), 'different grid'),
             ((u, math.tensor(kn[:16], spatial(x=16, y=16)), 1.0), 'different grid'),
             ((u, math.tensor(np.stack([kn, kn], -1), spatial(x=32, y=16) & channel(vector='x,y')), 1.0), 'diffusivity dims'),
             ((u, math.tensor(kb, batch(c=2) & spatial(x=32, y=16)), 1.0), 'batch dims'),
             ((u, kf, 1.0, flow.Solve('biCG-stab(2)', 1e-5, 1e-5)), 'solver')]
    for args, word in cases:
        del flow.FALLTHROUGH_LOG[:], phi.STOCK_CALLS[:]
        assert flow.diffuse.implicit(*args) == 'stock implicit' and phi.STOCK_CALLS[0][0] == 'diffuse.implicit'
        assert flow.FALLTHROUGH_LOG[0][0] == 'diffuse.implicit' and word in flow.FALLTHROUGH_LOG[0][1], flow.FALLTHROUGH_LOG


@pytest.mark.gpu
def test_mirror_on_the_gpu():
    import phiflow_b200.flow as flow
    check_mirror_varying(flow)
    assert _ops().last_cg_operator() == 'helmholtz_varying'


@pytest.mark.gpu
def test_heat_flow_example_on_the_gpu():
    check_heat_flow_example()


@pytest.mark.gpu
def test_facade_on_the_gpu():
    import test_gpu_diffuse_implicit as G
    with G.facade(_ops(), 'cuda') as module:
        check_facade_varying(module)
