"""
The fp64 path (math.set_global_precision(64)) through libphicuda.so against oracle_np under precision(64): stencils bit for bit or
within float64 ulp bounds, semi-Lagrangian advection, the register-marching CG (truncated iterates, full solves, warm starts, batch
entries stopping independently), make_incompressible, the Taylor-Green notebook at 25^2 and the 3-D Taylor-Green vortex at 32^3.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import oracle_np as O
from oracle_fp64 import taylor_green_step
from phiflow_b200 import _lib, _ops as ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = np.finfo(np.float64).eps
F64 = torch.float64

BCS = {
    'periodic': lambda d: O.uniform_bc(d, 'periodic'),
    'zg': lambda d: O.uniform_bc(d, 'zg'),
    'zero': lambda d: O.uniform_bc(d, 0.0),
    'const': lambda d: tuple((0.7, -1.3) for _ in range(d)),
    'mix': lambda d: (('periodic', 'periodic'), ('zg', 0.25)) + ((('zg', 'zg'),) if d == 3 else ()),
    'mix2': lambda d: ((0.5, 'zg'), ('periodic', 'periodic')) + (((0.1, -0.2),) if d == 3 else ()),
}
SHAPES = {2: [((13, 9), (0.3, 0.7)), ((64, 33), (1.0, 1.0))], 3: [((9, 6, 7), (0.5, 0.25, 1.5)), ((33, 16, 12), (1.0, 1.0, 1.0))]}


def cases():
    for d in (2, 3):
        for res, dx in SHAPES[d]:
            for name in BCS:
                yield pytest.param(res, dx, name, id=f"{name}-{'x'.join(map(str, res))}")


def rng_arrays(shapes, batch, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((batch,) + tuple(s)) for s in shapes]


@pytest.mark.parametrize('res,dx,name', list(cases()))
def test_divergence_and_grad_sub_bitwise(res, dx, name):
    d, batch = len(res), 2
    vbc = BCS[name](d)
    dom = ops.Domain(res, dx, batch, vbc=vbc, dtype=F64)
    v = rng_arrays(O.staggered_shapes(res, vbc), batch, 1)
    p = rng_arrays([res], batch, 2)[0]
    dv = dom.faces_from_numpy(v, vbc)
    div = dom.centered_to_numpy(ops.divergence(dom, vbc, dv), squeeze=False)
    ops.grad_sub(dom, vbc, dv, dom.centered_from_numpy(p))
    got = dom.faces_to_numpy(dv, vbc, squeeze=False)
    with O.precision(64):
        for b in range(batch):
            ref = O.divergence_staggered([c[b] for c in v], dx, O.component_bcs(vbc, d))
            assert ref.dtype == np.float64
            np.testing.assert_array_equal(div[b], ref)
            grad = O.gradient_faces(p[b], dx, O.pressure_bc(vbc), vbc)
            for c in range(d):
                np.testing.assert_array_equal(got[c][b], v[c][b] - grad[c])


@pytest.mark.parametrize('res,dx,name', list(cases()))
def test_laplace_and_axpy_ulp(res, dx, name):
    d, batch = len(res), 2
    bc = BCS[name](d)
    dom = ops.Domain(res, dx, batch, dtype=F64)
    x = rng_arrays([res], batch, 3)[0]
    dx_ = dom.centered_from_numpy(x)
    lap = dom.centered_to_numpy(ops.laplace(dom, bc, dx_), squeeze=False)
    coeff = 0.0123
    axpy = dom.centered_to_numpy(ops.laplace_axpy(dom, bc, dx_, coeff), squeeze=False)
    assert ops.last_launch_info()['kernel'] == _lib.KERNEL_LAPLACE_MARCH
    scale = (np.abs(x).max() + max(abs(c) for ax in bc for c in ax if not isinstance(c, str)) if name in ('const', 'mix', 'mix2')
             else np.abs(x).max()) * 4 * sum(1 / h ** 2 for h in dx)
    with O.precision(64):
        for b in range(batch):
            ref = O.laplace(x[b], dx, bc)
            assert np.abs(lap[b] - ref).max() <= 8 * EPS * scale
            ref2 = x[b] + coeff * ref
            assert np.abs(axpy[b] - ref2).max() <= 8 * EPS * (np.abs(x).max() + coeff * scale)


@pytest.mark.parametrize('d', [2, 3])
@pytest.mark.parametrize('name', ['periodic', 'zg', 'const', 'mix'])
def test_semi_lagrangian_centered_and_staggered(d, name):
    res = (20, 13) if d == 2 else (12, 9, 10)
    dx = (0.5, 0.8) if d == 2 else (0.5, 0.8, 0.6)
    batch = 2
    vbc = BCS[name](d)
    lower = (0.0,) * d
    upper = tuple(n * h for n, h in zip(res, dx))
    dom = ops.Domain(res, dx, batch, vbc=vbc, dtype=F64)
    v = [1.5 * a for a in rng_arrays(O.staggered_shapes(res, vbc), batch, 4)]
    s = rng_arrays([res], batch, 5)[0]
    dt = 0.7
    dv = dom.faces_from_numpy(v, vbc)
    got_s = dom.centered_to_numpy(ops.advect_centered(dom, vbc, dv, vbc, dom.centered_from_numpy(s), dt), squeeze=False)
    got_v = dom.faces_to_numpy(ops.advect_staggered(dom, vbc, dv, vbc, dv, dt), vbc, squeeze=False)
    tol = lambda m: 4 * max(res) * EPS * m
    with O.precision(64):
        for b in range(batch):
            vb = [c[b] for c in v]
            ref = O.semi_lagrangian_centered(s[b], vbc, vb, vbc, lower, upper, dt)
            assert ref.dtype == np.float64
            assert np.abs(got_s[b] - ref).max() <= tol(np.abs(s).max())
            refv = O.semi_lagrangian_staggered(vb, vbc, vb, vbc, res, lower, upper, dt)
            for c in range(d):
                assert np.abs(got_v[c][b] - refv[c]).max() <= tol(max(np.abs(a).max() for a in v))


SYSTEMS = {'periodic': 'periodic', 'closed': 0.0, 'open': 'zg'}     # velocity boundaries: closed walls / open (Dirichlet pressure)


def poisson_case(system, d, batch, seed):
    res = (24, 17) if d == 2 else (12, 10, 9)
    dx = (0.5, 0.75) if d == 2 else (0.5, 0.75, 0.6)
    vbc = O.uniform_bc(d, SYSTEMS[system])
    rng = np.random.default_rng(seed)
    rhs = rng.standard_normal((batch,) + res) * np.array([1.0, 10.0, 0.1][:batch]).reshape((batch,) + (1,) * d)
    return res, dx, vbc, rhs


def oracle_cg(rhs, x0, res, dx, vbc, rtol, atol, max_iter):
    with O.precision(64):
        A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
        y = rhs - np.mean(rhs) if not O.is_flexible(vbc) else rhs
        return O.cg(A, y, x0, rtol, atol, max_iter)


def gpu_cg(res, dx, vbc, rhs, x0, rtol, atol, max_iter):
    batch = rhs.shape[0]
    dom = ops.Domain(res, dx, batch, vbc=vbc, dtype=F64)
    prm = ops.cg_params(vbc, rtol=rtol, atol=atol, max_iter=max_iter, dtype=F64)
    x = ops.cg_poisson(dom, vbc, dom.centered_from_numpy(rhs), dom.centered_from_numpy(x0), prm)
    info = ops.last_launch_info()
    assert info['kernel'] == _lib.KERNEL_CG_MARCH
    return dom.centered_to_numpy(x, squeeze=False), ops.read_results(dom).copy(), not O.is_flexible(vbc)


def centred(x, project):
    return x - np.mean(x) if project else x


@pytest.mark.parametrize('d', [2, 3])
@pytest.mark.parametrize('system', list(SYSTEMS))
@pytest.mark.parametrize('k', [1, 2, 3, 5, 8])
def test_cg_truncated_iterates(d, system, k):
    res, dx, vbc, rhs = poisson_case(system, d, 1, 10 + k)
    x0 = np.zeros((1,) + res)
    x, rec, proj = gpu_cg(res, dx, vbc, rhs, x0, 1e-14, 1e-14, k)
    ref = oracle_cg(rhs[0], x0[0], res, dx, vbc, 1e-14, 1e-14, k)
    assert rec['iterations'][0] == ref['iterations'] == k and not rec['converged'][0]
    xr = ref['x'].reshape(res)
    assert np.abs(centred(x[0], proj) - centred(xr, proj)).max() <= 1e-13 * np.abs(xr).max()


@pytest.mark.parametrize('d', [2, 3])
@pytest.mark.parametrize('system', list(SYSTEMS))
@pytest.mark.parametrize('rtol', [1e-12, 1e-10])
def test_cg_full_solves_batch_and_warm_start(d, system, rtol):
    batch = 3
    res, dx, vbc, rhs = poisson_case(system, d, batch, 20)
    rng = np.random.default_rng(21)
    x0 = np.zeros((batch,) + res)
    x0[1] = rng.standard_normal(res)                     # entry 1 starts warm, away from the solution
    x, rec, proj = gpu_cg(res, dx, vbc, rhs, x0, rtol, rtol, 2000)
    assert rec.dtype == ops._RESULT_DTYPE64
    for b in range(batch):
        ref = oracle_cg(rhs[b], x0[b], res, dx, vbc, rtol, rtol, 2000)
        assert ref['converged'] and rec['converged'][b] == 1 and rec['diverged'][b] == 0
        assert abs(int(rec['iterations'][b]) - ref['iterations']) <= 1, (b, rec['iterations'], ref['iterations'])
        assert rec['residual_sq'][b] <= rec['tol_sq'][b]
        assert rec['tol_sq'][b] == pytest.approx(ref['tol_sq'], rel=1e-10)
        xr = ref['x'].reshape(res)
        assert np.abs(centred(x[b], proj) - centred(xr, proj)).max() <= 1e3 * rtol * np.abs(xr).max()
    # the entries stopped independently: each batch entry's record is that of its own batch-1 solve
    for b in range(batch):
        xb, recb, _ = gpu_cg(res, dx, vbc, rhs[b:b + 1], x0[b:b + 1], rtol, rtol, 2000)
        assert abs(int(recb['iterations'][0]) - int(rec['iterations'][b])) <= 1
        assert np.abs(xb[0] - x[b]).max() <= 1e3 * rtol * np.abs(x[b]).max()


@pytest.mark.parametrize('d', [2, 3])
@pytest.mark.parametrize('system', ['periodic', 'closed', 'open'])
def test_make_incompressible(d, system):
    res = (24, 20) if d == 2 else (16, 12, 10)
    dx = (0.4, 0.3) if d == 2 else (0.4, 0.3, 0.5)
    vbc = O.uniform_bc(d, SYSTEMS[system])
    rng = np.random.default_rng(30)
    v = [rng.standard_normal(s) for s in O.staggered_shapes(res, vbc)]
    dom = ops.Domain(res, dx, 1, vbc=vbc, dtype=F64)
    dv = dom.faces_from_numpy(v, vbc)
    prm = ops.cg_params(vbc, rtol=1e-12, atol=1e-12, max_iter=3000, dtype=F64)
    dv, dp = ops.make_incompressible(dom, vbc, dv, None, prm)
    rec = ops.read_results(dom)
    assert rec['converged'][0] == 1
    div = dom.centered_to_numpy(ops.divergence(dom, vbc, dv))
    assert np.abs(div).max() <= 1e-10 / min(dx)
    with O.precision(64):
        vr, pr, info = O.make_incompressible(v, vbc, res, dx, 1e-12, 1e-12, 3000, use_matrix_offset=False)
    assert abs(int(rec['iterations'][0]) - info['iterations']) <= 1
    got = dom.faces_to_numpy(dv, vbc)
    for c in range(d):
        assert np.abs(got[c] - vr[c]).max() <= 1e-8 * max(np.abs(a).max() for a in vr)


def load_example(name):
    spec = importlib.util.spec_from_file_location(f'example_{name}', os.path.join(ROOT, 'examples', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_taylor_green_notebook():
    """examples/taylor_green.py at 25^2, all 199 steps, against the oracle's step run step for step."""
    tg = load_example('taylor_green')
    v, p, errs, iters = tg.run()
    res, dx = (tg.N, tg.N), (2 * np.pi / tg.N,) * 2
    vbc = O.uniform_bc(2, 'periodic')
    lower, upper = (0.0, 0.0), (2 * np.pi, 2 * np.pi)
    vo, po = tg.analytic_velocity(0.), tg.analytic_pressure(0.)
    oerrs, oiters = [tg.errors(vo, 0.)], []
    for k in range(tg.FRAMES - 1):
        vo, po, info = taylor_green_step(vo, po, tg.DT, tg.VISCOSITY, vbc, res, dx, lower, upper)
        assert info['converged']
        oerrs.append(tg.errors(vo, (k + 1) * tg.DT)); oiters.append(info['iterations'])
    assert len(iters) == tg.FRAMES - 1
    assert all(abs(a - b) <= 1 for a, b in zip(iters, oiters)), (iters, oiters)
    vmax = max(np.abs(c).max() for c in vo)
    for c in range(2):
        assert v[c].dtype == np.float64
        assert np.abs(v[c] - vo[c]).max() <= 1e-8 * vmax
    oerrs = np.array(oerrs)
    np.testing.assert_allclose(errs[:, 1], oerrs[:, 1], rtol=1e-6)


def test_taylor_green_3d_fp64():
    """The 3-D Taylor-Green vortex of test_config_c3_taylor_green_3d in fp64: semi_lagrangian -> make_incompressible at 32^3."""
    n = 32
    res, L = (n, n, n), 2 * np.pi
    dx = (L / n,) * 3
    lower, upper = (0.0,) * 3, (L,) * 3
    vbc = O.uniform_bc(3, 'periodic')
    ax = np.arange(n, dtype=np.float64) * dx[0]
    cc = ax + 0.5 * dx[0]
    X, Y, Z = np.meshgrid(ax, cc, cc, indexing='ij')
    u = np.sin(X) * np.cos(Y) * np.cos(Z)
    X, Y, Z = np.meshgrid(cc, ax, cc, indexing='ij')
    w = -np.cos(X) * np.sin(Y) * np.cos(Z)
    v = [u, w, np.zeros(res)]
    dom = ops.Domain(res, dx, 1, vbc=vbc, dtype=F64)
    dv, dp = dom.faces_from_numpy(v, vbc), dom.alloc_centered()
    prm = ops.cg_params(vbc, rtol=1e-12, atol=1e-12, dtype=F64)
    dt = 0.5 * dx[0]
    energy = [sum(float(np.sum(c ** 2)) for c in v)]
    p = np.zeros(res)
    for _ in range(3):
        dv2 = ops.advect_staggered(dom, vbc, dv, vbc, dv, dt)
        dv, dp = ops.make_incompressible(dom, vbc, dv2, dp, prm)
        assert ops.read_results(dom)['converged'][0] == 1
        with O.precision(64):
            v = O.semi_lagrangian_staggered(v, vbc, v, vbc, res, lower, upper, dt)
            v, p, info = O.make_incompressible(v, vbc, res, dx, 1e-12, 1e-12, x0=p, use_matrix_offset=False)
        got = dom.faces_to_numpy(dv, vbc)
        energy.append(sum(float(np.sum(c ** 2)) for c in got))
    div = dom.centered_to_numpy(ops.divergence(dom, vbc, dv))
    assert np.abs(div).max() <= 1e-10 / dx[0]
    for c in range(3):
        assert np.abs(got[c] - v[c]).max() <= 1e-9
    assert all(b <= a * (1 + 1e-12) for a, b in zip(energy, energy[1:]))
