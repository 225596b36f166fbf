"""
GPU parity tests proper: every CUDA entry point (called through the C ABI, phiflow_b200/_ops.py) against the CPU
oracle on identical seeded inputs, for every boundary type the reference tests cover
(tests/commit/physics/test_fluid.py:34-53, PhiML/tests/commit/math/test__ops.py:247-279), 2-D and 3-D, batched,
ragged sizes (not multiples of the vector width / tile sizes).

Tolerances (fp32, stated per test):
  * stencils: |err| <= 4 eps * (sum of |terms|)  -> rtol 2e-6 on the scale max|x|/dx^2
  * advection: interpolation weights differ from the reference by its own coordinate rounding, eps*resolution cells
    (the reference computes positions in world space, SURVEY.md Appendix B) -> atol = 8 eps * n_max * max|neighbour difference|
  * CG: both sides stop at |r|^2 <= max(rtol^2 |r0|^2, atol^2); solutions agree to 20*rtol*max|x|
"""
import numpy as np
import pytest
import torch

from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from phiflow_b200 import _ops as ops

EPS = float(np.finfo(np.float32).eps)

BCS2 = {
    'zero': ((0.0, 0.0), (0.0, 0.0)),
    'open': (('zg', 'zg'), ('zg', 'zg')),
    'periodic': (('periodic', 'periodic'), ('periodic', 'periodic')),
    'mixed': (('zg', 'zg'), (0.0, 'zg')),
    'per_x_wall_y': (('periodic', 'periodic'), (0.0, 0.0)),
}
BCS3 = {
    'zero3': ((0.0, 0.0),) * 3,
    'open3': (('zg', 'zg'),) * 3,
    'periodic3': (('periodic', 'periodic'),) * 3,
    'mixed3': (('periodic', 'periodic'), (0.0, 'zg'), ('zg', 0.0)),
    'wall_open3': (('periodic', 'periodic'), (0.0, 0.0), (0.0, 'zg')),
}
SCALAR_EXTRA = {'one': ((1.0, 1.0), (1.0, 1.0)), 'const_mix': ((0.5, 'zg'), (-2.0, 1.5))}
ALL_V = {**BCS2, **BCS3}
ALL_S = {**BCS2, **BCS3, **SCALAR_EXTRA}
SHAPES = {2: [(37, 22), (150, 9), (8, 5)], 3: [(21, 14, 9), (133, 10, 6)]}


def dx_of(d):
    return (0.5, 0.25) if d == 2 else (0.5, 0.25, 2.0)


def rand_staggered(rng, res, vbc, batch=None):
    shapes = O.staggered_shapes(res, vbc)
    pre = () if batch is None else (batch,)
    return [rng.standard_normal(pre + s).astype(np.float32) for s in shapes]


@pytest.mark.parametrize('name', sorted(ALL_S))
def test_laplace(name):
    bc = ALL_S[name]
    d = len(bc)
    rng = np.random.default_rng(1)
    for res in SHAPES[d]:
        for batch in (1, 3):
            dom = ops.Domain(res, dx_of(d), batch)
            a = rng.standard_normal((batch,) + res).astype(np.float32)
            out = dom.centered_to_numpy(ops.laplace(dom, bc, dom.centered_from_numpy(a)), squeeze=False)
            ref = np.stack([O.laplace(a[b], dx_of(d), bc) for b in range(batch)])
            scale = np.abs(a).max() * sum(4.0 / h ** 2 for h in dx_of(d))
            np.testing.assert_allclose(out, ref, rtol=0, atol=4 * EPS * scale)
            out2 = dom.centered_to_numpy(ops.laplace_axpy(dom, bc, dom.centered_from_numpy(a), 0.01), squeeze=False)
            np.testing.assert_allclose(out2, a + np.float32(0.01) * ref, rtol=0, atol=4 * EPS * scale)


@pytest.mark.parametrize('name', sorted(ALL_V))
def test_divergence_and_grad_sub(name):
    vbc = ALL_V[name]
    d = len(vbc)
    rng = np.random.default_rng(2)
    for res in SHAPES[d]:
        for batch in (1, 2):
            dom = ops.Domain(res, dx_of(d), batch, vbc=vbc)
            v = rand_staggered(rng, res, vbc, batch)
            dv = dom.faces_from_numpy(v, vbc)
            div = dom.centered_to_numpy(ops.divergence(dom, vbc, dv), squeeze=False)
            ref = np.stack([O.divergence_staggered([c[b] for c in v], dx_of(d), O.component_bcs(vbc, d)) for b in range(batch)])
            scale = max(np.abs(c).max() for c in v) * sum(2.0 / h for h in dx_of(d))
            np.testing.assert_allclose(div, ref, rtol=0, atol=4 * EPS * scale)
            p = rng.standard_normal((batch,) + res).astype(np.float32)
            ops.grad_sub(dom, vbc, dv, dom.centered_from_numpy(p))
            got = dom.faces_to_numpy(dv, vbc, squeeze=False)
            pbc = O.pressure_bc(vbc)
            for b in range(batch):
                grad = O.gradient_faces(p[b], dx_of(d), pbc, vbc)
                for c in range(d):
                    pscale = np.abs(p).max() * 2.0 / dx_of(d)[c] + np.abs(v[c]).max()
                    np.testing.assert_allclose(got[c][b], v[c][b] - grad[c], rtol=0, atol=4 * EPS * pscale)


def _advect_tol(res, field_arrays):
    nmax = max(res)
    dmax = max(np.abs(np.diff(a, axis=ax)).max() for a in field_arrays for ax in range(a.ndim) if a.shape[ax] > 1)
    return 8 * EPS * nmax * max(dmax, 1e-3) + 4 * EPS * max(np.abs(a).max() for a in field_arrays)


@pytest.mark.parametrize('vname', sorted(ALL_V))
@pytest.mark.parametrize('sname', ['zero', 'open', 'periodic', 'one'])
def test_advect_centered(vname, sname):
    vbc = ALL_V[vname]
    d = len(vbc)
    sbc = O.uniform_bc(d, {'zero': 0.0, 'open': 'zg', 'periodic': 'periodic', 'one': 1.0}[sname])
    if sname == 'periodic' and vname not in ('periodic', 'periodic3'):
        pytest.skip('periodic smoke only on periodic domains')
    rng = np.random.default_rng(3)
    res = SHAPES[d][0]
    dx = dx_of(d)
    lower = tuple(0.0 for _ in res)
    upper = tuple(r * h for r, h in zip(res, dx))
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    v = [c * np.float32(1.7) for c in rand_staggered(rng, res, vbc)]
    s = rng.standard_normal(res).astype(np.float32)
    dt = 0.8
    dv = dom.faces_from_numpy(v, vbc)
    ds = dom.centered_from_numpy(s)
    got = dom.centered_to_numpy(ops.advect_centered(dom, vbc, dv, sbc, ds, dt))
    ref = O.semi_lagrangian_centered(s, sbc, v, vbc, lower, upper, dt)
    with O.precision(64):
        exact = O.semi_lagrangian_centered(s, sbc, v, vbc, lower, upper, dt)
    tol = _advect_tol(res, [s])
    np.testing.assert_allclose(got, ref, rtol=0, atol=tol)
    # against exact arithmetic the kernel is at least as accurate as the reference formulation
    assert np.abs(got - exact).max() <= max(np.abs(ref - exact).max() * 1.5, 16 * EPS * np.abs(s).max())
    got_mc = dom.centered_to_numpy(ops.mac_cormack_centered(dom, vbc, dv, sbc, ds, dt))
    ref_mc = O.mac_cormack_centered(s, sbc, v, vbc, lower, upper, dt)
    # every cell: on these inputs the oracle's world-space lookups have the kernels' floors (tests/test_advect_reference_host.py),
    # so the clamp limits agree and no cell needs an allowance
    np.testing.assert_allclose(got_mc, ref_mc, rtol=0, atol=tol)


@pytest.mark.parametrize('name', sorted(ALL_S))
def test_grid_sample(name):
    """phicuda_grid_sample_f32 = math.grid_sample at caller-provided coordinates (PhiML/phiml/math/_ops.py:936-1015), the
    Backend.grid_sample entry of the reference-side plugin; oracle.grid_sample is pinned against vendored-phiml fixtures.
    Includes the reference's known answers (PhiML/tests/commit/math/test__ops.py:232-245)."""
    bc = ALL_S[name]
    d = len(bc)
    rng = np.random.default_rng(12)
    res = (23, 14) if d == 2 else (13, 9, 7)
    batch, npts = 2, 4000
    dom = ops.Domain(res, (1.0,) * d, batch)
    grid = rng.standard_normal((batch,) + res).astype(np.float32)
    # points inside, on cell boundaries, and up to 3 cells outside on every side
    coords = (rng.uniform(-3.0, 1.0, (batch, npts, d)) + rng.uniform(0, 1, (batch, npts, d)) * (np.array(res) + 2.0)).astype(np.float32)
    coords[:, :50] = np.round(coords[:, :50])
    out = ops.grid_sample(dom, bc, dom.centered_from_numpy(grid), torch.from_numpy(coords).cuda()).cpu().numpy()
    ref = np.stack([O.grid_sample(grid[b], coords[b], bc) for b in range(batch)])
    np.testing.assert_allclose(out, ref, rtol=0, atol=1e-5 * np.abs(grid).max())
    if name == 'zero':
        dom1 = ops.Domain((3, 2), (1.0, 1.0), 1)                      # test__ops.py:232-238: grid = x + y, x in (1, 2, 3), y in (0, 3)
        g = dom1.centered_from_numpy(np.array([[1.0, 4.0], [2.0, 5.0], [3.0, 6.0]], np.float32))
        pts = torch.tensor([[[0.0, 0.0], [0.5, 0.0], [0.0, 0.5], [-2.0, -1.0]]], dtype=torch.float32).cuda()
        np.testing.assert_allclose(ops.grid_sample(dom1, bc, g, pts).cpu().numpy()[0], [1.0, 1.5, 2.5, 0.0], atol=1e-6)


@pytest.mark.parametrize('vname', sorted(ALL_V))
def test_advect_staggered_self(vname):
    vbc = ALL_V[vname]
    d = len(vbc)
    rng = np.random.default_rng(4)
    for res in SHAPES[d][:2]:
        dx = dx_of(d)
        lower = tuple(0.0 for _ in res)
        upper = tuple(r * h for r, h in zip(res, dx))
        dom = ops.Domain(res, dx, 1, vbc=vbc)
        v = [c * np.float32(1.3) for c in rand_staggered(rng, res, vbc)]
        dt = 0.6
        dv = dom.faces_from_numpy(v, vbc)
        got = dom.faces_to_numpy(ops.advect_staggered(dom, vbc, dv, vbc, dv, dt), vbc)
        ref = O.semi_lagrangian_staggered(v, vbc, v, vbc, res, lower, upper, dt)
        tol = _advect_tol(res, v)
        for c in range(d):
            np.testing.assert_allclose(got[c], ref[c], rtol=0, atol=tol)


def test_self_advect_staggered_known_answer():
    """tests/commit/physics/test_advect.py:41-45 on the GPU path."""
    res = (4, 3)
    vbc = O.uniform_bc(2, 0.0)
    dom = ops.Domain(res, (1.0, 1.0), 1, vbc=vbc)
    vx = np.zeros((3, 3), np.float32)
    vy = np.array([[0, 0], [1, 1], [1, 1], [0, 0]], np.float32)
    dv = dom.faces_from_numpy([vx, vy], vbc)
    got = dom.faces_to_numpy(ops.advect_staggered(dom, vbc, dv, vbc, dv, 1.0), vbc)
    np.testing.assert_allclose(got[1].T, [[0, 0, 0, 0], [0, 1, 1, 0]], atol=1e-6)
    np.testing.assert_allclose(got[0], 0, atol=1e-6)


@pytest.mark.parametrize('vname', sorted(ALL_V))
def test_advection_identities(vname):
    """tests/commit/physics/test_advect.py:12-18: adv(f, v, 0) == adv(f, 0*v, 1) == f."""
    vbc = ALL_V[vname]
    d = len(vbc)
    rng = np.random.default_rng(5)
    res = SHAPES[d][0]
    dom = ops.Domain(res, dx_of(d), 1, vbc=vbc)
    v = rand_staggered(rng, res, vbc)
    s = rng.standard_normal(res).astype(np.float32)
    sbc = O.uniform_bc(d, 'zg')
    dv = dom.faces_from_numpy(v, vbc)
    zero = dom.alloc_faces()
    ds = dom.centered_from_numpy(s)
    for fun in (ops.advect_centered, ops.mac_cormack_centered):
        np.testing.assert_allclose(dom.centered_to_numpy(fun(dom, vbc, dv, sbc, ds, 0.0)), s, atol=1e-5)
        np.testing.assert_allclose(dom.centered_to_numpy(fun(dom, vbc, zero, sbc, ds, 1.0)), s, atol=1e-5)
    for vel, dt in ((dv, 0.0), (zero, 1.0)):
        got = dom.faces_to_numpy(ops.advect_staggered(dom, vbc, vel, vbc, dv, dt), vbc)
        for c in range(d):
            np.testing.assert_allclose(got[c], v[c], atol=1e-5)


@pytest.mark.parametrize('vname', sorted(ALL_V))
def test_buoyancy_and_axpy(vname):
    vbc = ALL_V[vname]
    d = len(vbc)
    rng = np.random.default_rng(6)
    res = SHAPES[d][0]
    dom = ops.Domain(res, dx_of(d), 2, vbc=vbc)
    sbc = O.uniform_bc(d, 'zg')
    v = rand_staggered(rng, res, vbc, 2)
    s = rng.standard_normal((2,) + res).astype(np.float32)
    factor = (0.0, 0.1) if d == 2 else (0.05, 0.0, 0.1)
    dv = dom.faces_from_numpy(v, vbc)
    ops.add_buoyancy(dom, vbc, sbc, dom.centered_from_numpy(s), factor, 0.5, dv)
    got = dom.faces_to_numpy(dv, vbc, squeeze=False)
    for b in range(2):
        for c in range(d):
            faces = O.centered_to_faces(s[b] * np.float32(factor[c]), sbc, vbc)[c]
            np.testing.assert_allclose(got[c][b], v[c][b] + faces * np.float32(0.5), rtol=0, atol=1e-6)
    y = rng.standard_normal((2,) + res).astype(np.float32)
    dy = dom.centered_from_numpy(y)
    ops.axpy_centered(dom, 0.2, dom.centered_from_numpy(s), dy)
    np.testing.assert_allclose(dom.centered_to_numpy(dy, squeeze=False), y + np.float32(0.2) * s, rtol=0, atol=1e-6)


@pytest.mark.parametrize('vname', sorted(ALL_V))
@pytest.mark.parametrize('rtol', [1e-3, 1e-5])
def test_cg_poisson(vname, rtol):
    vbc = ALL_V[vname]
    d = len(vbc)
    rng = np.random.default_rng(7)
    res = (40, 24) if d == 2 else (20, 12, 10)
    dx = dx_of(d)
    batch = 3
    dom = ops.Domain(res, dx, batch, vbc=vbc)
    rhs = rng.standard_normal((batch,) + res).astype(np.float32)
    rhs[1] *= 10.0                                     # entries converge after different iteration counts
    pbc = O.pressure_bc(vbc)
    A = O.poisson_matrix(res, dx, pbc)
    rank_def = not O.is_flexible(vbc)
    prm = ops.cg_params(vbc, rtol=rtol, atol=1e-5, max_iter=1000)
    x = ops.cg_poisson(dom, vbc, dom.centered_from_numpy(rhs), None, prm)
    got = dom.centered_to_numpy(x, squeeze=False)
    info = ops.read_results(dom)
    for b in range(batch):
        y = rhs[b] - rhs[b].mean() if rank_def else rhs[b]
        ref = O.cg(A, y, np.zeros(res, np.float32), rtol, 1e-5, 1000, None)
        assert info['converged'][b] == 1 and info['diverged'][b] == 0
        assert abs(int(info['iterations'][b]) - ref['iterations']) <= max(2, ref['iterations'] // 10), (info['iterations'][b], ref['iterations'])
        # true residual of the returned solution meets the stopping rule
        r = y.ravel() - A.dot(got[b].ravel().astype(np.float64))
        tol_sq = max(rtol ** 2 * float(np.sum(y.astype(np.float64) ** 2)), 1e-10)
        # (the recurrence residual CG tests drifts from the true residual by O(eps * cond) in fp32: allow a factor 4)
        assert float(np.sum(r * r)) <= (4 if rtol > 1e-4 else 40) * tol_sq + 1e-9
        xr = ref['x'].reshape(res)
        if rank_def:
            xr = xr - xr.mean()
            assert abs(got[b].mean()) < 1e-4 * max(1.0, np.abs(got[b]).max())
        np.testing.assert_allclose(got[b], xr, rtol=0, atol=20 * rtol * np.abs(xr).max())


@pytest.mark.parametrize('vname', ['periodic3', 'mixed3', 'periodic'])
def test_cg_truncated_iterates_match_oracle(vname):
    """The solution after exactly k iterations equals the reference recurrence for odd and even k: the ring kernel applies the
    x update only every second iteration and settles the last step at the end (Shewchuk CG, _linalg.py:72-87)."""
    vbc = ALL_V[vname]
    d = len(vbc)
    res = (64, 48) if d == 2 else (64, 12, 10)
    dx = dx_of(d)
    rng = np.random.default_rng(21)
    batch = 2
    dom = ops.Domain(res, dx, batch, vbc=vbc)
    rhs = rng.standard_normal((batch,) + res).astype(np.float32)
    rhs[1] *= 3.0
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    rank_def = not O.is_flexible(vbc)
    for k in (1, 2, 3, 4, 7):
        prm = ops.cg_params(vbc, rtol=1e-12, atol=0.0, max_iter=k)
        got = dom.centered_to_numpy(ops.cg_poisson(dom, vbc, dom.centered_from_numpy(rhs), None, prm), squeeze=False)
        info = ops.read_results(dom)
        for b in range(batch):
            y = rhs[b] - rhs[b].mean() if rank_def else rhs[b]
            ref = O.cg(A, y, np.zeros(res, np.float32), 1e-12, 0.0, k, None)
            assert info['iterations'][b] == k == ref['iterations'] and info['converged'][b] == 0
            xr = ref['x'].reshape(res)
            if rank_def:
                xr = xr - xr.mean()
            np.testing.assert_allclose(got[b], xr, rtol=0, atol=2e-5 * max(1.0, np.abs(xr).max()))


@pytest.mark.parametrize('vname', ['open', 'mixed', 'mixed3', 'periodic3'])
@pytest.mark.parametrize('rtol', [1e-3, 1e-5])
def test_cg_adaptive_matches_oracle(vname, rtol):
    """Solve('CG-adaptive') (_linalg.py:93-128; what Solve('auto') runs in PhiML 1.7): same iterates as the oracle restatement,
    which is pinned against the vendored PhiML in tests/golden/phiml_cg_adaptive.npz."""
    vbc = ALL_V[vname]
    d = len(vbc)
    rng = np.random.default_rng(9)
    res = (40, 24) if d == 2 else (20, 12, 10)
    dx = dx_of(d)
    batch = 2
    dom = ops.Domain(res, dx, batch, vbc=vbc)
    rhs = rng.standard_normal((batch,) + res).astype(np.float32)
    rhs[1] *= 5.0
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    rank_def = not O.is_flexible(vbc)
    prm = ops.cg_params(vbc, rtol=rtol, atol=1e-5, max_iter=1000, method='CG-adaptive')
    got = dom.centered_to_numpy(ops.cg_poisson(dom, vbc, dom.centered_from_numpy(rhs), None, prm), squeeze=False)
    info = ops.read_results(dom)
    for b in range(batch):
        y = rhs[b] - rhs[b].mean() if rank_def else rhs[b]
        ref = O.cg_adaptive(A, y, np.zeros(res, np.float32), rtol, 1e-5, 1000, None)
        assert info['converged'][b] == int(ref['converged']) and info['diverged'][b] == 0
        assert abs(int(info['iterations'][b]) - ref['iterations']) <= max(2, ref['iterations'] // 10), (info['iterations'][b], ref['iterations'])
        xr = ref['x'].reshape(res)
        if rank_def:
            xr = xr - xr.mean()
        np.testing.assert_allclose(got[b], xr, rtol=0, atol=20 * rtol * np.abs(xr).max())
    # truncated iterates, odd and even counts (deferred x update)
    for k in (1, 2, 3):
        prm = ops.cg_params(vbc, rtol=1e-12, atol=0.0, max_iter=k, method='CG-adaptive')
        got = dom.centered_to_numpy(ops.cg_poisson(dom, vbc, dom.centered_from_numpy(rhs), None, prm), squeeze=False)
        for b in range(batch):
            y = rhs[b] - rhs[b].mean() if rank_def else rhs[b]
            ref = O.cg_adaptive(A, y, np.zeros(res, np.float32), 1e-12, 0.0, k, None)
            xr = ref['x'].reshape(res)
            if rank_def:
                xr = xr - xr.mean()
            np.testing.assert_allclose(got[b], xr, rtol=0, atol=2e-5 * max(1.0, np.abs(xr).max()))


def test_cg_matrix_offset_matches_reference_formulation():
    """With the rank-1 offset c of _optimize.py:705-714 the iterates follow the reference's (A + c 11^T) system."""
    vbc = BCS3['periodic3']
    res, dx = (16, 12, 10), (1.0, 1.0, 1.0)
    rng = np.random.default_rng(8)
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    rhs = rng.standard_normal(res).astype(np.float32)
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    c = O.estimate_matrix_offset(A, rhs.size, np.random.default_rng(0))
    prm = ops.cg_params(vbc, rtol=1e-5, atol=1e-5, matrix_offset=c)
    got = dom.centered_to_numpy(ops.cg_poisson(dom, vbc, dom.centered_from_numpy(rhs), None, prm))
    info = ops.read_results(dom)
    ref = O.cg(A, rhs - rhs.mean(), np.zeros(res, np.float32), 1e-5, 1e-5, 1000, c)
    assert info['converged'][0] == 1
    assert abs(int(info['iterations'][0]) - ref['iterations']) <= max(2, ref['iterations'] // 10)
    np.testing.assert_allclose(got, ref['x'].reshape(res) - ref['x'].mean(), rtol=0, atol=2e-4 * np.abs(ref['x']).max())


def test_cg_known_answers_and_failure_modes():
    """PhiML/tests/commit/math/test__optimize.py:62-70 (known answer, 2 iterations) and :128-143 (not converged)."""
    vbc = (('zg', 'zg'), ('zg', 'zg'))            # open velocity boundary -> Dirichlet-0 pressure, as laplace(ZERO)
    res, dx = (3, 1), (1.0, 1e3)                  # effectively 1-D: the y terms vanish like 1/dy^2
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    rhs = np.ones(res, np.float32)
    got = dom.centered_to_numpy(ops.cg_poisson(dom, vbc, dom.centered_from_numpy(rhs), None, ops.cg_params(vbc)))
    info = ops.read_results(dom)
    np.testing.assert_allclose(got[:, 0], [-1.5, -2, -1.5], atol=1e-3)
    assert info['iterations'][0] == 2 and info['converged'][0] == 1
    # max_iterations exhausted -> converged flag stays 0 (the Python layer raises NotConverged from it)
    res2 = (32, 32)
    dom2 = ops.Domain(res2, (1.0, 1.0), 1, vbc=vbc)
    rhs2 = np.random.default_rng(0).standard_normal(res2).astype(np.float32)
    ops.cg_poisson(dom2, vbc, dom2.centered_from_numpy(rhs2), None, ops.cg_params(vbc, rtol=1e-6, atol=0, max_iter=3))
    info = ops.read_results(dom2)
    assert info['iterations'][0] == 3 and info['converged'][0] == 0 and info['diverged'][0] == 0


@pytest.mark.parametrize('big', [False, True])
@pytest.mark.parametrize('vname', ['zero', 'open', 'periodic', 'mixed', 'periodic3', 'mixed3', 'wall_open3', 'open3'])
def test_make_incompressible(vname, big):
    """tests/commit/physics/test_fluid.py:19-32: divergence after projection ~ 0; agreement with the oracle.
    big: x extent a multiple of 128 -> warp-shuffle x neighbours inside the GENERIC ring kernel (2-D 128x24 tiles mix its fast
    and boundary code paths).  The 3-D case (128, 16, 8) still runs the generic kernel on the generic consumer path: the
    branch-free instantiations need nx % 256 == 0 and are covered, with an assertion on the selected variant, by
    tests/test_gpu_variants.py."""
    vbc = ALL_V[vname]
    d = len(vbc)
    rng = np.random.default_rng(9)
    if big:
        res = (128, 24) if d == 2 else (128, 16, 8)
    else:
        res = (16, 20) if d == 2 else (12, 10, 8)
    dx = tuple(100.0 / r for r in res)
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    v = [c * np.float32(0.1) for c in rand_staggered(rng, res, vbc)]
    dv = dom.faces_from_numpy(v, vbc)
    prm = ops.cg_params(vbc, rtol=1e-5, atol=1e-5)
    dv, p = ops.make_incompressible(dom, vbc, dv, None, prm)
    info = ops.read_results(dom)
    assert info['converged'][0] == 1
    div = dom.centered_to_numpy(ops.divergence(dom, vbc, dv))
    vscale = max(np.abs(c).max() for c in v) * sum(2.0 / h for h in dx)
    assert np.abs(div).max() < max(5e-5, 1e-4 * vscale)
    v_ref, p_ref, inf = O.make_incompressible(v, vbc, res, dx, rtol=1e-5, atol=1e-5, use_matrix_offset=False)
    got = dom.faces_to_numpy(dv, vbc)
    for c in range(d):
        np.testing.assert_allclose(got[c], v_ref[c], rtol=0, atol=1e-4 * max(np.abs(v[c]).max(), 1e-3))


@pytest.mark.parametrize('vname,mac', [('zero', False), ('zero', True), ('periodic3', False), ('mixed3', True)])
def test_plume_step(vname, mac):
    """The fused incompressible_step against the oracle's restatement of the notebook step, 3 steps with warm start."""
    vbc = ALL_V[vname]
    d = len(vbc)
    res = (32, 40) if d == 2 else (16, 12, 20)
    lower = tuple(0.0 for _ in res)
    upper = tuple(100.0 for _ in res)
    dx = tuple(100.0 / r for r in res)
    sbc = O.uniform_bc(d, 'zg')
    center = (50.0, 9.5) if d == 2 else (50.0, 50.0, 9.5)
    buoy = (0.0, 0.1) if d == 2 else (0.0, 0.0, 0.1)
    inflow = O.sphere_soft_mask(center, 10.0, lower, upper, res)
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    v = [np.zeros(s, np.float32) for s in O.staggered_shapes(res, vbc)]
    s = np.zeros(res, np.float32)
    p = np.zeros(res, np.float32)
    dv, ds, dp = dom.faces_from_numpy(v, vbc), dom.centered_from_numpy(s), dom.centered_from_numpy(p)
    dinflow = dom.centered_from_numpy(inflow)
    prm = ops.cg_params(vbc, rtol=1e-3, atol=1e-5)
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    for step in range(3):
        ops.plume_step(dom, vbc, sbc, dv, ds, dp, dinflow, 0.5, 0.2, buoy, prm, mac_cormack=mac)
        v, s, p, info = O.plume_step(v, s, p, 0.5, vbc, sbc, lower, upper, res, inflow, 0.2, buoy, rtol=1e-3, atol=1e-5,
                                     smoke_advection='mac_cormack' if mac else 'semi_lagrangian', use_matrix_offset=False, matrix=A)
        assert ops.read_results(dom)['converged'][0] == 1
    np.testing.assert_allclose(dom.centered_to_numpy(ds), s, rtol=0, atol=2e-4 * max(np.abs(s).max(), 1e-3))
    got = dom.faces_to_numpy(dv, vbc)
    vmax = max(np.abs(c).max() for c in v)
    for c in range(d):
        np.testing.assert_allclose(got[c], v[c], rtol=0, atol=2e-2 * vmax)      # bounded by the CG tolerance (rtol 1e-3)
    div = dom.centered_to_numpy(ops.divergence(dom, vbc, dv))
    rhs_scale = vmax * sum(2.0 / h for h in dx)
    assert np.abs(div).max() < 1e-2 * rhs_scale


def test_config_c1_smoke_plume_128_2d():
    """BASELINE configs[0] (examples/grids/Smoke_Plume at 128x128, closed box, CG 1e-3 warm start): 8 steps vs the oracle."""
    res = (128, 128)
    lower, upper = (0.0, 0.0), (100.0, 100.0)
    dx = (100.0 / 128, 100.0 / 128)
    vbc, sbc = O.uniform_bc(2, 0.0), O.uniform_bc(2, 'zg')
    inflow = O.sphere_soft_mask((50.0, 9.5), 5.0, lower, upper, res)
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    v = [np.zeros(s, np.float32) for s in O.staggered_shapes(res, vbc)]
    s = np.zeros(res, np.float32); p = np.zeros(res, np.float32)
    dv, ds, dp = dom.faces_from_numpy(v, vbc), dom.centered_from_numpy(s), dom.centered_from_numpy(p)
    dinflow = dom.centered_from_numpy(inflow)
    prm = ops.cg_params(vbc, rtol=1e-3, atol=1e-5)
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    for _ in range(8):
        ops.plume_step(dom, vbc, sbc, dv, ds, dp, dinflow, 0.5, 0.2, (0.0, 0.1), prm, mac_cormack=True)
        v, s, p, info = O.plume_step(v, s, p, 0.5, vbc, sbc, lower, upper, res, inflow, 0.2, (0.0, 0.1), rtol=1e-3, atol=1e-5,
                                     smoke_advection='mac_cormack', use_matrix_offset=False, matrix=A)
        assert ops.read_results(dom)['converged'][0] == 1 and info['converged']
    got_s = dom.centered_to_numpy(ds)
    np.testing.assert_allclose(got_s, s, rtol=0, atol=5e-4 * np.abs(s).max())
    got = dom.faces_to_numpy(dv, vbc)
    vmax = max(np.abs(c).max() for c in v)
    for c in range(2):
        np.testing.assert_allclose(got[c], v[c], rtol=0, atol=2e-2 * vmax)
    assert np.abs(s).max() > 0.5 and vmax > 1e-2


def test_config_c3_taylor_green_3d():
    """BASELINE configs[2] at 32^3: Taylor-Green vortex on [0, 2pi]^3, periodic, steps of semi_lagrangian -> make_incompressible;
    gates: divergence after projection, agreement with the oracle, kinetic energy does not grow."""
    n = 32
    res = (n, n, n)
    L = 2 * np.pi
    dx = (L / n,) * 3
    lower, upper = (0.0,) * 3, (L,) * 3
    vbc = O.uniform_bc(3, 'periodic')
    ax = np.arange(n, dtype=np.float64) * dx[0]
    cc = ax + 0.5 * dx[0]
    X, Y, Z = np.meshgrid(ax, cc, cc, indexing='ij')
    u = (np.sin(X) * np.cos(Y) * np.cos(Z)).astype(np.float32)              # x-faces: (face x, centre y, centre z)
    X, Y, Z = np.meshgrid(cc, ax, cc, indexing='ij')
    w = (-np.cos(X) * np.sin(Y) * np.cos(Z)).astype(np.float32)
    v = [u, w, np.zeros(res, np.float32)]
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    dv = dom.faces_from_numpy(v, vbc)
    dp = dom.alloc_centered()
    prm = ops.cg_params(vbc, rtol=1e-5, atol=1e-6)
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    dt = 0.5 * dx[0]
    energy = [sum(float(np.sum(c.astype(np.float64) ** 2)) for c in v)]
    p = np.zeros(res, np.float32)
    for _ in range(3):
        dv2 = ops.advect_staggered(dom, vbc, dv, vbc, dv, dt)
        dv, dp = ops.make_incompressible(dom, vbc, dv2, dp, prm)
        v = O.semi_lagrangian_staggered(v, vbc, v, vbc, res, lower, upper, dt)
        v, p, info = O.make_incompressible(v, vbc, res, dx, rtol=1e-5, atol=1e-6, x0=p, use_matrix_offset=False, matrix=A)
        got = dom.faces_to_numpy(dv, vbc)
        energy.append(sum(float(np.sum(c.astype(np.float64) ** 2)) for c in got))
    div = dom.centered_to_numpy(ops.divergence(dom, vbc, dv))
    assert np.abs(div).max() <= 5e-5 * 1.0 / dx[0]
    for c in range(3):
        np.testing.assert_allclose(got[c], v[c], rtol=0, atol=2e-4)
    assert all(b <= a * (1 + 1e-6) for a, b in zip(energy, energy[1:]))
    assert abs(energy[-1] / energy[0] - 1) < 0.05


@pytest.mark.parametrize('vname', ['zero', 'open', 'periodic', 'mixed', 'zero3', 'periodic3', 'wall_open3'])
@pytest.mark.parametrize('big', [False, True])
def test_make_incompressible_with_obstacle(vname, big):
    """SURVEY N4 (phi/physics/fluid.py:121-162 with obstacles): masked divergence, masked CG, masked gradient vs the oracle
    (whose masked matrix is pinned against the reference's traced matrix in tests/test_oracle_golden.py)."""
    vbc = ALL_V[vname]
    d = len(vbc)
    rng = np.random.default_rng(11)
    if big:
        res = (128, 20) if d == 2 else (128, 12, 8)
    else:
        res = (14, 11) if d == 2 else (10, 8, 7)
    dx = tuple(50.0 / r for r in res)
    acc = np.ones(res, np.float32)
    if d == 2:
        acc[res[0] // 3:res[0] // 2, 2:6] = 0
        acc[0:2, res[1] - 3:] = 0                        # an obstacle touching the domain boundary
    else:
        acc[res[0] // 3:res[0] // 2, 2:5, 1:4] = 0
    hard = O.hard_bcs_faces(acc, vbc)
    v = [c * np.float32(0.1) for c in rand_staggered(rng, res, vbc)]
    vmask = [h.copy() for h in hard]                     # any face factor works for the test; use the hard mask itself
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    dv = dom.faces_from_numpy(v, vbc)
    ops.mul_faces(dom, vbc, dv, dom.faces_from_numpy(vmask, vbc))
    dacc = dom.centered_from_numpy(acc)
    prm = ops.cg_params(vbc, rtol=1e-5, atol=1e-6)
    dv, dp = ops.make_incompressible(dom, vbc, dv, None, prm, accessible=dacc)
    launch = ops.last_launch_info()          # obstacles run on the TMA ring (mask staged as an extra haloed array), not the marching kernel
    assert launch['kernel'] == 3 and launch['masked'] == 1 and launch['generic'] == 1, launch
    info = ops.read_results(dom)
    assert info['converged'][0] == 1 and info['diverged'][0] == 0
    v_ref, p_ref, inf = O.make_incompressible_obstacles(v, vbc, res, dx, acc, vmask, rtol=1e-5, atol=1e-6)
    assert abs(int(info['iterations'][0]) - inf['iterations']) <= max(3, inf['iterations'] // 8), (info['iterations'], inf['iterations'])
    got = dom.faces_to_numpy(dv, vbc)
    for c in range(d):
        np.testing.assert_allclose(got[c], v_ref[c], rtol=0, atol=2e-4 * max(np.abs(v[c]).max(), 1e-3))
    p = dom.centered_to_numpy(dp)
    assert np.abs(p[acc == 0]).max() == 0.0                                   # pressure stays zero inside obstacles
    div = dom.centered_to_numpy(ops.divergence(dom, vbc, dv)) * acc
    vscale = max(np.abs(c).max() for c in v) * sum(2.0 / h for h in dx)
    assert np.abs(div).max() < 2e-4 * vscale


def test_config_c5_kolmogorov_batched_2d():
    """BASELINE configs[4] at 8 x 32^2: batched 2-D periodic Kolmogorov flow (forcing sin(4y) on the x component,
    examples/grids/Higher_order_Kolmogorov.ipynb:83-84, here with the order-2 operator-split step of SURVEY 8d):
    every batch entry is an independent system and must match its own un-batched oracle run."""
    n, batch = 32, 8
    res = (n, n)
    L = 2 * np.pi
    dx = (L / n, L / n)
    lower, upper = (0.0, 0.0), (L, L)
    vbc = O.uniform_bc(2, 'periodic')
    fbc = O.uniform_bc(2, 'periodic')
    yc = (np.arange(n) + 0.5) * dx[1]
    forcing = np.broadcast_to(np.sin(4 * yc)[None, :], res).astype(np.float32)
    v0 = [np.stack([(0.01 * np.random.default_rng(100 + b).standard_normal(res)).astype(np.float32) for b in range(batch)]) for _ in range(2)]
    dom = ops.Domain(res, dx, batch, vbc=vbc)
    dv = dom.faces_from_numpy(v0, vbc)
    dforce = dom.centered_from_numpy(forcing)
    dp = dom.alloc_centered()
    prm = ops.cg_params(vbc, rtol=1e-4, atol=1e-6)
    dt = 0.05
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    v = [[v0[0][b], v0[1][b]] for b in range(batch)]
    p = [np.zeros(res, np.float32) for _ in range(batch)]
    for _ in range(3):
        dv2 = ops.advect_staggered(dom, vbc, dv, vbc, dv, dt)
        ops.add_buoyancy(dom, vbc, fbc, dforce, (1.0, 0.0), dt, dv2)
        dv, dp = ops.make_incompressible(dom, vbc, dv2, dp, prm)
        assert ops.read_results(dom)['converged'].all()
        for b in range(batch):
            vb = O.semi_lagrangian_staggered(v[b], vbc, v[b], vbc, res, lower, upper, dt)
            faces = O.centered_to_faces(forcing * np.float32(1.0), fbc, vbc)
            vb = [vb[0] + faces[0] * np.float32(dt), vb[1]]
            vb, p[b], info = O.make_incompressible(vb, vbc, res, dx, rtol=1e-4, atol=1e-6, x0=p[b], use_matrix_offset=False, matrix=A)
            v[b] = vb
    got = dom.faces_to_numpy(dv, vbc, squeeze=False)
    for b in range(batch):
        for c in range(2):
            np.testing.assert_allclose(got[c][b], v[b][c], rtol=0, atol=5e-5)
    its = ops.read_results(dom)['iterations']
    assert its.min() >= 1 and len(set(its.tolist())) >= 1
