"""
CG-adaptive with obstacles on the host: the oracle's solver on the obstacle pressure operator against PhiML, and the mirror's policy
(`Solve()` / `Solve('CG-adaptive')` with obstacles run CG-adaptive, `Solve('CG')` plain CG), `geom.infinite_cylinder` and the
Wake_Flow example over the oracle-backed engine.  The kernel is tests/test_gpu_cg_adaptive_masked.py's business.
"""
import importlib.util
import os

import numpy as np
import pytest

from oracle import oracle_np as O
from oracle_masked import MaskedMethodEngine
import _phiml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, 'tests', 'golden', 'phiml_cg_adaptive_masked.npz'))


def spec_from_arr(a):
    return tuple(tuple('periodic' if np.isnan(s) else ('zg' if np.isinf(s) else float(s)) for s in ax) for ax in a)


@pytest.mark.parametrize('name', ['open', 'mixed', 'mixed3'])
@pytest.mark.parametrize('tag,rtol', [('r3', 1e-3), ('r5', 1e-5)])
def test_cg_adaptive_masked_matches_phiml_solve_linear(name, tag, rtol):
    """Solve('CG-adaptive') of PhiML 1.7.2 on the traced masked_laplace_obs vs oracle.cg_adaptive on masked_poisson_matrix_sparse:
    equal iteration counts, x within the tolerance of the fixture test without obstacles."""
    vbc, dx = spec_from_arr(GOLD[f'{name}/bc']), GOLD[f'{name}/dx']
    acc, rhs, x0 = GOLD[f'{name}/accessible'], GOLD[f'{name}/rhs'], GOLD[f'{name}/x0']
    A = O.masked_poisson_matrix_sparse(rhs.shape, dx, vbc, acc)
    info = O.cg_adaptive(A, rhs, x0, rtol, 1e-5, 1000, None)
    assert info['converged'] and not info['diverged']
    assert info['iterations'] == int(GOLD[f'{name}/{tag}/iterations'])
    x_ref = GOLD[f'{name}/{tag}/x']
    np.testing.assert_allclose(info['x'].reshape(rhs.shape), x_ref, rtol=0, atol=20 * rtol * np.abs(x_ref).max())


LIVE = [('open', (('zg', 'zg'), ('zg', 'zg')), (13, 9), (0.5, 1.25)),
        ('mixed', (('zg', 'zg'), (0.0, 'zg')), (16, 11), (1.0, 0.5)),
        ('mixed3', (('periodic', 'periodic'), (0.0, 'zg'), ('zg', 0.0)), (8, 6, 7), (0.5, 1.0, 2.0))]


@pytest.mark.parametrize('name,vbc,res,dx', LIVE, ids=[c[0] for c in LIVE])
def test_cg_adaptive_masked_live_phiml(name, vbc, res, dx):
    """The same against phiml.backend.NUMPY.linear_solve('CG-adaptive', ...) (_linalg.py:93-128, unmodified) run live on fresh masked
    systems: full solves, a warm start non-zero inside the obstacles and truncated runs.  Skipped without the reference's PhiML."""
    if not _phiml.ensure_phiml():
        pytest.skip("the reference's PhiML is not installed (oracle/_ref)")
    from phiml.backend import NUMPY
    rng = np.random.default_rng(31 + len(res))
    acc = np.ones(res, np.float32)
    acc[res[0] // 3:res[0] // 2 + 1, 2:4] = 0
    acc[0:2, -2:] = 0
    A = O.masked_poisson_matrix_sparse(res, dx, vbc, acc)
    y = (rng.standard_normal(res) * acc).astype(np.float32)
    warm = (0.1 * rng.standard_normal(res)).astype(np.float32)
    zero = np.zeros(res, np.float32)
    n = y.size
    for rtol, max_iter, x0 in [(1e-5, 1000, zero), (1e-3, 1000, warm), (1e-5, 1000, warm), (1e-5, 3, warm), (1e-5, 7, zero)]:
        ref = NUMPY.linear_solve('CG-adaptive', A, y.reshape(1, n), x0.reshape(1, n).copy(), np.array([rtol], np.float32),
                                 np.array([1e-5], np.float32), np.array([[max_iter]]), None, None)
        mine = O.cg_adaptive(A, y, x0, rtol, 1e-5, max_iter, None)
        ref_x = np.asarray(ref.x)[0]
        assert abs(int(np.asarray(ref.iterations)[0]) - mine['iterations']) <= 1, (rtol, max_iter)
        scale = max(float(np.abs(ref_x).max()), 1e-3)
        np.testing.assert_allclose(mine['x'], ref_x, rtol=0, atol=2e-5 * scale + (0 if max_iter < 1000 else 20 * rtol * scale))


@pytest.fixture(scope='module')
def F():
    import phiflow_b200.flow as flow
    saved = flow.ops, flow._DEVICE
    flow.ops = MaskedMethodEngine
    flow.set_device('cpu')
    try:
        yield flow
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])


def test_cg_params_with_obstacles(F):
    """'auto' and 'CG-adaptive' run CG-adaptive (method 1) with or without obstacles; 'CG' runs plain CG (method 0)."""
    v = F.StaggeredGrid(0, 0, F.Box(x=10, y=10), x=8, y=8)
    assert F._cg_params(v, F.Solve()).method == 1
    assert F._cg_params(v, F.Solve('auto')).method == 1
    assert F._cg_params(v, F.Solve('CG-adaptive', 1e-5)).method == 1
    assert F._cg_params(v, F.Solve('CG', 1e-5)).method == 0


def test_make_incompressible_obstacle_solvers(F):
    """make_incompressible(v, obstacle, Solve(...)) hands the solver to the engine: Solve() follows the CG-adaptive oracle, Solve('CG')
    the plain one, and the two stopping rules give different iteration counts from a warm start."""
    rng = np.random.default_rng(5)
    vbc = O.uniform_bc(2, 0.0)
    res = (24, 20)
    v = F.StaggeredGrid([rng.standard_normal(s).astype(np.float32) for s in O.staggered_shapes(res, vbc)], 0, F.Box(x=24, y=20), x=24, y=20)
    obstacle = F.Box(x=(8, 14), y=(5, 9))
    _, p = F.fluid.make_incompressible(v, obstacle, F.Solve('CG-adaptive', 1e-5, 1e-5))
    counts = {}
    w = v * 1.01
    for name, solve in [('auto', F.Solve(x0=p)), ('CG', F.Solve('CG', 1e-5, 1e-5, x0=p))]:
        with F.SolveTape() as tape:
            F.fluid.make_incompressible(w, obstacle, solve)
        assert tape[0].converged.all()
        counts[name] = int(tape[0].iterations[0])
    # plain CG stops relative to the warm start's small residual, CG-adaptive relative to |y'|: fewer iterations
    assert counts['auto'] < counts['CG'], counts


def example(name):
    spec = importlib.util.spec_from_file_location(f'example_{name}', os.path.join(ROOT, 'examples', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_wake_flow_example(F):
    """examples/wake_flow.py (Wake_Flow.ipynb) runs 3 steps at 32 x 16 x 4: no flow into the cylinder, periodic y and z kept."""
    v, p = example('wake_flow').main(res=32, nz=4, steps=3)
    vx = v.numpy()[0]
    inside = F.geom.infinite_cylinder(x=20, y=50, radius=10, inf_dim='z').lies_inside(v.face_points(0))
    assert inside.any() and float(np.abs(vx[inside]).max()) < 1e-5
    assert float(np.abs(vx).max()) > 1.0 and np.isfinite(p.numpy()).all()


def test_infinite_cylinder_masks(F):
    """geom.infinite_cylinder(x, y, radius, inf_dim='z') = a Sphere over (x, y) in every z plane, for lies_inside and signed_distance
    (the accessible mask and the face factors of _obstacle_masks)."""
    cyl = F.geom.infinite_cylinder(x=20, y=50, radius=10, inf_dim='z')
    sph = F.Sphere(x=20, y=50, radius=10)
    grid = F.CenteredGrid(0, 0, F.Box(x=200, y=100, z=5), x=32, y=16, z=4)
    pts = grid.points()
    inside = cyl.lies_inside(pts)
    assert inside.any() and not inside.all()
    for k in range(pts.shape[2]):
        np.testing.assert_array_equal(inside[:, :, k], sph.lies_inside(pts[:, :, k, :2]))
        np.testing.assert_array_equal(cyl.signed_distance(pts[:, :, k]), sph.signed_distance(pts[:, :, k, :2]))
    v = F.StaggeredGrid((8., 0, 0), {'x-': F.vec(x=2, y=0, z=0), 'x+': F.ZERO_GRADIENT, 'y': F.PERIODIC, 'z': F.PERIODIC},
                        x=32, y=16, z=4, bounds=F.Box(x=200, y=100, z=5))
    acc, _ = F._obstacle_masks(v, cyl)
    want = (~np.repeat(sph.lies_inside(pts[:, :, :1, :2]), 4, axis=2)).astype(np.float32)
    np.testing.assert_array_equal(v.dom.centered_to_numpy(acc), want)
    with pytest.raises(NotImplementedError):
        F.geom.infinite_cylinder(x=20, y=50, z=1, radius=10, inf_dim='z')
