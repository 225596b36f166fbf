"""
The one-call step with obstacles on the host, over the oracle-backed engine of tests/oracle_plume_obstacles.py: the mirror's
`fluid.incompressible_step(..., obstacles=...)` against the sequenced mirror calls of Batched_Smoke / Fluid_Logo, the obstacle-mask
memo, union obstacles, and examples/fluid_logo.py.  The kernels are tests/test_gpu_plume_step_obstacles.py's business.
"""
import numpy as np
import pytest

from oracle import oracle_np as O
from oracle_plume_obstacles import ObstacleStepEngine
from test_cg_adaptive_masked_host import example


@pytest.fixture()
def F():
    import phiflow_b200.flow as flow
    saved = flow.ops, flow._DEVICE
    flow.ops = ObstacleStepEngine
    flow.set_device('cpu')
    flow._MASKS.clear()
    try:
        yield flow
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])
        flow._MASKS.clear()


def _state(F, rng, res, batch=1):
    dom = F.Box(x=100, y=80)
    v = F.StaggeredGrid([rng.standard_normal((batch,) + s).astype(np.float32) if batch > 1 else rng.standard_normal(s).astype(np.float32)
                         for s in O.staggered_shapes(res, O.uniform_bc(2, 0.0))], 0, dom, batch=batch, x=res[0], y=res[1])
    s = F.CenteredGrid(np.abs(rng.standard_normal(((batch,) if batch > 1 else ()) + res)).astype(np.float32), F.ZERO_GRADIENT, dom,
                       batch=batch, x=res[0], y=res[1])
    inflow = F.CenteredGrid(F.Box(x=(40, 60), y=(5, 12)), F.ZERO_GRADIENT, dom, batch=batch, x=res[0], y=res[1])
    return v, s, inflow


@pytest.mark.parametrize('method,advection', [('CG-adaptive', 'semi_lagrangian'), ('CG', 'mac_cormack')])
def test_step_equals_sequenced_mirror_calls(F, method, advection):
    """incompressible_step(v, s, p, dt, inflow, rate, buoyancy, Solve(...), obstacles=o) == the notebook cells advect -> + inflow ->
    resample(s * b, to=v) -> semi_lagrangian -> + buoyancy * dt -> make_incompressible(v, o, Solve(..., x0=p)), on a batch of 2, two
    steps (the second from the first one's pressure)."""
    rng = np.random.default_rng(3)
    res = (20, 16)
    v, s, inflow = _state(F, rng, res, batch=2)
    obstacle = F.union(F.Box(x=(30, 50), y=(40, 55)), F.Box(x=(50, 56), y=(40, 70)))
    rate, b, dt = 0.3, (0.0, 0.1), 1.0
    v1, s1, p1 = v, s, None
    v2, s2, p2 = v, s, None
    for _ in range(2):
        with F.SolveTape() as tape:
            v1, s1, p1 = F.fluid.incompressible_step(v1, s1, p1, dt, inflow=inflow, inflow_rate=rate, buoyancy=b,
                                                     solve=F.Solve(method, 1e-5, 1e-5), smoke_advection=advection, obstacles=obstacle)
        adv = F.advect.mac_cormack if advection == 'mac_cormack' else F.advect.semi_lagrangian
        s2 = adv(s2, v2, dt) + inflow * rate
        buoy = F.resample(s2 * b, to=v2)
        v2 = F.advect.semi_lagrangian(v2, v2, dt) + buoy * dt
        with F.SolveTape() as tape2:
            v2, p2 = F.fluid.make_incompressible(v2, obstacle, F.Solve(method, 1e-5, 1e-5, x0=p2))
        assert tape[0].iterations.tolist() == tape2[0].iterations.tolist() and tape[0].converged.all()
        np.testing.assert_array_equal(s1.numpy(), s2.numpy())
        np.testing.assert_array_equal(p1.numpy(), p2.numpy())
        for a, c in zip(v1.numpy(), v2.numpy()):
            np.testing.assert_array_equal(a, c)


def test_step_inputs_unmodified(F):
    rng = np.random.default_rng(4)
    v, s, inflow = _state(F, rng, (16, 12))
    before = [a.copy() for a in v.numpy()] + [s.numpy().copy()]
    F.fluid.incompressible_step(v, s, None, 1.0, inflow=inflow, inflow_rate=1.0, solve=F.Solve('CG-adaptive', 1e-5),
                                obstacles=F.Box(x=(30, 50), y=(40, 55)))
    for a, c in zip(before, [a for a in v.numpy()] + [s.numpy()]):
        np.testing.assert_array_equal(a, c)


def test_masks_are_rasterised_once(F, monkeypatch):
    """A step loop and make_incompressible with the same obstacle (an equal geometry object, not the same one) rasterise once, and the
    memoised masks are bit for bit those of _obstacle_masks; another geometry or grid rasterises again."""
    calls = []
    real = F._obstacle_masks
    monkeypatch.setattr(F, '_obstacle_masks', lambda vel, obs: calls.append(1) or real(vel, obs))
    rng = np.random.default_rng(5)
    v, s, inflow = _state(F, rng, (16, 12))
    p = None
    for _ in range(3):
        v, s, p = F.fluid.incompressible_step(v, s, p, 1.0, inflow=inflow, inflow_rate=1.0, solve=F.Solve('CG-adaptive', 1e-5),
                                              obstacles=F.Box(x=(30, 50), y=(40, 55)))
    F.fluid.make_incompressible(v, F.Box(x=(30, 50), y=(40, 55)), F.Solve(x0=p))
    assert len(calls) == 1
    acc, fac = F._obstacle_masks_cached(v, F.Box(x=(30, 50), y=(40, 55)))
    acc0, fac0 = real(v, F.Box(x=(30, 50), y=(40, 55)))
    assert len(calls) == 1
    assert np.array_equal(acc.numpy(), acc0.numpy()) and all(np.array_equal(a.numpy(), b.numpy()) for a, b in zip(fac, fac0))
    F._obstacle_masks_cached(v, F.Box(x=(30, 50), y=(40, 56)))
    w = F.StaggeredGrid(0, 0, F.Box(x=100, y=80), x=20, y=12)
    F._obstacle_masks_cached(w, F.Box(x=(30, 50), y=(40, 55)))
    assert len(calls) == 3


def test_union_obstacle_masks(F):
    """A union obstacle: accessible = outside every member; face factors = 1 - max of the members' fractions (the union's signed
    distance is the members' minimum, phi/geom/_geom_ops.py:100-102), which differs from the product of separate obstacles where
    the members touch."""
    a, b = F.Box(x=(20, 40), y=(20, 40)), F.Box(x=(40, 60), y=(20, 40))
    v = F.StaggeredGrid(0, 0, F.Box(x=100, y=80), x=25, y=20)
    acc_u, fac_u = F._obstacle_masks(v, F.union(a, b))
    acc_s, fac_s = F._obstacle_masks(v, (a, b))
    np.testing.assert_array_equal(acc_u.numpy(), acc_s.numpy())
    radius = np.float32(np.sqrt(sum((h * 0.5) ** 2 for h in v.dx)))
    for c in range(2):
        pts = v.face_points(c)
        frac = [np.clip(np.float32(1) - g.signed_distance(pts) / radius, 0, 1) for g in (a, b)]
        want = np.float32(1) - np.maximum(frac[0], frac[1])
        np.testing.assert_array_equal(v.dom.faces_to_numpy(fac_u, v.vspec)[c], want)
    assert any(not np.array_equal(x.numpy(), y.numpy()) for x, y in zip(fac_u, fac_s))


def test_fluid_logo_example(F):
    """examples/fluid_logo.py (Fluid_Logo.ipynb) for 3 steps at 32 x 32: every solve converges, smoke rises from the inflows and does not
    enter the logo."""
    smoke, v, p, its = example('fluid_logo').main(res=32, steps=3)
    assert len(its) == 3 and all(n > 0 for n in its)
    s = smoke.numpy()
    assert float(s.sum()) > 1.0 and np.isfinite(p.numpy()).all()
    geometry = F.union([F.Box(x=(15 + x * 7, 15 + (x + 1) * 7), y=(41, 83)) for x in range(1, 10, 2)])
    assert float(np.abs(s[geometry.lies_inside(smoke.points())]).max()) < 1e-6
