"""
The facade `phiflow_b200/phi_cuda/flow.py` (the `phi.cuda.flow` a notebook would import), EXECUTED - against a test double of `phi`
(tests/stubs/phi: Fields holding real phiml Tensors / Extrapolations under phi 3.4's attribute names, stock functions that only record
calls), because PhiFlow 3.4 itself cannot be imported with the PhiML 1.7.2 this image has.  What is real here: phiml (Tensors, Solve,
SolveTape, NotConverged, the default-backend machinery), the facade, the adapter; the engine is the oracle-backed stand-in of
tests/test_phi_cuda_adapter.py (no GPU in this container).  What it proves: the wrappers run, route eligible calls to the engine and
everything else to the stock function with a recorded reason, and speak phiml's solve protocol (SolveTape records, NotConverged,
`suppress`).  It does not prove compatibility with phi 3.4 beyond the attribute names cited in the double.
"""
import os
import sys

import numpy as np
import pytest

from _phiml import ensure_phiml

if not ensure_phiml():
    pytest.skip('PhiML not available (neither installed nor in oracle/_ref)', allow_module_level=True)

from phiml import math  # noqa: E402
from phiml import backend as phiml_backend  # noqa: E402
from phiml.math import extrapolation as E, spatial, batch, dual, channel  # noqa: E402

from oracle import oracle_np as O  # noqa: E402
from phiflow_b200.phi_cuda import _adapter as A  # noqa: E402
from test_phi_cuda_adapter import FakeOps  # noqa: E402

STUBS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'stubs')


def make_flow_fixture(real_engine: bool):
    """Module-scoped fixture that imports the facade over the test double - with the oracle-backed stand-in engine here, with the
    real CUDA engine in tests/test_gpu_phi_cuda_facade.py - and undoes every global side effect afterwards."""
    @pytest.fixture(scope='module')
    def flow():
        try:
            import phi  # noqa: F401
            if 'test-double' not in getattr(phi, '__version__', ''):
                pytest.skip('a real PhiFlow is importable here; this file is for images where it is not')
        except ImportError:
            pass
        previous_default = phiml_backend.default_backend()
        engine, device = A.ENGINE, A.DEVICE
        if not real_engine:
            A.ENGINE, A.DEVICE = FakeOps, 'cpu'
        sys.path.insert(0, STUBS)
        try:
            import importlib
            yield importlib.import_module('phiflow_b200.phi_cuda.flow')
        finally:
            phiml_backend.set_global_default_backend(previous_default)
            A.ENGINE, A.DEVICE = engine, device
            sys.path.remove(STUBS)
            for name in [m for m in sys.modules if m == 'phi' or m.startswith('phi.') or m == 'phiflow_b200.phi_cuda.flow']:
                del sys.modules[name]
    return flow


flow = make_flow_fixture(real_engine=False)


def _velocity(flow, rng, ext, res=(16, 20), nb=2):
    dims = ('x', 'y')
    vspec = A.to_vspec(ext, dims)
    comps, arrays = [], []
    for s in O.staggered_shapes(res, vspec):
        a = rng.standard_normal((nb,) + s).astype(np.float32)
        arrays.append(a)
        comps.append(math.tensor(a, batch(b=nb) & spatial(**dict(zip(dims, s)))))
    values = math.stack(comps, dual(vector=dims))
    return flow.StaggeredGrid(values, ext, flow.Box(x=100, y=100), x=res[0], y=res[1]), arrays, vspec


def _divergence_by_phiml(v, ext, dims=('x', 'y')):
    dx = v.dx
    div = 0
    for d in dims:
        comp = v.values[{'~vector': d}]
        lo, hi = ext.valid_outer_faces(d)
        baked = math.pad(comp, {d: (0 if lo else 1, 0 if hi else 1)}, ext)
        div = div + (baked[{d: slice(1, None)}] - baked[{d: slice(None, -1)}]) / float(dx.vector[d])
    return div


def test_import_exports_and_default_backend(flow):
    assert phiml_backend.default_backend().name == 'phicuda'            # as phi/torch/flow.py:27-35 does for torch
    assert flow.fluid.make_incompressible is flow.make_incompressible
    assert flow.advect.semi_lagrangian is flow.semi_lagrangian and flow.advect.mac_cormack is flow.mac_cormack
    assert flow.field.laplace is flow.laplace and flow.field.divergence is flow.divergence
    import phi.physics.fluid as stock_fluid
    assert stock_fluid.make_incompressible is not flow.make_incompressible      # the stock module is not modified
    assert flow.fluid._pressure_extrapolation is stock_fluid._pressure_extrapolation   # everything else is the stock module's


@pytest.mark.parametrize('name', ['zero', 'periodic', 'mixed'])
def test_make_incompressible_fields_in_fields_out(flow, name):
    ext = {'zero': E.ZERO, 'periodic': E.PERIODIC, 'mixed': E.combine_sides(x=E.BOUNDARY, y=(E.ZERO, E.BOUNDARY))}[name]
    v, arrays, _ = _velocity(flow, np.random.default_rng(1), ext)
    del flow.FALLTHROUGH_LOG[:]
    with math.SolveTape() as tape:
        v2, p = flow.fluid.make_incompressible(v, (), flow.Solve('CG', 1e-5, 1e-5))
    assert not flow.FALLTHROUGH_LOG
    assert v2.is_staggered and v2.extrapolation is v.extrapolation and v2.bounds == v.bounds and v2.resolution == v.resolution
    assert not p.is_staggered and set(p.values.shape.names) == {'b', 'x', 'y'}
    assert p.extrapolation == flow.fluid._pressure_extrapolation(ext)
    div = _divergence_by_phiml(v2, ext)
    assert float(np.abs(div.numpy(div.shape.names)).max()) < 5e-5 * float(max(np.abs(a).max() for a in arrays))
    # the solve is visible to SolveTapes like a math.solve_linear call (PhiML/phiml/math/_optimize.py:735-743)
    info = tape[0]
    assert info.method == 'phicuda' and info.iterations.shape.names == ('b',) and (info.iterations.numpy('b') > 0).all()
    assert bool(info.converged.all) and not bool(info.diverged.any)
    assert info.x is p


def test_not_converged_is_raised_and_can_be_suppressed(flow):
    v, _, _ = _velocity(flow, np.random.default_rng(2), E.ZERO)
    with pytest.raises(math.NotConverged) as err:
        flow.fluid.make_incompressible(v, (), flow.Solve('CG', 1e-6, 1e-6, max_iterations=3))
    assert err.value.result.method == 'phicuda' and (err.value.result.iterations.numpy('b') == 3).all()
    assert 'did not converge' in str(err.value.result.msg)
    v2, p = flow.fluid.make_incompressible(v, (), flow.Solve('CG', 1e-6, 1e-6, max_iterations=3, suppress=[math.NotConverged]))
    assert v2.is_staggered and np.isfinite(p.values.numpy(p.values.shape.names)).all()


def test_ineligible_calls_fall_through_with_a_reason(flow):
    import phi
    v, _, _ = _velocity(flow, np.random.default_rng(3), E.ZERO)
    cases = [
        (dict(solve=flow.Solve('biCG-stab(2)', 1e-5, 1e-5)), 'solver'),
        (dict(solve=flow.Solve('CG', 1e-5, 1e-5), obstacles=[object()]), 'obstacles'),
        (dict(solve=flow.Solve('CG', 1e-5, 1e-5), order=4), 'order'),
        (dict(solve=flow.Solve('CG', 1e-5, 1e-5), active=object()), 'active'),
        (dict(solve=flow.Solve('CG', 1e-5, 1e-5, preconditioner='ilu')), 'preconditioned'),
    ]
    for kwargs, word in cases:
        del flow.FALLTHROUGH_LOG[:], phi.STOCK_CALLS[:]
        out = flow.fluid.make_incompressible(v, **kwargs)
        assert out == 'stock make_incompressible' and phi.STOCK_CALLS[0][0] == 'fluid.make_incompressible'
        assert flow.FALLTHROUGH_LOG[0][0] == 'make_incompressible' and word in flow.FALLTHROUGH_LOG[0][1], flow.FALLTHROUGH_LOG
    # SYMMETRIC walls: valid PhiFlow, outside the fast path
    del flow.FALLTHROUGH_LOG[:]
    vs = flow.StaggeredGrid(v.values, E.SYMMETRIC, v.bounds, x=16, y=20)
    assert flow.fluid.make_incompressible(vs, (), flow.Solve('CG', 1e-5, 1e-5)) == 'stock make_incompressible'
    with math.precision(64):
        assert flow.fluid.make_incompressible(v, (), flow.Solve('CG', 1e-5, 1e-5)) == 'stock make_incompressible'
        assert 'precision 64' in flow.FALLTHROUGH_LOG[-1][1]
    assert flow.fluid.make_incompressible('not a field', (), flow.Solve('CG', 1e-5, 1e-5)) == 'stock make_incompressible'


def test_centered_velocity_runs_the_wide_stencil_path(flow):
    """tests/commit/physics/test_fluid.py:34-36 on Fields: CenteredGrid velocity, default Solve() = 'auto' = CG-adaptive."""
    res = (16, 20)
    pts = O.points_of((0.0, 0.0), (100.0, 100.0), res)
    a = np.zeros((16, 20, 2), np.float32)
    a[:, :, 1] = 0.1 * (np.sum((pts - np.array((40.0, 10.0), np.float32)) ** 2, -1) <= 25.0)
    v = flow.CenteredGrid(math.tensor(a, spatial(x=16, y=20) & channel(vector='x,y')), E.ZERO, flow.Box(x=100, y=100), x=16, y=20)
    del flow.FALLTHROUGH_LOG[:]
    v2, p = flow.fluid.make_incompressible(v, (), flow.Solve())
    assert not flow.FALLTHROUGH_LOG and not v2.is_staggered and v2.values.shape.get_item_names('vector') == ('x', 'y')
    div = 0
    for d in ('x', 'y'):
        padded = math.pad(v2.values.vector[d], {d: (1, 1)}, E.ZERO)
        div = div + (padded[{d: slice(2, None)}] - padded[{d: slice(None, -2)}]) / (2 * float(v.dx.vector[d]))
    assert float(np.abs(div.numpy('x,y')).max()) < 5e-5
    # plain CG is not run on this operator: stock
    assert flow.fluid.make_incompressible(v, (), flow.Solve('CG', 1e-5, 1e-5)) == 'stock make_incompressible'


def test_advection_wrappers(flow):
    import phi
    v, arrays, vspec = _velocity(flow, np.random.default_rng(4), E.ZERO, res=(12, 10), nb=1)
    lower, upper = (0.0, 0.0), (100.0, 100.0)
    del flow.FALLTHROUGH_LOG[:]
    out = flow.advect.semi_lagrangian(v, v, 0.3)
    ref = O.semi_lagrangian_staggered([a[0] for a in arrays], vspec, [a[0] for a in arrays], vspec, (12, 10), lower, upper, 0.3)
    for c, d in enumerate('xy'):
        np.testing.assert_allclose(out.values[{'~vector': d, 'b': 0}].numpy('x,y'), ref[c], atol=2e-5)
    s = np.random.default_rng(5).standard_normal((12, 10)).astype(np.float32)
    smoke = flow.CenteredGrid(math.tensor(s, spatial(x=12, y=10)), E.ZERO_GRADIENT, v.bounds, x=12, y=10)
    adv = flow.advect.mac_cormack(smoke, v, 0.3)
    ref_mc = O.mac_cormack_centered(s, O.uniform_bc(2, 'zg'), [a[0] for a in arrays], vspec, lower, upper, 0.3)
    np.testing.assert_allclose(adv.values.b[0].numpy('x,y'), ref_mc, atol=5e-5)
    adv2 = flow.advect.advect(smoke, v, 0.3)                           # advect() of a grid = semi_lagrangian (phi/physics/advect.py:27-44)
    np.testing.assert_allclose(adv2.values.b[0].numpy('x,y'),
                               O.semi_lagrangian_centered(s, O.uniform_bc(2, 'zg'), [a[0] for a in arrays], vspec, lower, upper, 0.3), atol=2e-5)
    assert not flow.FALLTHROUGH_LOG and adv.extrapolation is smoke.extrapolation
    # another integrator, another grid -> stock
    assert flow.advect.semi_lagrangian(smoke, v, 0.3, integrator=phi.physics.advect.rk4) == 'stock semi_lagrangian'
    other = flow.CenteredGrid(math.tensor(s[:10], spatial(x=10, y=10)), E.ZERO_GRADIENT, v.bounds, x=10, y=10)
    assert flow.advect.semi_lagrangian(other, v, 0.3) == 'stock semi_lagrangian'
    assert flow.advect.mac_cormack(v, v, 0.3) == 'stock mac_cormack'
    assert [r[0] for r in flow.FALLTHROUGH_LOG] == ['semi_lagrangian', 'semi_lagrangian', 'mac_cormack']


def test_stencil_wrappers(flow):
    s = np.random.default_rng(6).standard_normal((12, 10)).astype(np.float32)
    box = flow.Box(x=12, y=5)
    u = flow.CenteredGrid(math.tensor(s, spatial(x=12, y=10)), E.ZERO_GRADIENT, box, x=12, y=10)
    lap = flow.field.laplace(u)
    np.testing.assert_allclose(lap.values.numpy('x,y'), math.laplace(u.values, dx=u.dx, padding=E.ZERO_GRADIENT).numpy('x,y'), atol=4e-5)
    assert lap.extrapolation == E.ZERO_GRADIENT.spatial_gradient().spatial_gradient()
    assert flow.field.laplace(u, order=4) == 'stock laplace'
    v, arrays, vspec = _velocity(flow, np.random.default_rng(7), E.ZERO, res=(12, 10), nb=1)
    div = flow.field.divergence(v)
    assert not div.is_staggered and div.extrapolation == E.ZERO.spatial_gradient()
    np.testing.assert_allclose(div.values.numpy('b,x,y'), _divergence_by_phiml(v, E.ZERO).numpy('b,x,y'), atol=2e-5)
    assert flow.field.divergence(u) == 'stock divergence'
