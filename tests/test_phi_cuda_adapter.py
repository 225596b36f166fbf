"""
Reference-side adapter (phiflow_b200/phi_cuda, row B1) against REAL phiml objects from the vendored PhiML 1.7.2
(an installed phiml, or oracle/_ref as installed by __graft_entry__.build()): boundary translation, named-dim layouts incl. the
non-uniform staggered TensorStack, the eligibility matrix of SURVEY.md section 3.4, and the hot-path functions with phiml Tensors
in and out.  There is no GPU here, so the compute engine is replaced by an oracle-backed stand-in with the SAME interface as
phiflow_b200._ops (device arrays in, device arrays updated in place) - this file tests the plumbing around the C ABI, the
kernels themselves are tested against the oracle in the -m gpu tests, and tests/test_gpu_phi_cuda.py repeats this file's cases
with the real engine against the reference library run live.
"""
import os
import sys

import numpy as np
import pytest
import torch

from _phiml import ensure_phiml  # noqa: E402

if not ensure_phiml():
    pytest.skip('PhiML not available (neither installed nor in oracle/_ref)', allow_module_level=True)

from phiml import math  # noqa: E402
from phiml.math import extrapolation as E, spatial, batch, dual, channel  # noqa: E402

from oracle import oracle_np as O  # noqa: E402
from phiflow_b200 import _ops  # noqa: E402
from phiflow_b200.phi_cuda import _adapter as A  # noqa: E402


from oracle_engine import OracleEngine as FakeOps  # noqa: E402  (oracle-backed stand-in for phiflow_b200._ops, CPU tensors in the device layout)


@pytest.fixture()
def fake_engine(monkeypatch):
    monkeypatch.setattr(A, 'ENGINE', FakeOps)
    monkeypatch.setattr(A, 'DEVICE', 'cpu')
    return FakeOps


# ---- (i) boundary translation ---------------------------------------------------------------------------------------------------
def test_extrapolation_translation_table():
    dims = ('x', 'y')
    assert A.to_spec(E.ZERO, dims) == ((0.0, 0.0), (0.0, 0.0))
    assert A.to_spec(E.ONE, dims) == ((1.0, 1.0), (1.0, 1.0))
    assert A.to_spec(E.PERIODIC, dims) == (('periodic', 'periodic'),) * 2
    assert A.to_spec(E.ZERO_GRADIENT, dims) == (('zg', 'zg'),) * 2
    assert E.BOUNDARY is E.ZERO_GRADIENT
    assert A.to_spec(E.ConstantExtrapolation(2.5), ('x', 'y', 'z')) == ((2.5, 2.5),) * 3
    # combine_sides (tests/commit/physics/test_fluid.py:50-53)
    mixed = E.combine_sides(x=E.BOUNDARY, y=(E.ZERO, E.BOUNDARY))
    assert A.to_spec(mixed, dims) == (('zg', 'zg'), (0.0, 'zg'))
    assert A.to_vspec(mixed, dims) == (('zg', 'zg'), (0.0, 'zg'))
    per_wall = E.combine_sides(x=E.PERIODIC, y=E.ZERO)
    assert A.to_spec(per_wall, dims) == (('periodic', 'periodic'), (0.0, 0.0))
    # vector constants: one spec per component (inflow boundary: different constants, same kinds)
    inflow = E.ConstantExtrapolation(math.tensor([1.0, 0.0], channel(vector='x,y')))
    assert A.to_vspec(inflow, dims) == [((1.0, 1.0), (1.0, 1.0)), ((0.0, 0.0), (0.0, 0.0))]
    both = E.combine_sides(x=(inflow, E.BOUNDARY), y=E.ZERO)
    assert A.to_vspec(both, dims) == [((1.0, 'zg'), (0.0, 0.0)), ((0.0, 'zg'), (0.0, 0.0))]
    # faces stored per side follow valid_outer_faces (extrapolation.py:57-62, tests/commit/field/test__grid.py:25-37)
    assert A.stored_face_counts(A.to_vspec(mixed, dims), (16, 20)) == [(17, 20), (16, 20)]
    for d, ext in (('x', E.ZERO), ('x', E.PERIODIC), ('x', E.BOUNDARY)):
        lo, hi = ext.valid_outer_faces(d)
        spec = A.to_vspec(ext, dims)
        assert _ops.stored_faces(spec, 0) == (lo, hi)


@pytest.mark.parametrize('ext', [E.SYMMETRIC, E.REFLECT, E.NONE, E.ANTISYMMETRIC if hasattr(E, 'ANTISYMMETRIC') else E.SYMMETRIC])
def test_unsupported_boundaries_are_not_eligible(ext):
    with pytest.raises(A.NotEligible):
        A.to_spec(ext, ('x', 'y'))
    assert A.eligible(('x', 'y'), ext) is not None


def test_periodic_on_one_side_only_is_rejected():
    with pytest.raises(A.NotEligible):
        A.to_spec(E.combine_sides(x=(E.PERIODIC, E.ZERO), y=E.ZERO), ('x', 'y'))


# ---- (iii) eligibility matrix (SURVEY.md section 3.4) ------------------------------------------------------------------------------
def test_eligibility_matrix():
    dims = ('x', 'y', 'z')
    assert A.eligible(dims, E.ZERO, solve_method='CG') is None
    assert A.eligible(dims, E.PERIODIC, solve_method='auto') is None
    assert A.eligible(dims, E.combine_sides(x=E.PERIODIC, y=E.ZERO, z=(E.ZERO, E.BOUNDARY)), solve_method='CG-adaptive') is None
    assert 'order' in A.eligible(dims, E.ZERO, order=4)
    assert 'solver' in A.eligible(dims, E.ZERO, solve_method='biCG-stab(2)')
    assert 'solver' in A.eligible(dims, E.ZERO, solve_method='scipy-direct')
    assert 'obstacles' in A.eligible(dims, E.ZERO, obstacles=[object()])
    assert 'active' in A.eligible(dims, E.ZERO, active=object())
    assert 'CenteredGrid' in A.eligible(dims, E.ZERO, staggered=False)
    assert 'preconditioned' in A.eligible(dims, E.ZERO, preconditioner='ilu')
    assert '1-D' in A.eligible(('x',), E.ZERO)
    assert 'non-uniform' in A.eligible(dims, E.ZERO, uniform=False)
    with math.precision(64):                      # Taylor_Green / Kolmogorov notebooks: never silently downcast
        assert 'precision 64' in A.eligible(dims, E.ZERO)
    assert A.eligible(dims, E.ZERO) is None


# ---- (ii) layouts -------------------------------------------------------------------------------------------------------------------
def _staggered_values(rng, res, vspec, dims, batch_shape=None):
    shapes = O.staggered_shapes(res, vspec)
    comps, arrays = [], []
    for c, s in enumerate(shapes):
        pre = () if batch_shape is None else batch_shape.sizes
        a = rng.standard_normal(pre + s).astype(np.float32)
        arrays.append(a)
        shape = spatial(**dict(zip(dims, s)))
        comps.append(math.tensor(a, (batch_shape & shape) if batch_shape is not None else shape))
    return math.stack(comps, dual(vector=dims)), arrays


def test_nonuniform_staggered_stack_roundtrip(fake_engine):
    """combine_sides(x=BOUNDARY, y=(ZERO, BOUNDARY)): components of 17x20 and 16x20 faces form a non-uniform TensorStack that
    has no single native array (SURVEY.md section 8b) - it is exported per component and rebuilt with math.stack(..., dual(vector))."""
    dims, res = ('x', 'y'), (16, 20)
    ext = E.combine_sides(x=E.BOUNDARY, y=(E.ZERO, E.BOUNDARY))
    vspec = A.to_vspec(ext, dims)
    bshape = batch(b=3)
    values, arrays = _staggered_values(np.random.default_rng(0), res, vspec, dims, bshape)
    assert not values.shape.is_uniform
    comps = A.split_components(values, dims)
    assert [tuple(c.shape.get_size(d) for d in dims) for c in comps] == [(17, 20), (16, 20)]
    dom = _ops.Domain(res, (1.0, 1.0), 3, vbc=vspec, device='cpu')
    dev = A.pull_staggered(dom, comps, vspec, bshape, dims)
    # device layout: (batch, y, x), x contiguous; y component starts at face 1 along y (the wall face 0 is not stored)
    assert dev[0].shape == (3, dom.fext[1], dom.fext[0])
    np.testing.assert_array_equal(dev[0][1, :20, :17].numpy(), arrays[0][1].T)
    np.testing.assert_array_equal(dev[1][2, 1:21, :16].numpy(), arrays[1][2].T)
    assert float(dev[1][:, 0].abs().max()) == 0.0
    back = A.push_staggered(dom, dev, vspec, bshape, dims)
    assert back.shape.names == values.shape.names or set(back.shape.names) == set(values.shape.names)
    for d, a in zip(dims, arrays):
        np.testing.assert_array_equal(back[{'~vector': d}].numpy(('b',) + dims), a)
    # wrong face counts are refused (e.g. values built for another boundary)
    with pytest.raises(A.NotEligible):
        A.pull_staggered(dom, comps, A.to_vspec(E.ZERO, dims), bshape, dims)


def test_centered_roundtrip_keeps_dim_names_and_order(fake_engine):
    dims, res = ('x', 'y', 'z'), (5, 4, 3)
    a = np.arange(2 * 5 * 4 * 3, dtype=np.float32).reshape(2, 5, 4, 3)
    t = math.tensor(a, batch(batch=2) & spatial(x=5, y=4, z=3))
    dom = _ops.Domain(res, (1.0,) * 3, 2, device='cpu')
    dev = A.pull_centered(dom, t, t.shape.batch, dims)
    assert dev.shape == (2, 3, 4, 8)                         # z, y, x with x padded to a multiple of 4
    assert float(dev[1, 2, 3, 4]) == a[1, 4, 3, 2]           # reference order is x outermost, z contiguous (SURVEY A13)
    back = A.push_centered(dom, dev, t.shape.batch, dims)
    np.testing.assert_array_equal(back.numpy('batch,x,y,z'), a)
    # a tensor stored in another dim order gives the same device array
    t2 = math.tensor(np.transpose(a, (0, 3, 1, 2)), batch(batch=2) & spatial(z=3, x=5, y=4))
    assert torch.equal(A.pull_centered(dom, t2, t2.shape.batch, dims), dev)


# ---- (iv) hot-path functions: phiml Tensors in, phiml Tensors out ----------------------------------------------------------------------
@pytest.mark.parametrize('name', ['zero', 'boundary', 'periodic', 'mixed'])
def test_make_incompressible_with_phiml_tensors(fake_engine, name):
    """The cases of tests/commit/physics/test_fluid.py:38-53 (16x20 StaggeredGrid) on values / extrapolation / dx as a Field holds
    them.  Checks: named dims and face counts of the result, pressure on the cell grid, divergence-free by the REFERENCE's own
    arithmetic (phiml pad + forward differences, phi/field/_field_math.py:617-626)."""
    dims, res = ('x', 'y'), (16, 20)
    ext = {'zero': E.ZERO, 'boundary': E.BOUNDARY, 'periodic': E.PERIODIC, 'mixed': E.combine_sides(x=E.BOUNDARY, y=(E.ZERO, E.BOUNDARY))}[name]
    dx = {'x': 100.0 / 16, 'y': 100.0 / 20}
    vspec = A.to_vspec(ext, dims)
    values, arrays = _staggered_values(np.random.default_rng(3), res, vspec, dims, batch(b=2))
    new_values, pressure, info = A.make_incompressible(values, ext, dx, dims, res, method='CG', rel_tol=1e-5, abs_tol=1e-5)
    assert set(pressure.shape.names) == {'b', 'x', 'y'} and pressure.shape.get_size('x') == 16 and pressure.shape.get_size('y') == 20
    assert info['converged'].all() and not info['diverged'].any() and (info['iterations'] > 0).all()
    for c, d in enumerate(dims):
        comp = new_values[{'~vector': d}]
        assert tuple(comp.shape.get_size(k) for k in dims) == arrays[c].shape[1:]
    # divergence with the reference's arithmetic: bake the boundary faces with math.pad, forward differences
    div = 0
    for c, d in enumerate(dims):
        comp = new_values[{'~vector': d}]
        lo, hi = ext.valid_outer_faces(d)
        baked = math.pad(comp, {d: (0 if lo else 1, 0 if hi else 1)}, ext[{'vector': d}] if name != 'mixed' else ext)
        div = div + (baked[{d: slice(1, None)}] - baked[{d: slice(None, -1)}]) / dx[d]
    assert float(np.abs(div.numpy(div.shape.names)).max()) < 5e-5 * max(1.0, float(max(np.abs(a).max() for a in arrays)))
    # and the fall-through contract: ineligible requests raise NotEligible, nothing is computed
    with pytest.raises(A.NotEligible):
        A.make_incompressible(values, ext, dx, dims, res, method='biCG-stab(2)')
    with math.precision(64):
        with pytest.raises(A.NotEligible):
            A.make_incompressible(values, ext, dx, dims, res, method='CG')


@pytest.mark.parametrize('name', ['zero', 'boundary'])
def test_make_incompressible_centered_velocity_with_phiml_tensors(fake_engine, name):
    """tests/commit/physics/test_fluid.py:34-36: CenteredGrid velocity (channel dim `vector`), ZERO and BOUNDARY; result checked with
    the reference's own centred divergence (math.spatial_gradient 'central' + padding by the velocity boundary, _field_math.py:627-632)."""
    dims, res = ('x', 'y'), (16, 20)
    ext = {'zero': E.ZERO, 'boundary': E.BOUNDARY}[name]
    dx = {'x': 100.0 / 16, 'y': 100.0 / 20}
    # the reference test's input: buoyancy of a sphere of smoke (smooth; white noise has components outside the range of the
    # singular wide-stencil operator and cannot be projected to 5e-5)
    pts = O.points_of((0.0, 0.0), (100.0, 100.0), res)
    a = np.zeros((2, 16, 20, 2), np.float32)
    for b, centre in enumerate(((40.0, 10.0), (55.0, 30.0))):
        a[b, :, :, 1] = 0.1 * (np.sum((pts - np.array(centre, np.float32)) ** 2, -1) <= 25.0)
    values = math.tensor(a, batch(b=2) & spatial(x=16, y=20) & channel(vector='x,y'))
    new_values, pressure, info = A.make_incompressible_centered(values, ext, dx, dims, res, method='auto')
    assert set(new_values.shape.names) == {'b', 'x', 'y', 'vector'} and new_values.shape.get_item_names('vector') == ('x', 'y')
    assert set(pressure.shape.names) == {'b', 'x', 'y'} and not info['diverged'].any()
    div = 0
    for d in dims:
        comp = new_values.vector[d]
        padded = math.pad(comp, {d: (1, 1)}, ext)
        div = div + (padded[{d: slice(2, None)}] - padded[{d: slice(None, -2)}]) / (2 * dx[d])
    assert float(np.abs(div.numpy(div.shape.names)).max()) < 5e-5
    with pytest.raises(A.NotEligible):
        A.make_incompressible_centered(values, ext, dx, dims, res, method='CG')       # plain CG: not on this operator


def test_semi_lagrangian_and_stencils_with_phiml_tensors(fake_engine):
    dims, res = ('x', 'y'), (12, 10)
    ext = E.ZERO
    dx = {'x': 1.0, 'y': 0.5}
    vspec = A.to_vspec(ext, dims)
    values, arrays = _staggered_values(np.random.default_rng(4), res, vspec, dims)
    out = A.semi_lagrangian_staggered(values, ext, values, ext, dx, dims, res, 0.3)
    ref = O.semi_lagrangian_staggered(arrays, vspec, arrays, vspec, res, (0.0, 0.0), (12.0, 5.0), 0.3)
    for c, d in enumerate(dims):
        np.testing.assert_allclose(out[{'~vector': d}].numpy(dims), ref[c], atol=1e-6)
    s = np.random.default_rng(5).standard_normal(res).astype(np.float32)
    st = math.tensor(s, spatial(x=12, y=10))
    adv = A.semi_lagrangian_centered(st, E.BOUNDARY, values, ext, dx, dims, res, 0.3)
    np.testing.assert_allclose(adv.numpy(dims), O.semi_lagrangian_centered(s, O.uniform_bc(2, 'zg'), arrays, vspec, (0.0, 0.0), (12.0, 5.0), 0.3), atol=1e-6)
    # laplace against the vendored phiml itself (PhiML/phiml/math/_nd.py:825-861)
    lap = A.laplace(st, E.ZERO_GRADIENT, dx, dims, res)
    ref_lap = math.laplace(st, dx=math.vec(x=1.0, y=0.5), padding=E.ZERO_GRADIENT)
    np.testing.assert_allclose(lap.numpy(dims), ref_lap.numpy(dims), atol=2e-5)
    div = A.divergence(values, ext, dx, dims, res)
    np.testing.assert_allclose(div.numpy(dims), O.divergence_staggered(arrays, (1.0, 0.5), O.component_bcs(vspec, 2)), atol=1e-6)


# ---- the Backend subclass -----------------------------------------------------------------------------------------------------------
def test_backend_registration_and_fall_through(fake_engine):
    from phiml.backend import Backend, BACKENDS
    from phiflow_b200.phi_cuda._backend import get_backend, PhiCudaBackend, PoissonOperator
    b = get_backend()
    assert isinstance(b, PhiCudaBackend) and b in BACKENDS and b.name == 'phicuda'
    assert [x.name for x in BACKENDS].count('phicuda') == 1
    assert b.supports(Backend.grid_sample) and b.supports(Backend.linear_solve)
    f = lambda x: x + 1
    assert b.jit_compile(f) is f                         # ctypes launches are never traced (SURVEY.md Appendix C)
    # unknown linear operators go to the stock torch implementation
    mat = torch.tensor([[4.0, 1.0], [1.0, 3.0]])
    y = torch.tensor([[1.0, 2.0]])
    res = b.linear_solve('CG', mat, y, torch.zeros_like(y), np.array([1e-6]), np.array([1e-6]), np.array([[100]]), None, None)
    np.testing.assert_allclose(np.asarray(res.x)[0], np.linalg.solve(mat.numpy(), y.numpy()[0]), atol=1e-4)
    # grid_sample on tensors the fast path does not own (fp64: never downcast) -> exactly what the stock torch backend answers
    # (values or NotImplemented, after which phiml runs its own fallback, _ops.py:983-1015); fp32 on the engine's device -> the plugin
    from phiml.backend.torch._torch_backend import TorchBackend
    grid = torch.arange(12, dtype=torch.float32).reshape(1, 4, 3, 1)
    pts = torch.tensor([[[0.5, 0.0], [1.5, 1.0], [2.25, 1.5]]])
    np.testing.assert_allclose(np.asarray(b.grid_sample(grid, pts, 'boundary')).ravel(), [1.5, 5.5, 8.25], atol=1e-5)
    with math.precision(64):                     # (under precision 32 the torch backend itself casts fp64 natives to fp32)
        out, stock = b.grid_sample(grid.double(), pts.double(), 'boundary'), TorchBackend.grid_sample(b, grid.double(), pts.double(), 'boundary')
        if stock is NotImplemented:
            assert out is NotImplemented
        else:
            assert out.dtype == torch.float64
            np.testing.assert_allclose(np.asarray(out).ravel(), np.asarray(stock).ravel(), atol=1e-12)
    assert A.grid_sample_native(grid, pts, 'symmetric') is NotImplemented
    assert A.grid_sample_native(grid.double(), pts.double(), 'boundary') is NotImplemented
    with pytest.raises(NotImplementedError):
        b.linear_solve('biCG-stab(2)', PoissonOperator((4, 4), (1.0, 1.0), A.to_vspec(E.ZERO, ('x', 'y'))), y, y, [1e-5], [1e-5], np.array([[10]]), None, None)


# ---- phiml's own dispatch: math.grid_sample / Backend.linear_solve reach the plugin -----------------------------------------------------
@pytest.mark.parametrize('ext', [E.ZERO, E.ZERO_GRADIENT, E.PERIODIC], ids=['zeros', 'boundary', 'periodic'])
@pytest.mark.parametrize('res', [(9, 7), (6, 5, 4)], ids=['2d', '3d'])
def test_math_grid_sample_dispatches_to_the_plugin(fake_engine, monkeypatch, res, ext):
    """PhiML/phiml/math/_ops.py:973-1003: with phicuda as the default backend, math.grid_sample hands the native grid
    (batch, x, y[, z], channel) and coordinates (batch, points, d) to PhiCudaBackend.grid_sample.  Reference: the same call on
    the stock NumPy backend."""
    from phiml.math import instance
    from phiflow_b200.phi_cuda._backend import get_backend
    calls = []
    real = A.grid_sample_native
    monkeypatch.setattr(A, 'grid_sample_native', lambda g, c, m: calls.append(m) or real(g, c, m))
    d = len(res)
    names = 'xyz'[:d]
    rng = np.random.default_rng(d)
    g = rng.standard_normal((2,) + res + (2,)).astype(np.float32)
    c = (rng.random((2, 40, d)) * (np.array(res) + 3.0) - 2.0).astype(np.float32)
    gshape = batch(b=2) & spatial(**dict(zip(names, res))) & channel(comp=2)
    cshape = batch(b=2) & instance(points=40) & channel(vector=','.join(names))
    ref = math.grid_sample(math.tensor(g, gshape), math.tensor(c, cshape), ext)
    with get_backend():
        out = math.grid_sample(math.tensor(g, gshape, convert=True), math.tensor(c, cshape, convert=True), ext)
    assert calls == [ext.native_grid_sample_mode]
    assert isinstance(out.native(out.shape), torch.Tensor)
    np.testing.assert_allclose(out.numpy('b,points,comp'), ref.numpy('b,points,comp'), atol=1e-5)


@pytest.mark.parametrize('method', ['CG', 'CG-adaptive'])
def test_backend_linear_solve_with_poisson_operator(fake_engine, method):
    """Same system through the reference's solver (phiml NUMPY backend = _linalg.py unmodified) and through
    PhiCudaBackend.linear_solve with the PoissonOperator tag: natives are (batch, cells) in the reference's x-outermost order."""
    from phiml.backend import NUMPY
    from phiflow_b200.phi_cuda._backend import get_backend, PoissonOperator
    res, dx = (12, 10), (1.0, 0.5)
    vbc = ((0.0, 0.0), (0.0, 'zg'))
    Amat = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    y = np.random.default_rng(2).standard_normal((2, 120)).astype(np.float32)
    x0 = np.zeros_like(y)
    tol, mi = np.full(2, 1e-5, np.float32), np.full((1, 2), 1000)
    ref = NUMPY.linear_solve(method, Amat, y, x0, tol, tol, mi, None, None)
    got = get_backend().linear_solve(method, PoissonOperator(res, dx, vbc), torch.from_numpy(y), torch.from_numpy(x0), tol, tol, mi, None, None)
    assert 'phicuda' in got.method
    # the reference's batched run rounds differently from its own single-entry run (strided sums over the transposed matvec result:
    # entry 1 stops at 50 iterations in a batch of two, at 49 alone), the stand-in solves entry by entry
    assert np.abs(np.asarray(got.iterations) - np.asarray(ref.iterations)).max() <= 1
    np.testing.assert_allclose(got.x.numpy(), np.asarray(ref.x), atol=2e-5 * np.abs(ref.x).max())
    assert np.asarray(got.converged).all()
