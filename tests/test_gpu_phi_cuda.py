"""
Row B1 on the GPU: the reference-side plugin `phiflow_b200/phi_cuda` with REAL phiml objects (the unmodified PhiML 1.7.2 that
`__graft_entry__.build()` installs into oracle/_ref, see tests/_phiml.py) and the REAL engine
(libphicuda.so through phiflow_b200._ops).  The comparison side is the reference library itself, run live on the box's CPU:

  * `phiml.math.grid_sample` with the NumPy backend   vs  the same call under `with get_backend():` -> phicuda_grid_sample_f32
  * `phiml.backend.NUMPY.linear_solve('CG' | 'CG-adaptive', csr, ...)` (= PhiML/phiml/backend/_linalg.py:23-128, unmodified)
                                                   vs  `PhiCudaBackend.linear_solve(..., PoissonOperator, ...)` -> k_cg_ring
  * `phiml.math.laplace`, pad + forward differences   vs  the adapter functions on phiml Tensors
  * fluid.make_incompressible on Field.values / Field.extrapolation (tests/commit/physics/test_fluid.py:38-53 cases) vs the oracle,
    and divergence-free by the reference's own arithmetic.

tests/test_phi_cuda_adapter.py runs the same plumbing on the CPU with an oracle-backed stand-in for the engine.
"""
import numpy as np
import pytest
import torch

from _phiml import ensure_phiml

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip('needs a CUDA device', allow_module_level=True)
if not ensure_phiml():
    pytest.skip('PhiML not available (neither installed nor in oracle/_ref)',
                allow_module_level=True)

from phiml import math  # noqa: E402
from phiml.backend import NUMPY  # noqa: E402
from phiml.math import extrapolation as E, spatial, batch, dual, channel, instance  # noqa: E402

from oracle import oracle_np as O  # noqa: E402
from phiflow_b200 import _ops  # noqa: E402
from phiflow_b200.phi_cuda import _adapter as A  # noqa: E402
from phiflow_b200.phi_cuda._backend import get_backend, PhiCudaBackend, PoissonOperator  # noqa: E402


def test_engine_is_the_cuda_library():
    assert A.ENGINE is _ops and A.DEVICE == 'cuda'
    b = get_backend()
    assert isinstance(b, PhiCudaBackend) and b.name == 'phicuda'
    with b:
        t = math.tensor(np.zeros((3, 2), np.float32), spatial(x=3, y=2), convert=True)
        assert t.default_backend is b
        assert t.native(t.shape).is_cuda


# ---- math.grid_sample: stock NumPy backend vs the phicuda backend through phiml's own dispatch -------------------------------------
@pytest.fixture()
def count_native_calls(monkeypatch):
    calls = {'native': 0, 'fallback': 0}
    real = A.grid_sample_native

    def wrapped(grid, coords, mode):
        out = real(grid, coords, mode)
        calls['fallback' if out is NotImplemented else 'native'] += 1
        return out
    monkeypatch.setattr(A, 'grid_sample_native', wrapped)
    return calls


@pytest.mark.parametrize('ext', [E.ZERO, E.ZERO_GRADIENT, E.PERIODIC], ids=['zeros', 'boundary', 'periodic'])
@pytest.mark.parametrize('res', [(37, 22), (19, 14, 11)], ids=['2d', '3d'])
def test_math_grid_sample_runs_the_cuda_kernel(res, ext, count_native_calls):
    """PhiML/phiml/math/_ops.py:973-1003 calls backend.grid_sample(native grid, native coordinates, mode); with phicuda as the
    default backend that is phicuda_grid_sample_f32.  Points reach two cells outside the grid on every side."""
    d = len(res)
    names = 'xyz'[:d]
    rng = np.random.default_rng(7 + d)
    nb, npts = 3, 4001
    g = rng.standard_normal((nb,) + res).astype(np.float32)
    c = (rng.random((nb, npts, d)) * (np.array(res) + 3.0) - 2.0).astype(np.float32)
    c[:, :d] = np.eye(d, dtype=np.float32) * (np.array(res, np.float32) - 1)     # exact grid points, incl. the upper edge
    gshape = batch(b=nb) & spatial(**dict(zip(names, res)))
    cshape = batch(b=nb) & instance(points=npts) & channel(vector=','.join(names))
    ref = math.grid_sample(math.tensor(g, gshape), math.tensor(c, cshape), ext)
    assert ref.default_backend is NUMPY
    with get_backend():
        gt, ct = math.tensor(g, gshape, convert=True), math.tensor(c, cshape, convert=True)
        out = math.grid_sample(gt, ct, ext)
    assert count_native_calls == {'native': 1, 'fallback': 0}
    assert out.shape == ref.shape and out.native(out.shape).is_cuda
    np.testing.assert_allclose(out.numpy('b,points'), ref.numpy('b,points'), atol=4e-6 * float(np.abs(g).max()), rtol=0)


def test_grid_sample_with_channels_and_spatial_point_sets(count_native_calls):
    """Grids with a channel dim (all staggered components at once) and coordinates on a spatial lattice - the shapes
    advect.semi_lagrangian produces (phi/physics/advect.py:156-179, phi/field/_resample.py:238)."""
    rng = np.random.default_rng(11)
    g = rng.standard_normal((2, 12, 10, 3)).astype(np.float32)
    c = (rng.random((2, 12, 10, 2)) * np.array([13.0, 11.0]) - 1.0).astype(np.float32)
    gshape = batch(b=2) & spatial(x=12, y=10) & channel(comp=3)
    cshape = batch(b=2) & spatial(x=12, y=10) & channel(vector='x,y')
    ref = math.grid_sample(math.tensor(g, gshape), math.tensor(c, cshape), E.ZERO_GRADIENT)
    with get_backend():
        out = math.grid_sample(math.tensor(g, gshape, convert=True), math.tensor(c, cshape, convert=True), E.ZERO_GRADIENT)
    assert count_native_calls['native'] == 1 and count_native_calls['fallback'] == 0
    np.testing.assert_allclose(out.numpy('b,x,y,comp'), ref.numpy('b,x,y,comp'), atol=2e-5, rtol=0)


def test_ineligible_grid_sample_falls_through_to_the_stock_backend(count_native_calls):
    """fp64 grids are never downcast: the override answers what TorchBackend answers."""
    g = np.arange(20, dtype=np.float64).reshape(1, 5, 4)
    c = np.array([[[0.5, 0.5], [3.25, 2.0]]])
    with math.precision(64):
        ref = math.grid_sample(math.tensor(g, batch(b=1) & spatial(x=5, y=4)), math.tensor(c, batch(b=1) & instance(points=2) & channel(vector='x,y')), E.ZERO)
        with get_backend():
            out = math.grid_sample(math.tensor(g, batch(b=1) & spatial(x=5, y=4), convert=True),
                                   math.tensor(c, batch(b=1) & instance(points=2) & channel(vector='x,y'), convert=True), E.ZERO)
    assert count_native_calls['native'] == 0
    np.testing.assert_allclose(out.numpy('b,points'), ref.numpy('b,points'), atol=1e-12)


# ---- Backend.linear_solve: the reference's own CG (unmodified _linalg.py on the box's CPU) vs the persistent CUDA kernel ----------
SOLVE_CASES = {
    'wall2d': ((48, 40), (1.0, 0.5), O.uniform_bc(2, 0.0)),
    'open2d': ((48, 40), (1.0, 1.0), O.uniform_bc(2, 'zg')),
    'periodic3d': ((24, 16, 20), (1.0, 1.0, 1.0), O.uniform_bc(3, 'periodic')),
    'mixed3d': ((20, 16, 12), (0.5, 1.0, 1.0), (('periodic', 'periodic'), (0.0, 0.0), (0.0, 'zg'))),
}


@pytest.mark.parametrize('method', ['CG', 'CG-adaptive'])
@pytest.mark.parametrize('case', list(SOLVE_CASES))
def test_linear_solve_matches_the_reference_cg(case, method):
    res, dx, vbc = SOLVE_CASES[case]
    n, nb = int(np.prod(res)), 3
    Amat = O.poisson_matrix(res, dx, O.pressure_bc(vbc))         # == the matrix phiml traces for masked_laplace (tests/golden)
    rng = np.random.default_rng(5)
    # smooth right-hand sides (a few low modes + noise) in the reference's flattening: x outermost
    y = rng.standard_normal((nb,) + res).astype(np.float32)
    if not O.is_flexible(vbc):
        y -= y.mean(axis=tuple(range(1, len(res) + 1)), keepdims=True)
    y = y.reshape(nb, n)
    x0 = np.zeros_like(y)
    rtol = atol = np.full(nb, 1e-5, np.float32)
    max_iter = np.full((1, nb), 1000)
    ref = NUMPY.linear_solve(method, Amat, y, x0, rtol, atol, max_iter, None, None)
    b = get_backend()
    got = b.linear_solve(method, PoissonOperator(res, dx, vbc), torch.from_numpy(y).cuda(), torch.from_numpy(x0).cuda(), rtol, atol,
                         max_iter, None, None)
    assert 'phicuda' in got.method
    gi, ri = np.asarray(got.iterations), np.asarray(ref.iterations)
    assert np.asarray(got.converged).all() and np.asarray(ref.converged).all()
    assert not np.asarray(got.diverged).any()
    # same algorithm, different fp32 summation order: the stopping iteration may move by a few
    assert np.all(np.abs(gi - ri) <= np.maximum(3, 0.1 * ri)), (gi, ri)
    xg, xr = got.x.cpu().numpy(), np.asarray(ref.x)
    if not O.is_flexible(vbc):                                      # rank-deficient: compare up to the constant mode
        xg, xr = xg - xg.mean(1, keepdims=True), xr - xr.mean(1, keepdims=True)
    scale = np.abs(xr).max()
    assert np.abs(xg - xr).max() <= 2e-3 * scale, np.abs(xg - xr).max() / scale
    # and both satisfy the system to the requested tolerance
    for i in range(nb):
        r = y[i].astype(np.float64) - Amat.astype(np.float64) @ xg[i].astype(np.float64)
        tol_sq = max(1e-10 * float(np.sum(y[i].astype(np.float64) ** 2)), 1e-10)
        assert float(np.sum(r * r)) <= 40 * tol_sq + 1e-9          # same bound as tests/test_gpu_kernels.py::test_cg_poisson


# ---- the adapter functions on phiml Tensors, real engine ----------------------------------------------------------------------
def _staggered_values(rng, res, vspec, dims, batch_shape=None):
    shapes = O.staggered_shapes(res, vspec)
    comps, arrays = [], []
    for s in shapes:
        pre = () if batch_shape is None else batch_shape.sizes
        a = rng.standard_normal(pre + s).astype(np.float32)
        arrays.append(a)
        shape = spatial(**dict(zip(dims, s)))
        comps.append(math.tensor(a, (batch_shape & shape) if batch_shape is not None else shape))
    return math.stack(comps, dual(vector=dims)), arrays


@pytest.mark.parametrize('method', ['CG', 'auto'])
@pytest.mark.parametrize('name', ['zero', 'boundary', 'periodic', 'mixed'])
def test_make_incompressible_on_phiml_tensors(name, method):
    dims, res = ('x', 'y'), (16, 20)
    ext = {'zero': E.ZERO, 'boundary': E.BOUNDARY, 'periodic': E.PERIODIC, 'mixed': E.combine_sides(x=E.BOUNDARY, y=(E.ZERO, E.BOUNDARY))}[name]
    dx = {'x': 100.0 / 16, 'y': 100.0 / 20}
    vspec = A.to_vspec(ext, dims)
    values, arrays = _staggered_values(np.random.default_rng(3), res, vspec, dims, batch(b=2))
    new_values, pressure, info = A.make_incompressible(values, ext, dx, dims, res, method=method, rel_tol=1e-5, abs_tol=1e-5)
    assert pressure.native(pressure.shape).is_cuda
    assert info['converged'].all() and not info['diverged'].any() and (info['iterations'] > 0).all()
    # (a) divergence-free by the reference's arithmetic: bake the boundary faces with math.pad, forward differences
    div = 0
    for d in dims:
        comp = new_values[{'~vector': d}]
        lo, hi = ext.valid_outer_faces(d)
        baked = math.pad(comp, {d: (0 if lo else 1, 0 if hi else 1)}, ext[{'vector': d}] if name != 'mixed' else ext)
        div = div + (baked[{d: slice(1, None)}] - baked[{d: slice(None, -1)}]) / dx[d]
    vmax = float(max(np.abs(a).max() for a in arrays))
    assert float(np.abs(div.numpy(div.shape.names)).max()) < 5e-5 * max(1.0, vmax)
    # (b) the projected velocity equals the oracle's (plain CG: same iterates up to rounding; 'auto' = CG-adaptive stops elsewhere,
    #     both are within the solve tolerance of the exact projection)
    for b in range(2):
        v_ref, p_ref, _ = O.make_incompressible([a[b] for a in arrays], vspec, res, (dx['x'], dx['y']), rtol=1e-5, atol=1e-5, use_matrix_offset=False)
        for c, d in enumerate(dims):
            got = new_values[{'~vector': d, 'b': b}].numpy(dims)
            assert np.abs(got - v_ref[c]).max() <= 2e-3 * vmax, (d, np.abs(got - v_ref[c]).max())


def test_advection_and_stencils_on_phiml_tensors():
    dims, res = ('x', 'y', 'z'), (12, 10, 9)
    ext = E.combine_sides(x=E.PERIODIC, y=E.ZERO, z=(E.ZERO, E.BOUNDARY))
    dx = {'x': 1.0, 'y': 0.5, 'z': 2.0}
    lower, upper = (0.0,) * 3, (12.0, 5.0, 18.0)
    vspec = A.to_vspec(ext, dims)
    values, arrays = _staggered_values(np.random.default_rng(4), res, vspec, dims)
    out = A.semi_lagrangian_staggered(values, ext, values, ext, dx, dims, res, 0.3)
    ref = O.semi_lagrangian_staggered(arrays, vspec, arrays, vspec, res, lower, upper, 0.3)
    for c, d in enumerate(dims):
        np.testing.assert_allclose(out[{'~vector': d}].numpy(dims), ref[c], atol=2e-5)
    s = np.random.default_rng(5).standard_normal(res).astype(np.float32)
    st = math.tensor(s, spatial(x=12, y=10, z=9))
    adv = A.semi_lagrangian_centered(st, E.BOUNDARY, values, ext, dx, dims, res, 0.3)
    np.testing.assert_allclose(adv.numpy(dims), O.semi_lagrangian_centered(s, O.uniform_bc(3, 'zg'), arrays, vspec, lower, upper, 0.3), atol=2e-5)
    # laplace against the reference library itself (PhiML/phiml/math/_nd.py:825-861), all three boundary kinds
    for lap_ext in (E.ZERO_GRADIENT, E.PERIODIC, E.ZERO):
        lap = A.laplace(st, lap_ext, dx, dims, res)
        ref_lap = math.laplace(st, dx=math.vec(x=1.0, y=0.5, z=2.0), padding=lap_ext)
        np.testing.assert_allclose(lap.numpy(dims), ref_lap.numpy(dims), atol=4e-5)
    # divergence against pad + forward differences in phiml (phi/field/_field_math.py:617-626)
    div = A.divergence(values, ext, dx, dims, res)
    ref_div = 0
    for d in dims:
        comp = values[{'~vector': d}]
        lo, hi = ext.valid_outer_faces(d)
        baked = math.pad(comp, {d: (0 if lo else 1, 0 if hi else 1)}, ext)
        ref_div = ref_div + (baked[{d: slice(1, None)}] - baked[{d: slice(None, -1)}]) / dx[d]
    np.testing.assert_allclose(div.numpy(dims), ref_div.numpy(dims), atol=2e-5)
