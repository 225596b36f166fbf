"""
Pins the CPU oracle (oracle/oracle_np.py) against
  (1) fixtures recorded from the reference's own arithmetic layer (tests/golden/phiml_golden.npz, produced by
      tests/golden/make_golden.py from the vendored phiml 1.7.2 NumPy backend), and
  (2) the known-answer tests of the reference's test-suite (SURVEY.md §4), re-expressed on raw arrays.
CPU only.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle_np as O  # noqa: E402

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'phiml_golden.npz'))


def spec_from_arr(arr):
    def one(v):
        if np.isnan(v):
            return O.PERIODIC
        if np.isinf(v):
            return O.ZG
        return float(v)
    return tuple((one(lo), one(hi)) for lo, hi in arr)


def names(prefix):
    return sorted({k.split('/')[1] for k in GOLD.files if k.startswith(prefix + '/')})


@pytest.mark.parametrize('name', names('pad'))
def test_pad_matches_phiml(name):
    a = GOLD[f'pad/{name}/in']
    bc = spec_from_arr(GOLD[f'pad/{name}/bc'])
    d = a.ndim
    np.testing.assert_array_equal(O.pad(a, [(2, 1)] * d, bc), GOLD[f'pad/{name}/out_2_1'])
    widths = [(1, -1), (-1, 2)] + [(0, 0)] * (d - 2)
    np.testing.assert_array_equal(O.pad(a, widths, bc), GOLD[f'pad/{name}/out_neg'])


@pytest.mark.parametrize('name', names('laplace'))
def test_laplace_matches_phiml(name):
    a = GOLD[f'pad/{name}/in']
    bc = spec_from_arr(GOLD[f'pad/{name}/bc'])
    dx = GOLD[f'laplace/{name}/dx']
    ref = GOLD[f'laplace/{name}/out']
    np.testing.assert_allclose(O.laplace(a, dx, bc), ref, rtol=0, atol=2e-6 * np.abs(ref).max())


@pytest.mark.parametrize('name', names('fluid'))
def test_divergence_gradient_matrix_match_phiml(name):
    vbc = spec_from_arr(GOLD[f'fluid/{name}/bc'])
    dx = GOLD[f'fluid/{name}/dx']
    d = len(vbc)
    v = [GOLD[f'fluid/{name}/v{c}'] for c in range(d)]
    res = GOLD[f'fluid/{name}/p'].shape
    assert [c.shape for c in v] == O.staggered_shapes(res, vbc)
    div = O.divergence_staggered(v, dx, O.component_bcs(vbc, d))
    np.testing.assert_allclose(div, GOLD[f'fluid/{name}/div'], rtol=0, atol=1e-5)
    p = GOLD[f'fluid/{name}/p']
    pbc = O.pressure_bc(vbc)
    grad = O.gradient_faces(p, dx, pbc, vbc)
    for c in range(d):
        np.testing.assert_allclose(grad[c], GOLD[f'fluid/{name}/grad{c}'], rtol=0, atol=1e-5)
    A = O.poisson_matrix(res, dx, pbc)
    if f'fluid/{name}/matrix' in GOLD.files:
        np.testing.assert_allclose(A.toarray(), GOLD[f'fluid/{name}/matrix'], rtol=1e-6, atol=1e-6)
    lap_p = A.dot(p.ravel()).reshape(res)
    ref = GOLD[f'fluid/{name}/lap_p']
    np.testing.assert_allclose(lap_p, ref, rtol=0, atol=3e-6 * np.abs(ref).max())
    # the matrix equals the laplace stencil with the pressure boundary (Appendix A of SURVEY.md)
    np.testing.assert_allclose(O.laplace(p, dx, pbc), ref, rtol=0, atol=3e-6 * np.abs(ref).max())


@pytest.mark.parametrize('name', names('sample'))
def test_grid_sample_matches_phiml(name):
    bc = spec_from_arr(GOLD[f'sample/{name}/bc'])
    grid = GOLD[f'sample/{name}/grid']
    coords = GOLD[f'sample/{name}/coords']
    np.testing.assert_allclose(O.grid_sample(grid, coords, bc), GOLD[f'sample/{name}/out'], rtol=0, atol=2e-6)
    np.testing.assert_array_equal(O.closest_grid_values(grid, coords, bc), GOLD[f'sample/{name}/closest'])


def test_half_shift_average_matches_sample_subgrid():
    a = GOLD['subgrid/in']
    np.testing.assert_array_equal(O._half_shift_average(a, 0)[:, :6], GOLD['subgrid/x_half'])
    np.testing.assert_array_equal(O._half_shift_average(O._half_shift_average(a, 0), 1), GOLD['subgrid/xy_half'])
    np.testing.assert_array_equal(O._half_shift_average(a, 1)[1:7], GOLD['subgrid/y_half_off1'])


@pytest.mark.parametrize('name', names('cg'))
@pytest.mark.parametrize('tag,rtol', [('r3', 1e-3), ('r5', 1e-5)])
def test_cg_matches_phiml_solve_linear(name, tag, rtol):
    vbc = spec_from_arr(GOLD[f'cg/{name}/bc'])
    dx = GOLD[f'cg/{name}/dx']
    rhs = GOLD[f'cg/{name}/rhs']
    res = rhs.shape
    pbc = O.pressure_bc(vbc)
    A = O.poisson_matrix(res, dx, pbc)
    rank_def = not O.is_flexible(vbc)
    offset = O.estimate_matrix_offset(A, rhs.size, np.random.default_rng(7)) if rank_def else None
    info = O.cg(A, rhs, np.zeros(res, np.float32), rtol, 1e-5, 1000, offset)
    x_ref = GOLD[f'cg/{name}/{tag}/x']
    it_ref = int(GOLD[f'cg/{name}/{tag}/iterations'])
    assert info['converged'] and not info['diverged']
    # iteration counts agree up to fp32 rounding-order effects (the random probe only enters at the 1e-7 level)
    assert abs(info['iterations'] - it_ref) <= max(2, it_ref // 10), (info['iterations'], it_ref)
    scale = np.abs(x_ref).max()
    np.testing.assert_allclose(info['x'].reshape(res), x_ref, rtol=0, atol=20 * rtol * scale)


GOLD_ACG = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'phiml_cg_adaptive.npz'))


@pytest.mark.parametrize('name', ['open', 'mixed', 'mixed3'])
@pytest.mark.parametrize('tag,rtol', [('r3', 1e-3), ('r5', 1e-5)])
def test_cg_adaptive_matches_phiml_solve_linear(name, tag, rtol):
    """Solve('CG-adaptive') of the vendored PhiML (_linalg.py:93-128) vs oracle.cg_adaptive on the same pressure systems."""
    vbc = spec_from_arr(GOLD_ACG[f'{name}/bc'])
    dx = GOLD_ACG[f'{name}/dx']
    rhs = GOLD_ACG[f'{name}/rhs']
    res = rhs.shape
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    assert O.is_flexible(vbc)
    info = O.cg_adaptive(A, rhs, np.zeros(res, np.float32), rtol, 1e-5, 1000, None)
    it_ref = int(GOLD_ACG[f'{name}/{tag}/iterations'])
    assert info['converged'] and not info['diverged']
    assert abs(info['iterations'] - it_ref) <= max(2, it_ref // 10), (info['iterations'], it_ref)
    assert info['function_evaluations'] == info['iterations'] + 1
    assert int(GOLD_ACG[f'{name}/{tag}/function_evaluations']) == it_ref + 1
    x_ref = GOLD_ACG[f'{name}/{tag}/x']
    np.testing.assert_allclose(info['x'].reshape(res), x_ref, rtol=0, atol=20 * rtol * np.abs(x_ref).max())


GOLD_COL = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'phiml_collocated.npz'))


@pytest.mark.parametrize('name', ['zero', 'open', 'periodic', 'mixed', 'one', 'mixed3', 'lid', 'inflow3'])
def test_collocated_gradient_divergence_matrix_match_phiml(name):
    """CenteredGrid-velocity variant (SURVEY.md Appendix A; fluid.py:154-155,197-202): central gradient, centred divergence
    and the traced wide-stencil operator of the vendored PhiML vs the oracle.  'lid' and 'inflow3' carry per-component constants
    (a vector-valued ConstantExtrapolation): each component's divergence term sees its own constant, the operator none."""
    arr = GOLD_COL[f'{name}/bc']
    vbc = [spec_from_arr(a) for a in arr] if arr.ndim == 3 else spec_from_arr(arr)
    dx = GOLD_COL[f'{name}/dx']
    p = GOLD_COL[f'{name}/p']
    d = p.ndim
    pbc = O.pressure_bc(vbc)
    kinds = O.kinds_of(vbc)
    for c, g in enumerate(O.gradient_centered(p, dx, pbc)):
        np.testing.assert_allclose(g, GOLD_COL[f'{name}/grad{c}'], rtol=1e-6, atol=1e-6)
    comps = [GOLD_COL[f'{name}/v{c}'] for c in range(d)]
    np.testing.assert_allclose(O.divergence_centered(comps, dx, O.component_bcs(vbc, d)), GOLD_COL[f'{name}/div'], rtol=1e-6, atol=2e-6)
    np.testing.assert_allclose(O.wide_laplace(p, dx, pbc, kinds), GOLD_COL[f'{name}/lap'], rtol=1e-5, atol=1e-5)
    A = O.wide_poisson_matrix(p.shape, dx, kinds)
    np.testing.assert_allclose(A.toarray(), GOLD_COL[f'{name}/matrix'], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(A.dot(p.ravel()).reshape(p.shape), GOLD_COL[f'{name}/lap'], rtol=1e-5, atol=1e-5)


def test_collocated_interior_row_is_the_wide_stencil():
    """Appendix A: [1 0 -2 0 1] / (4 dx^2) per axis in the interior."""
    A = O.wide_poisson_matrix((9,), (0.5,), ((0.0, 0.0),)).toarray()
    np.testing.assert_allclose(A[4, 2:7], np.array([1, 0, -2, 0, 1]) / (4 * 0.25), atol=1e-6)


@pytest.mark.parametrize('vbc', [((0.0, 0.0), (0.0, 0.0)), (('zg', 'zg'), ('zg', 'zg'))])
def test_collocated_projection_removes_centred_divergence(vbc):
    """tests/commit/physics/test_fluid.py:17-28,34-36 (CenteredGrid with ZERO and BOUNDARY): two rounds of buoyancy from a
    sphere of smoke + make_incompressible on a 16 x 20 grid over [0,100]^2; the centred divergence ends below 5e-5."""
    res, dx = (16, 20), (100 / 16, 100 / 20)
    pts = O.points_of((0.0, 0.0), (100.0, 100.0), res)
    smoke = (np.sum((pts - np.array([40.0, 10.0], np.float32)) ** 2, -1) <= 25.0).astype(np.float32)
    v = [np.zeros(res, np.float32), np.zeros(res, np.float32)]
    for _ in range(2):
        v = [v[0], v[1] + smoke * np.float32(0.1)]
        v, p, info = O.make_incompressible_centered(v, vbc, res, dx)          # 'auto' = CG-adaptive in the vendored PhiML
        assert not info['diverged'] and (info['converged'] or not O.is_flexible(vbc))
    div = O.divergence_centered(v, dx, O.component_bcs(vbc, 2))
    assert np.abs(div).max() < 5e-5, np.abs(div).max()                       # the reference test's own tolerance
    # plain CG is the wrong solver for this operator: its boundary rows make it non-symmetric (walls and open sides alike)
    A = O.wide_poisson_matrix(res, dx, vbc).toarray()
    assert np.abs(A - A.T).max() > 1e-3


# ----------------------------------------------------------------------------------------------------
# known-answer tests of the reference suite
# ----------------------------------------------------------------------------------------------------

def test_staggered_grid_sizes_by_extrapolation():
    """tests/commit/field/test__grid.py:25-37"""
    res = (20, 10)
    assert O.staggered_shapes(res, O.uniform_bc(2, O.ZERO)) == [(19, 10), (20, 9)]
    assert O.staggered_shapes(res, O.uniform_bc(2, O.PERIODIC)) == [(20, 10), (20, 10)]
    assert O.staggered_shapes(res, O.uniform_bc(2, O.ZG)) == [(21, 10), (20, 11)]


def test_grid_sample_known_answers():
    """PhiML/tests/commit/math/test__ops.py:232-245"""
    grid = np.array([[1, 2], [3, 4]], np.float32)        # dims (x, y) -> tensor([[1,2],[3,4]], spatial('x,y'))
    coords = np.array([[0, 0], [0.5, 0], [0, 0.5], [-2, -1]], np.float32)
    np.testing.assert_allclose(O.grid_sample(grid, coords, O.uniform_bc(2, O.ZERO)), [1, 2, 1.5, 0], atol=1e-6)
    grid1 = np.array([0, 1], np.float32)
    coords1 = np.array([[-1], [1], [0.5]], np.float32)
    np.testing.assert_allclose(O.grid_sample(grid1, coords1, O.uniform_bc(1, O.ZERO)), [0, 1, 0.5], atol=1e-6)


def test_closest_grid_values_known_answer():
    """PhiML/tests/commit/math/test__ops.py:317-321: 1-D grid [0,1,2,3], coordinate 0.5 -> neighbours (0, 1)."""
    grid = np.array([0, 1, 2, 3], np.float32)
    closest = O.closest_grid_values(grid, np.array([[0.5]], np.float32), O.uniform_bc(1, O.ZERO))
    np.testing.assert_array_equal(closest, [[0, 1]])


def test_poisson_1d_known_answers():
    """PhiML/tests/commit/math/test__optimize.py:62-70, 145-153: laplace(ZERO) x = 1 -> [-1.5, -2, -1.5];
    Dirichlet ONE -> [-0.5, -1, -0.5] (constant part moved to the right-hand side)."""
    A = O.poisson_matrix((3,), (1.0,), ((0.0, 0.0),))
    y = np.ones(3, np.float32)
    info = O.cg(A, y, np.zeros(3, np.float32), 1e-5, 1e-5, 100)
    np.testing.assert_allclose(info['x'], [-1.5, -2, -1.5], atol=1e-3)
    assert info['iterations'] == 2                      # test__optimize.py:95-112 (SolveTape contract)
    y_one = y - np.array([1, 0, 1], np.float32)         # ghost value 1 on both sides
    info = O.cg(A, y_one, np.zeros(3, np.float32), 1e-5, 1e-5, 100)
    np.testing.assert_allclose(info['x'], [-0.5, -1, -0.5], atol=1e-3)


def test_self_advect_staggered_known_answer():
    """tests/commit/physics/test_advect.py:41-45: 4x3 staggered box field (walls) advected by itself, dt=1."""
    res = (4, 3)
    vbc = O.uniform_bc(2, O.ZERO)
    shapes = O.staggered_shapes(res, vbc)
    # StaggeredGrid(Box(x=(.9, 2.6), y=(.9, 2)), 0, x=4, y=3) * (0, 1): y-faces whose centres lie inside the box are 1
    vx = np.zeros(shapes[0], np.float32)
    vy = np.zeros(shapes[1], np.float32)
    lo_y, up_y, res_y = O.component_grid((0, 0), (4, 3), res, vbc, 1)
    pts = O.points_of(lo_y, up_y, res_y)
    inside = (pts[..., 0] >= .9) & (pts[..., 0] <= 2.6) & (pts[..., 1] >= .9) & (pts[..., 1] <= 2)
    vy[inside] = 1
    out = O.semi_lagrangian_staggered([vx, vy], vbc, [vx, vy], vbc, res, (0, 0), (4, 3), 1.0)
    np.testing.assert_allclose(out[1].T, [[0, 0, 0, 0], [0, 1, 1, 0]], atol=1e-6)   # numpy('y,x')
    np.testing.assert_allclose(out[0], 0, atol=1e-6)


@pytest.mark.parametrize('bc', [O.uniform_bc(2, O.ZERO), O.uniform_bc(2, O.ZG), O.uniform_bc(2, O.PERIODIC)])
def test_advection_identities(bc):
    """tests/commit/physics/test_advect.py:12-18: adv(s, v, 0) == adv(s, 0*v, 1) == s."""
    rng = np.random.default_rng(0)
    res = (8, 6)
    vbc = bc
    v = [rng.standard_normal(s).astype(np.float32) for s in O.staggered_shapes(res, vbc)]
    zero_v = [np.zeros_like(c) for c in v]
    s = rng.standard_normal(res).astype(np.float32)
    sbc = O.uniform_bc(2, O.ZG)
    for fun in (O.semi_lagrangian_centered, O.mac_cormack_centered):
        np.testing.assert_allclose(fun(s, sbc, v, vbc, (0, 0), (8, 6), 0.0), s, atol=1e-5)
        np.testing.assert_allclose(fun(s, sbc, zero_v, vbc, (0, 0), (8, 6), 1.0), s, atol=1e-5)
    out = O.semi_lagrangian_staggered(v, vbc, v, vbc, res, (0, 0), (8, 6), 0.0)
    for a, b in zip(out, v):
        np.testing.assert_allclose(a, b, atol=1e-5)
    out = O.semi_lagrangian_staggered(v, vbc, zero_v, vbc, res, (0, 0), (8, 6), 1.0)
    for a, b in zip(out, v):
        np.testing.assert_allclose(a, b, atol=1e-5)


@pytest.mark.parametrize('vbc', [O.uniform_bc(2, O.ZERO), O.uniform_bc(2, O.ZG), O.uniform_bc(2, O.PERIODIC),
                                 ((O.ZG, O.ZG), (O.ZERO, O.ZG))])
def test_make_incompressible_removes_divergence(vbc):
    """tests/commit/physics/test_fluid.py:19-53: 16x20 grid, 2 buoyancy+projection steps, divergence ~ 0 (5e-5)."""
    res = (16, 20)
    lower, upper = (0, 0), (100, 100)
    dx = [100 / 16, 100 / 20]
    shapes = O.staggered_shapes(res, vbc)
    smoke = O.sphere_soft_mask((50, 10), 5, lower, upper, res)          # CenteredGrid(Sphere(x=50, y=10, radius=5))
    sbc = O.uniform_bc(2, O.ZERO)
    v = [np.zeros(s, np.float32) for s in shapes]
    for _ in range(2):
        faces = O.centered_to_faces(smoke, sbc, vbc)
        v = [v[0] + faces[0] * np.float32(0), v[1] + faces[1] * np.float32(0.1)]
        v, p, info = O.make_incompressible(v, vbc, res, dx, rtol=1e-5, atol=1e-5)
        assert info['converged']
    div = O.divergence_staggered(v, dx, O.component_bcs(vbc, 2))
    assert np.abs(div).max() < 5e-5


@pytest.mark.parametrize('name', names('obst'))
def test_obstacle_masks_and_masked_laplace_match_phiml(name):
    """SURVEY N4: hard_bcs = stagger(accessible, minimum) and masked_laplace with where(active, div, p)
    (phi/physics/fluid.py:130-137, 197-202), traced to a matrix by the reference's own jit_compile_linear."""
    vbc = spec_from_arr(GOLD[f'obst/{name}/bc'])
    dx = GOLD[f'obst/{name}/dx']
    acc = GOLD[f'obst/{name}/accessible']
    d = acc.ndim
    hard = O.hard_bcs_faces(acc, vbc)
    for c in range(d):
        np.testing.assert_array_equal(hard[c], GOLD[f'obst/{name}/hard{c}'])
    A = O.masked_poisson_matrix(acc.shape, dx, vbc, acc)
    p = GOLD[f'obst/{name}/p']
    ref = GOLD[f'obst/{name}/lap_p']
    np.testing.assert_allclose(A.dot(p.ravel()).reshape(acc.shape), ref, rtol=0, atol=4e-6 * np.abs(ref).max())
    if f'obst/{name}/matrix' in GOLD.files:
        np.testing.assert_allclose(A.toarray(), GOLD[f'obst/{name}/matrix'], rtol=1e-6, atol=1e-6)


def test_masked_matrix_sparse_assembly_matches_column_builder():
    """oracle.masked_poisson_matrix switches to an O(n) face-by-face assembly above DENSE_MASKED_MATRIX_LIMIT cells (the
    column-by-column builder needs an n x n dense array: 2.5 TB at 256 x 64 x 48).  Both must give the same matrix for every
    boundary kind and random obstacle masks; the column builder is the one pinned against the phiml-traced matrix."""
    import itertools
    rng = np.random.default_rng(0)
    kinds = [('periodic', 'periodic'), (0.0, 0.0), ('zg', 'zg'), (0.0, 'zg'), ('zg', 0.0)]
    old = O.DENSE_MASKED_MATRIX_LIMIT
    try:
        O.DENSE_MASKED_MATRIX_LIMIT = 10 ** 9
        for d, res in ((2, (7, 6)), (3, (5, 4, 6))):
            for combo in itertools.product(kinds, repeat=d):
                acc = (rng.uniform(size=res) > 0.25).astype(np.float32)
                dx = tuple(rng.uniform(0.3, 2.0, d))
                a = O.masked_poisson_matrix(res, dx, tuple(combo), acc).toarray()
                b = O.masked_poisson_matrix_sparse(res, dx, tuple(combo), acc).toarray()
                assert np.abs(a - b).max() <= 2e-6 * np.abs(a).max(), combo
    finally:
        O.DENSE_MASKED_MATRIX_LIMIT = old
    # and the switch itself: a grid above the limit never allocates the dense array
    big = O.masked_poisson_matrix((64, 32, 16), (1.0, 1.0, 1.0), ((0.0, 0.0),) * 3, np.ones((64, 32, 16), np.float32))
    assert big.shape == (32768, 32768) and big.nnz < 8 * 32768
