"""
The oracle against outputs of the reference LIBRARY (PhiML 1.7.2) on seeded inputs, for more shapes, boundary mixes and solver settings
than tests/golden/phiml_golden.npz holds.  The reference side was recorded into tests/golden/phiml_live.npz by
tests/golden/make_live_golden.py, which runs the functions below under PhiML; the inputs are regenerated here from the same seeds.

    O.pad / O.laplace / O.grid_sample / O.closest_grid_values     vs  phiml.math.pad / laplace / grid_sample / closest_grid_values
    O.cg / O.cg_adaptive on O.poisson_matrix                       vs  phiml.backend.NUMPY.linear_solve('CG' | 'CG-adaptive', ...)
                                                                       (= PhiML/phiml/backend/_linalg.py:23-128, unmodified)
"""
import os
import zlib

import numpy as np
import pytest

from oracle import oracle_np as O

AX = 'xyz'
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'phiml_live.npz')

SCALAR_BCS = {
    'zero': lambda d: O.uniform_bc(d, 0.0), 'const': lambda d: O.uniform_bc(d, 1.5), 'open': lambda d: O.uniform_bc(d, 'zg'),
    'periodic': lambda d: O.uniform_bc(d, 'periodic'),
    # one constant per mix: where two DIFFERENT constants meet in a corner ghost the reference pads them in the iteration order of a
    # Python set (extrapolation.py:1292-1301), i.e. the corner value is not defined by the reference itself
    'mixed': lambda d: ((('periodic', 'periodic'), (2.0, 'zg'), ('zg', 2.0)) if d == 3 else (('zg', 0.0), ('periodic', 'periodic'))),
    'walls_open_top': lambda d: ((0.0, 0.0),) * (d - 1) + ((0.0, 'zg'),),
}
RES = {2: [(9, 7), (16, 5)], 3: [(6, 5, 7)]}
DX = {2: (0.5, 1.25), 3: (0.5, 1.0, 2.0)}
PAD_WIDTHS = [(1, 2), (2, 1), (1, 1)]
NPTS = 300


@pytest.fixture(scope='module')
def golden():
    with np.load(GOLDEN) as f:
        return dict(f)


def pad_laplace_inputs(name, d):
    rng = np.random.default_rng(zlib.crc32(name.encode()) % 1000 + d)
    return [rng.standard_normal(res).astype(np.float32) for res in RES[d]]


def grid_sample_inputs(name, d):
    """points up to 2.5 cells outside on every side, plus the exact grid corners"""
    rng = np.random.default_rng(7 * d + len(name))
    res = RES[d][0]
    g = rng.standard_normal(res).astype(np.float32)
    pts = (rng.random((NPTS, d)) * (np.array(res) + 4.0) - 2.5).astype(np.float32)
    pts[:d] = np.eye(d, dtype=np.float32) * (np.array(res, np.float32) - 1)
    return g, pts


@pytest.mark.parametrize('d', [2, 3])
@pytest.mark.parametrize('name', sorted(SCALAR_BCS))
def test_pad_and_laplace(name, d, golden):
    bc = SCALAR_BCS[name](d)
    for i, a in enumerate(pad_laplace_inputs(name, d)):
        np.testing.assert_array_equal(O.pad(a, PAD_WIDTHS[:d], bc), golden[f'pad/{name}/{d}/{i}'])
        np.testing.assert_array_equal(O.laplace(a, DX[d], bc), golden[f'laplace/{name}/{d}/{i}'])


@pytest.mark.parametrize('d', [2, 3])
@pytest.mark.parametrize('name', sorted(SCALAR_BCS))
def test_grid_sample_and_closest_values(name, d, golden):
    """PhiML/phiml/math/_ops.py:878-1015: native modes (zeros / boundary / periodic) and the pad-one-layer fallback for constants
    other than 0 and for mixed boundaries; points up to 2.5 cells outside on every side."""
    bc = SCALAR_BCS[name](d)
    g, pts = grid_sample_inputs(name, d)
    res = g.shape
    want = golden[f'grid_sample/{name}/{d}']
    got = O.grid_sample(g, pts, bc)
    # the reference's fallback pads ONE layer, so for non-native modes it is only defined within one cell of the grid
    # (documented in math.grid_sample: "values lying further outside will not be sampled according to the extrapolation")
    native = name in ('zero', 'open', 'periodic')
    near = np.all((pts >= -1.0) & (pts <= np.array(res, np.float32)), axis=1)
    sel = np.ones(NPTS, bool) if native else near
    np.testing.assert_allclose(got[sel], want[sel], rtol=0, atol=2e-6 * float(np.abs(g).max()))
    want_c = golden[f'closest/{name}/{d}']
    got_c = O.closest_grid_values(g, pts, bc)
    np.testing.assert_array_equal(got_c[sel].reshape(want_c[sel].shape), want_c[sel])


VEL_BCS = {
    'wall': lambda d: O.uniform_bc(d, 0.0), 'open': lambda d: O.uniform_bc(d, 'zg'), 'periodic': lambda d: O.uniform_bc(d, 'periodic'),
    'mixed': lambda d: ((('periodic', 'periodic'), (0.0, 0.0), (0.0, 'zg')) if d == 3 else (('zg', 'zg'), (0.0, 'zg'))),
}


def cg_inputs(name, d):
    """(matrix, right-hand side, [(rtol, atol, max_iter, x0)]): full solves, truncated solves, warm starts, the plume's tolerance"""
    vbc = VEL_BCS[name](d)
    res = (12, 10) if d == 2 else (8, 6, 7)
    Amat = O.poisson_matrix(res, DX[d], O.pressure_bc(vbc))
    rng = np.random.default_rng(11 + d)
    y = rng.standard_normal(res).astype(np.float32)
    if not O.is_flexible(vbc):
        y -= y.mean(dtype=np.float32)
    x_warm = (0.1 * rng.standard_normal(res)).astype(np.float32)
    zero = np.zeros(res, np.float32)
    settings = [(1e-5, 1e-5, 1000, zero), (1e-3, 1e-5, 1000, x_warm), (1e-5, 1e-5, 1, zero), (1e-5, 1e-5, 2, zero),
                (1e-5, 1e-5, 3, x_warm), (1e-5, 1e-5, 7, zero)]
    return Amat, y, settings


@pytest.mark.parametrize('method', ['CG', 'CG-adaptive'])
@pytest.mark.parametrize('d', [2, 3])
@pytest.mark.parametrize('name', sorted(VEL_BCS))
def test_cg_iterates_equal_the_reference_solver(name, d, method, golden):
    """Same matrix, same right-hand side: the oracle's loop and the reference's `_linalg.cg` give the SAME iterates - bitwise-equal
    solutions and iteration counts - for full solves, truncated solves (max_iter 1, 2, 3, 7), warm starts and the plume's loose
    tolerance.  CG-adaptive: equal iteration counts and solutions to 2e-5 of scale, not bitwise - the reference forms the new
    direction as r - ((r.Ad) * d) / (d.Ad), element by element (_linalg.py:122), the oracle (and the CUDA kernel, which would otherwise
    divide per element) as r - ((r.Ad) / (d.Ad)) * d: one rounding apart per element and iteration."""
    Amat, y, settings = cg_inputs(name, d)
    solver = O.cg if method == 'CG' else O.cg_adaptive
    for j, (rtol, atol, max_iter, x0) in enumerate(settings):
        mine = solver(Amat, y, x0, rtol, atol, max_iter, None)
        ref_x = golden[f'cg/{method}/{name}/{d}/{j}/x']
        ref_iterations, ref_converged, ref_diverged = (int(v) for v in golden[f'cg/{method}/{name}/{d}/{j}/info'])
        if method == 'CG':
            assert ref_iterations == mine['iterations'], (rtol, max_iter)
            np.testing.assert_array_equal(ref_x, mine['x'].reshape(-1))
        else:
            assert abs(ref_iterations - mine['iterations']) <= 1, (rtol, max_iter)
            scale = max(float(np.abs(ref_x).max()), 1e-3)
            np.testing.assert_allclose(mine['x'].reshape(-1), ref_x, rtol=0, atol=2e-5 * scale + (0 if max_iter < 1000 else 20 * rtol * scale))
        assert bool(ref_converged) == bool(mine['converged']) and bool(ref_diverged) == bool(mine['diverged'])
