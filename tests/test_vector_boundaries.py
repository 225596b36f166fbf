"""
Vector-valued constant boundaries (`{'y+': vec(x=1, y=0)}`: the lid of Lid_Driven_Cavity.ipynb, inflow profiles) and staggered diffusion
(`diffuse.explicit(v, ...)` of Lid_Driven_Cavity / Variable_Boundaries), oracle side, pinned against outputs of PhiML 1.7.2 recorded into
tests/golden/phiml_live.npz by tests/golden/make_live_golden.py:

  * `math.pad` of a component stack with per-component constants      == oracle `pad` with the component's spec
  * pad along the own axis + forward differences (`field.divergence`)  == oracle `divergence_staggered`
  * `math.laplace` of the non-uniform staggered stack (what `field.laplace` / `diffuse.explicit` run, phi/field/_field_math.py:118-145)
                                                                      == per-component oracle `laplace` -> `diffuse_explicit`
VSPECS are the oracle specs that `phiflow_b200.phi_cuda._adapter.to_vspec` derives from the phiml extrapolations of the cases (the
generator checks that).  The CUDA side of the same cases is tests/test_gpu_vector_boundaries.py.
"""
import os

import numpy as np
import pytest

from oracle import oracle_np as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'phiml_live.npz')

# boundaries per case: cavity = walls with a lid moving along x at the upper y side; inflow = a constant vector at the lower x side,
# open at the upper; mixed = open except a wall at the lower y side
VSPECS = {
    2: {'cavity': [((0.0, 0.0), (0.0, 1.0)), ((0.0, 0.0), (0.0, 0.0))],
        'inflow': [((0.5, 'zg'), (0.0, 0.0)), ((-0.25, 'zg'), (0.0, 0.0))],
        'zero': ((0.0, 0.0), (0.0, 0.0)), 'periodic': (('periodic', 'periodic'), ('periodic', 'periodic')),
        'open': (('zg', 'zg'), ('zg', 'zg')), 'mixed': (('zg', 'zg'), (0.0, 'zg'))},
    3: {'cavity': [((0.0, 0.0), (0.0, 1.0), (0.0, 0.0)), ((0.0, 0.0), (0.0, 0.0), (0.0, 0.0)), ((0.0, 0.0), (0.0, 0.0), (0.0, 0.0))],
        'inflow': [((0.5, 'zg'), (0.0, 0.0), (0.0, 0.0)), ((-0.25, 'zg'), (0.0, 0.0), (0.0, 0.0)), ((0.125, 'zg'), (0.0, 0.0), (0.0, 0.0))],
        'zero': ((0.0, 0.0),) * 3, 'periodic': (('periodic', 'periodic'),) * 3, 'open': (('zg', 'zg'),) * 3,
        'mixed': (('zg', 'zg'), (0.0, 'zg'), ('zg', 'zg'))},
}
CASES = [(('x', 'y'), (10, 8), (1.0, 0.5)), (('x', 'y', 'z'), (6, 5, 7), (0.5, 1.0, 2.0))]


@pytest.fixture(scope='module')
def golden():
    with np.load(GOLDEN) as f:
        return dict(f)


def staggered_arrays(res, vspec, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal(s).astype(np.float32) for s in O.staggered_shapes(res, vspec)]


@pytest.mark.parametrize('dims,res,dx', CASES, ids=['2d', '3d'])
@pytest.mark.parametrize('name', ['cavity', 'inflow'])
def test_pad_and_divergence_with_vector_constants(dims, res, dx, name, golden):
    vspec = VSPECS[len(dims)][name]
    assert isinstance(vspec, list) and len(vspec) == len(dims)            # constants differ per component, kinds do not
    comp = O.component_bcs(vspec, len(dims))
    arrays = staggered_arrays(res, vspec)
    for c, d in enumerate(dims):
        got, want = golden[f'vb/pad/{name}/{len(dims)}/{c}'], O.pad(arrays[c], [(1, 2)] * len(dims), comp[c])
        # ghosts that are outside along ONE axis only: where two different constants meet in a corner the reference pads "all sides
        # of extrapolation A, then all sides of B", A / B ordered by pad_rank and, among constants, by SET order
        # (PhiML/phiml/math/extrapolation.py:1292-1301) - the corner value is not defined by the reference itself
        outside = sum(((np.arange(n) < 1) | (np.arange(n) >= n - 2)).reshape([-1 if a == ax else 1 for a in range(len(dims))])
                      for ax, n in enumerate(got.shape))
        np.testing.assert_array_equal(got[outside <= 1], want[outside <= 1])
    np.testing.assert_array_equal(golden[f'vb/div/{name}/{len(dims)}'], O.divergence_staggered(arrays, dx, comp))


@pytest.mark.parametrize('dims,res,dx', CASES, ids=['2d', '3d'])
@pytest.mark.parametrize('name', ['cavity', 'inflow', 'zero', 'periodic', 'open', 'mixed'])
def test_staggered_laplace_is_the_per_component_laplace(dims, res, dx, name, golden):
    vspec = VSPECS[len(dims)][name]
    comp = O.component_bcs(vspec, len(dims))
    arrays = staggered_arrays(res, vspec, seed=1)
    lap = [golden[f'vb/lap/{name}/{len(dims)}/{c}'] for c in range(len(dims))]
    for c in range(len(dims)):
        np.testing.assert_array_equal(lap[c], O.laplace(arrays[c], dx, comp[c]))
    # diffuse.explicit (phi/physics/diffuse.py:52-61): amount = diffusivity * (dt / substeps), u += amount * laplace(u)
    out = O.diffuse_explicit(arrays, vspec, dx, 0.1, 0.5, substeps=1)
    amount = np.float32(0.1 * (0.5 / 1))
    for c in range(len(dims)):
        np.testing.assert_array_equal(out[c], (arrays[c] + amount * lap[c]).astype(np.float32))


def test_oracle_projection_and_advection_accept_component_lists():
    """Lid-driven cavity on the oracle: the tangential lid velocity drives the flow through the advection ghosts only; the projection
    sees walls (normal components 0), so the divergence-free result keeps zero wall-normal flux."""
    dims, res, dx = ('x', 'y'), (12, 10), (1.0, 1.0)
    vspec = VSPECS[2]['cavity']
    assert O.staggered_shapes(res, vspec) == [(11, 10), (12, 9)] and not O.is_flexible(vspec)
    assert O.pressure_bc(vspec) == (('zg', 'zg'), ('zg', 'zg'))
    v = [np.zeros(s, np.float32) for s in O.staggered_shapes(res, vspec)]
    lower, upper = (0.0, 0.0), (12.0, 10.0)
    for _ in range(3):
        v = O.semi_lagrangian_staggered(v, vspec, v, vspec, res, lower, upper, 1.0)
        v = O.diffuse_explicit(v, vspec, dx, 0.1, 1.0)
        v, p, info = O.make_incompressible(v, vspec, res, dx, rtol=1e-5, atol=1e-5, use_matrix_offset=False)
    assert info['converged'] and float(np.abs(v[0]).max()) > 1e-3           # the lid has set the fluid in motion
    assert float(v[0][:, -1].mean()) > 0                                      # dragged along +x under the lid
    div = O.divergence_staggered(v, dx, O.component_bcs(vspec, 2))
    assert float(np.abs(div).max()) < 1e-4
