"""
Generates tests/golden/phiml_collocated.npz  --  run ONLY in the build container (reference mounted):

    python tests/golden/make_collocated_golden.py

The CenteredGrid-velocity ("collocated", wide stencil) variant of the pressure projection (SURVEY.md Appendix A,
phi/physics/fluid.py:154-155,197-202): central-difference gradient `math.spatial_gradient(difference='central')`
(_field_math.py:230-233 -> _nd.py:810-812), centred divergence via `shift(field, (-1, 1))` (_field_math.py:627-632) and the
operator traced from their composition.  The phi.field glue is restated on phiml tensors; shift / pad / tracing / CG are
executed by the vendored PhiML.  Fixtures for oracle.gradient_centered / divergence_centered / wide_poisson_matrix.
"""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402
from make_golden import math, Solve, channel, spatial  # noqa: E402

NAMES = G.NAMES


def grad_center(p, dx, pext):
    """field.spatial_gradient(p, at='center') (_field_math.py:230-233): list of components."""
    dims = p.shape.spatial.names
    g = math.spatial_gradient(p, math.wrap(dx, channel(vector=','.join(dims))), difference='central', padding=pext,
                              stack_dim=channel(vector=','.join(dims)))
    return [g.vector[d] for d in dims]


def div_center(comps, dx, vext):
    """field.divergence of a CenteredGrid (_field_math.py:627-632): sum_d (right_d - left_d) / (2 dx_d), ghosts from vext."""
    total = 0
    for i, (dim, comp) in enumerate(zip(comps[0].shape.spatial.names, comps)):
        left, right = math.shift(comp, (-1, 1), dims=dim, padding=vext, stack_dim=None)
        total = total + (right - left) / (2 * dx[i])
    return total


def vector_ext(spec):
    """Per-component constants: spec = one spec per component, the same kinds everywhere -> one Extrapolation whose constant
    sides hold a vector value (ConstantExtrapolation(vec(...)), as the Lid_Driven_Cavity notebook's {'y+': vec(x=1, y=0)})."""
    dims = NAMES[:len(spec)]
    sides = {}
    for ax in range(len(spec)):
        pair = []
        for side in range(2):
            kind = spec[0][ax][side]
            if isinstance(kind, str):
                pair.append(G.E.PERIODIC if kind == 'periodic' else G.E.ZERO_GRADIENT)
            else:
                pair.append(G.E.ConstantExtrapolation(math.vec(**{d: spec[c][ax][side] for c, d in enumerate(dims)})))
        sides[dims[ax]] = tuple(pair)
    return G.E.combine_sides(**sides)


def div_center_vector(comps, dx, vext):
    """field.divergence of a CenteredGrid with a vector-valued boundary: the stacked velocity is shifted with its own extrapolation,
    so component d sees its own constant (_field_math.py:627-632)."""
    dims = comps[0].shape.spatial.names
    v = math.stack(comps, channel(vector=','.join(dims)))
    total = 0
    for i, dim in enumerate(dims):
        left, right = math.shift(v, (-1, 1), dims=dim, padding=vext, stack_dim=None)
        total = total + (right.vector[dim] - left.vector[dim]) / (2 * dx[i])
    return total


def masked_laplace_wide(p, dx, pext, vext0):
    """fluid.masked_laplace(wide_stencil=True), no obstacles (fluid.py:197-202)."""
    return div_center(grad_center(p, dx, pext), dx, vext0)


def main():
    out = {}
    rng = np.random.default_rng(17)
    cases = [('zero', G.BC_SETS_2D['zero'], (8, 6), (0.5, 0.25)),
             ('open', G.BC_SETS_2D['open'], (8, 6), (0.5, 0.25)),
             ('periodic', G.BC_SETS_2D['periodic'], (8, 6), (1.0, 1.0)),
             ('mixed', G.BC_SETS_2D['mixed'], (8, 6), (1.0, 0.5)),
             ('one', G.BC_SETS_2D['one'], (7, 5), (1.0, 1.0)),
             ('mixed3', G.BC_SETS_3D['mixed'], (6, 5, 4), (1.0, 0.5, 1.0)),
             # per-component constants (a list of one spec per component): a lid and an inflow profile
             ('lid', [((0.0, 0.0), (0.0, 1.0)), ((0.0, 0.0), (0.0, 0.0))], (8, 6), (0.5, 0.25)),
             ('inflow3', [((0.5, 'zg'), ('periodic', 'periodic'), (0.0, 0.0)), ((-0.25, 'zg'), ('periodic', 'periodic'), (0.0, 0.0)),
                          ((0.125, 'zg'), ('periodic', 'periodic'), (0.0, 0.0))], (6, 5, 4), (1.0, 0.5, 1.0))]
    for name, spec, res, dx in cases:
        d = len(res)
        vector = isinstance(spec, list)
        kinds = spec[0] if vector else spec
        vext = vector_ext(spec) if vector else G.ext_from_spec(spec)
        vext0 = G.ext_from_spec(G.remove_const(kinds))
        pext = G.ext_from_spec(G.pressure_ext(kinds))
        p = rng.standard_normal(res).astype(np.float32)
        comps = [rng.standard_normal(res).astype(np.float32) for _ in range(d)]
        out[f'{name}/bc'] = np.stack([G.spec_to_arr(s) for s in spec]) if vector else G.spec_to_arr(spec)
        out[f'{name}/dx'] = np.array(dx)
        out[f'{name}/p'] = p
        for c in range(d):
            out[f'{name}/v{c}'] = comps[c]
        g = grad_center(G.to_tensor(p), dx, pext)
        for c in range(d):
            out[f'{name}/grad{c}'] = G.npy(g[c], d)
        div = (div_center_vector if vector else div_center)([G.to_tensor(c) for c in comps], dx, vext)
        out[f'{name}/div'] = G.npy(div, d)
        lin = math.jit_compile_linear(masked_laplace_wide, auxiliary_args='dx,pext,vext0')
        out[f'{name}/lap'] = G.npy(lin(G.to_tensor(p), dx=dx, pext=pext, vext0=vext0), d)
        mat = lin.sparse_matrix(G.to_tensor(p), dx=dx, pext=pext, vext0=vext0)
        n_tot = int(np.prod(res))
        order_ = ','.join(NAMES[:d]) + ',' + ','.join('~' + n for n in NAMES[:d])
        out[f'{name}/matrix'] = math.dense(mat).numpy(order_).reshape(n_tot, n_tot)
    np.savez_compressed(os.path.join(G.OUT, 'phiml_collocated.npz'), **out)
    print(f"wrote {len(out)} arrays")


if __name__ == '__main__':
    main()
