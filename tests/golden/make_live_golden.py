"""
Generates tests/golden/phiml_live.npz, the reference side of tests/test_oracle_live_phiml.py and tests/test_vector_boundaries.py.
Needs the reference's tensor library (PhiML 1.7.2) importable:

    PYTHONPATH=<PhiML source tree> python tests/golden/make_live_golden.py

The inputs come from the input functions of the two test modules (seeded), the outputs from phiml itself (NumPy backend).
"""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]
from phiml import math  # noqa: E402
from phiml.backend import NUMPY  # noqa: E402
from phiml.math import extrapolation as E, spatial, instance, channel, dual  # noqa: E402

import test_oracle_live_phiml as L  # noqa: E402
import test_vector_boundaries as V  # noqa: E402
from oracle import oracle_np as O  # noqa: E402
from phiflow_b200.phi_cuda import _adapter as A  # noqa: E402

AX = 'xyz'


def to_ext(bc):
    """oracle boundary spec -> phiml Extrapolation"""
    def side(s):
        return E.PERIODIC if s == 'periodic' else E.ZERO_GRADIENT if s == 'zg' else E.ConstantExtrapolation(float(s))
    if all(ax == bc[0] and ax[0] == ax[1] for ax in bc):
        return side(bc[0][0])
    return E.combine_sides(**{AX[i]: (side(lo), side(hi)) for i, (lo, hi) in enumerate(bc)})


def tensor_of(a):
    return math.tensor(a, spatial(**{AX[i]: n for i, n in enumerate(a.shape)}))


def scalar_cases(out):
    for name, make in L.SCALAR_BCS.items():
        for d in (2, 3):
            ext = to_ext(make(d))
            names = tuple(AX[:d])
            for i, a in enumerate(L.pad_laplace_inputs(name, d)):
                out[f'pad/{name}/{d}/{i}'] = math.pad(tensor_of(a), {names[k]: w for k, w in enumerate(L.PAD_WIDTHS[:d])}, ext).numpy(names)
                out[f'laplace/{name}/{d}/{i}'] = math.laplace(tensor_of(a), dx=math.vec(**dict(zip(names, L.DX[d]))), padding=ext).numpy(names)
            g, pts = L.grid_sample_inputs(name, d)
            coords = math.tensor(pts, instance(points=L.NPTS) & channel(vector=','.join(names)))
            out[f'grid_sample/{name}/{d}'] = math.grid_sample(tensor_of(g), coords, ext).numpy('points')
            close = math.closest_grid_values(tensor_of(g), coords, ext)
            out[f'closest/{name}/{d}'] = close.numpy(('points',) + tuple(f'closest_{n}' for n in names))


def cg_cases(out):
    for method in ('CG', 'CG-adaptive'):
        for name in L.VEL_BCS:
            for d in (2, 3):
                Amat, y, settings = L.cg_inputs(name, d)
                n = y.size
                for j, (rtol, atol, max_iter, x0) in enumerate(settings):
                    ref = NUMPY.linear_solve(method, Amat, y.reshape(1, n), x0.reshape(1, n).copy(), np.array([rtol], np.float32),
                                             np.array([atol], np.float32), np.array([[max_iter]]), None, None)
                    out[f'cg/{method}/{name}/{d}/{j}/x'] = np.asarray(ref.x)[0]
                    out[f'cg/{method}/{name}/{d}/{j}/info'] = np.array([int(np.asarray(ref.iterations)[0]), bool(np.asarray(ref.converged)[0]),
                                                                         bool(np.asarray(ref.diverged)[0])], np.int32)


def vector_boundaries(dims):
    lid = E.ConstantExtrapolation(math.vec(**{d: (1.0 if d == 'x' else 0.0) for d in dims}))
    inflow = E.ConstantExtrapolation(math.vec(**{d: v for d, v in zip(dims, (0.5, -0.25, 0.125))}))
    walls = {d: E.ZERO for d in dims}
    return {
        'cavity': E.combine_sides(**{**walls, dims[1]: (E.ZERO, lid)}),
        'inflow': E.combine_sides(**{**walls, dims[0]: (inflow, E.ZERO_GRADIENT)}),
        'zero': E.ZERO, 'periodic': E.PERIODIC, 'open': E.ZERO_GRADIENT,
        'mixed': E.combine_sides(**{**{d: E.BOUNDARY for d in dims}, dims[1]: (E.ZERO, E.BOUNDARY)}),
    }


def vector_cases(out):
    for dims, res, dx in V.CASES:
        nd = len(dims)
        for name, ext in vector_boundaries(dims).items():
            vspec = V.VSPECS[nd][name]
            assert A.to_vspec(ext, dims) == vspec, (name, dims)
            if name in ('cavity', 'inflow'):
                arrays = V.staggered_arrays(res, vspec)
                stack = math.stack([tensor_of(a) for a in arrays], channel(vector=dims))
                padded = math.pad(stack, {d: (1, 2) for d in dims}, ext)
                div = 0
                for c, d in enumerate(dims):
                    out[f'vb/pad/{name}/{nd}/{c}'] = padded[{'vector': d}].numpy(dims)
                    lo, hi = ext.valid_outer_faces(d)
                    baked = math.pad(stack, {d: (0 if lo else 1, 0 if hi else 1)}, ext)[{'vector': d}]
                    div = div + (baked[{d: slice(1, None)}] - baked[{d: slice(None, -1)}]) / dx[c]
                out[f'vb/div/{name}/{nd}'] = div.numpy(dims)
            arrays = V.staggered_arrays(res, vspec, seed=1)
            stack = math.stack([tensor_of(a) for a in arrays], dual(vector=dims))
            lap = math.map_d2c(math.laplace)(stack, dx=math.vec(**dict(zip(dims, dx))), padding=ext, dims=spatial)
            vdim = 'vector' if 'vector' in lap.shape else '~vector'
            for c, d in enumerate(dims):
                out[f'vb/lap/{name}/{nd}/{c}'] = lap[{vdim: d}].numpy(dims)


if __name__ == '__main__':
    out = {}
    scalar_cases(out)
    cg_cases(out)
    vector_cases(out)
    path = os.path.join(HERE, 'phiml_live.npz')
    np.savez_compressed(path, **out)
    print(f'{path}: {len(out)} arrays, {os.path.getsize(path)} bytes')
