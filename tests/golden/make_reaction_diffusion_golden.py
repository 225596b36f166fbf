"""
Generates tests/golden/phiml_reaction_diffusion.npz  --  run ONLY where the reference's PhiML is reachable:

    python tests/golden/make_reaction_diffusion_golden.py

The Reaction_Diffusion notebook's Gray-Scott step (examples/grids/Reaction_Diffusion.ipynb) with the vendored PhiML 1.7.2, float32:

    uvv = u * v**2
    su = du * laplace(u) - uvv + f * (1 - u)
    sv = dv * laplace(v) + uvv - (f + k) * v
    return u + dt * su, v + dt * sv

`phi` cannot be imported (it needs a newer phiml), so field.laplace is restated as what it calls for order 2:
math.laplace(values, dx, padding=extrapolation) (phi/field/_field_math.py:128); the rest is the notebook function verbatim on phiml
tensors.  Cases: 2-D ZERO / PERIODIC / ZERO_GRADIENT, a per-side mix, a 3-D mix, anisotropic dx, ragged sizes, batch 3, the
parameter sets maze, coral and dots, after 1 and 20 substeps each.  `ext/<kind>/u|v` records the extrapolation of u' and v' after
one step, evaluated by PhiML's own extrapolation arithmetic with the rules of field arithmetic (phi/field/_field.py:788-813: field
(-) field combines the extrapolations, field (-) number keeps the field's own; laplace: ext.spatial_gradient().spatial_gradient(),
_field_math.py:119).
"""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports phiml from /root/reference/PhiML)
from make_golden import math  # noqa: E402
from phiml.math import batch, spatial, tensor  # noqa: E402
from phiml.math import extrapolation as E  # noqa: E402

NAMES = 'xyz'
PARAMS = {'maze': dict(du=0.19, dv=0.05, f=0.06, k=0.062), 'coral': dict(du=0.16, dv=0.08, f=0.06, k=0.062),
          'dots': dict(du=0.19, dv=0.03, f=0.04, k=0.061)}
DT = 0.5
P, Z = 'periodic', 'zg'
# name: (resolution, boundary spec (x, y[, z]) of (lower, upper), dx, batch, parameter set)
CASES = {
    'zero': ((24, 16), ((0.0, 0.0), (0.0, 0.0)), (1.0, 1.0), 1, 'maze'),
    'periodic': ((24, 16), ((P, P), (P, P)), (1.0, 1.0), 1, 'coral'),
    'zg': ((24, 16), ((Z, Z), (Z, Z)), (1.0, 1.0), 1, 'dots'),
    'mixed': ((20, 12), ((0.0, Z), (P, P)), (1.0, 1.0), 1, 'maze'),
    'mixed3': ((12, 10, 8), ((P, P), (Z, 0.0), (0.0, Z)), (1.0, 1.0, 1.0), 1, 'coral'),
    'aniso': ((16, 12), ((Z, 0.0), (P, P)), (0.8, 1.5), 1, 'dots'),
    'ragged': ((37, 23), ((0.0, Z), (Z, 0.0)), (1.0, 1.0), 1, 'maze'),
    'batch': ((20, 16), ((0.0, 0.0), (0.0, 0.0)), (1.0, 1.0), 3, 'dots'),
}


def initial(res, nb, rng):
    """Seeded uniform noise: u in [0.3, 1), v in [0, 0.4) - every cell's reaction terms and both laplacians non-trivial."""
    u = rng.uniform(0.3, 1.0, (nb,) + res).astype(np.float32)
    v = rng.uniform(0.0, 0.4, (nb,) + res).astype(np.float32)
    return u, v


def phiml_tensor(a, nb):
    names = ','.join(NAMES[:a.ndim - 1])
    return tensor(a, batch('b'), spatial(names)) if nb else tensor(a[0], spatial(names))


def reaction_diffusion(u, v, du, dv, f, k, dt, ext, dx):
    laplace = lambda x: math.laplace(x, dx=list(dx), padding=ext)        # field.laplace order 2 (_field_math.py:128)
    uvv = u * v**2
    su = du * laplace(u) - uvv + f * (1 - u)
    sv = dv * laplace(v) + uvv - (f + k) * v
    return u + dt * su, v + dt * sv


def step_extrapolation(e):
    """The extrapolations of (u', v') for u and v with extrapolation e, by the rules of field arithmetic."""
    lap = e.spatial_gradient().spatial_gradient()
    uvv = e * e                                    # u * (v**2): v**2 keeps e (number), then field * field
    su = (lap - uvv) + e                           # du * lap keeps lap; f * (1 - u) keeps e
    sv = (lap + uvv) - e                           # (f + k) * v keeps e
    return e + su, e + sv                          # dt * s keeps s


def main():
    rng = np.random.default_rng(20261017)
    out = {}
    for name, (res, spec, dx, nb, pset) in CASES.items():
        u0, v0 = initial(res, nb, rng)
        out[f'{name}/u0'], out[f'{name}/v0'] = u0, v0
        out[f'{name}/bc'] = np.array([[np.nan if s == P else (np.inf if s == Z else s) for s in ax] for ax in spec], np.float64)
        out[f'{name}/dx'] = np.array(dx, np.float64)
        out[f'{name}/params'] = np.array(list(PARAMS[pset].values()) + [DT], np.float64)
        ext = G.ext_from_spec(spec)
        u, v = phiml_tensor(u0, nb > 1), phiml_tensor(v0, nb > 1)
        order = ','.join((['b'] if nb > 1 else []) + list(NAMES[:len(res)]))
        for s in range(1, 21):
            u, v = reaction_diffusion(u, v, dt=DT, ext=ext, dx=dx, **PARAMS[pset])
            if s in (1, 20):
                ua, va = u.numpy(order), v.numpy(order)
                assert ua.dtype == np.float32 and va.dtype == np.float32
                out[f'{name}/s{s}/u'] = ua if nb > 1 else ua[None]
                out[f'{name}/s{s}/v'] = va if nb > 1 else va[None]
    for kind, e in {'zero': E.ZERO, 'zg': E.ZERO_GRADIENT, 'periodic': E.PERIODIC, 'c0.3': E.ConstantExtrapolation(0.3)}.items():
        eu, ev = step_extrapolation(e)
        out[f'ext/{kind}/u'], out[f'ext/{kind}/v'] = np.array(repr(eu)), np.array(repr(ev))
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'phiml_reaction_diffusion.npz'), **out)
    for kind in ('zero', 'zg', 'periodic', 'c0.3'):
        print(kind, out[f'ext/{kind}/u'], out[f'ext/{kind}/v'])


if __name__ == '__main__':
    main()
