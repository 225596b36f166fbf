"""
Generates tests/golden/phiml_waves.npz  --  run ONLY where the reference's PhiML is reachable:

    python tests/golden/make_waves_golden.py

The Waves notebook's step (examples/grids/Waves.ipynb) with the vendored PhiML 1.7.2, float32:

    sphere = Sphere(center=h_c.bounds.center + math.rotate_vector(vec(x=0, y=-12.8/3), time), radius=1.)
    h_c, h_p = [field.where(sphere, mag * math.sin(t), f) for f in (h_c, h_p)]        # mag = .5, t = -PI/2
    h_n = 2.0 * h_c - h_p + dt * dt * (k_speed * h_c.laplace() - k_damp * (h_c - h_p))
    return h_n, h_c, time + dt

`phi` cannot be imported (it needs a newer phiml), so its glue is restated on phiml tensors from the cited lines: the cell centres
lower + linspace(0.5/n, 1 - 0.5/n, n) * size (UniformGrid.center, phi/geom/_grid.py:60-63, Box.local_to_global, _box.py:154-158),
Box.center = (lower + upper) / 2, field.where with a geometry = math.where(Sphere.lies_inside(centres), value, values)
(_field_math.py:997-1015, _resample.py:192-210, _sphere.py:103-105: sum over 'vector' of (p - c) ** 2 <= radius ** 2), and
Field.laplace = math.laplace(values, dx, padding=extrapolation) (_field_math.py:128).  rotate_vector, sin, where, laplace and the
arithmetic are PhiML's own.  Cases: one substep from seeded noise for ZERO_GRADIENT, PERIODIC, ZERO and non-zero constants mixed per
side, anisotropic dx, ragged sizes, batch 2 and 3-D, with no disc, a disc over a wall and k_damp != 0; the notebook's first two
frames (32 substeps at 128 x 128) with each substep's mask; the 4800 disc centres of the notebook's 300 frames x 16 substeps.
`ext/<kind>` records the extrapolation of h_n by PhiML's extrapolation arithmetic: ZERO, ZERO_GRADIENT and PERIODIC map to
themselves, a constant c to 0 (2.0 * h_c keeps c, so 2.0 * h_c - h_p has c - c = 0).
"""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports phiml from /root/reference/PhiML)
from make_golden import math  # noqa: E402
from phiml.math import batch, channel, spatial, tensor, vec, wrap  # noqa: E402
from phiml.math import extrapolation as E  # noqa: E402

NAMES = 'xyz'
P, Z = 'periodic', 'zg'
MAG, T = .5, -math.PI * 0.5
NB_DT = 1 / 60. / 16
# name: (resolution, upper corner of the bounds (lower = 0), boundary spec, batch, dt, k_speed, k_damp, disc centre or None, radius)
CASES = {
    'zg': ((24, 16), (24., 16.), ((Z, Z), (Z, Z)), 1, 0.2, 1.0, 0.0, (11.3, 7.9), 2.5),
    'periodic': ((24, 16), (24., 16.), ((P, P), (P, P)), 1, 0.2, 1.0, 0.3, (0.6, 8.2), 3.0),
    'zero': ((20, 12), (20., 12.), ((0.0, 0.0), (0.0, 0.0)), 1, 0.2, 0.7, 0.0, None, 1.0),
    'const': ((20, 12), (20., 12.), ((0.3, Z), (P, P)), 1, 0.2, 1.0, 0.0, (19.2, 5.5), 2.2),
    'const2': ((20, 12), (20., 12.), ((-0.7, 0.25), (Z, 0.0)), 1, 0.25, 1.0, 0.1, (4.1, 0.3), 2.6),
    'aniso': ((16, 12), (12.8, 18.), ((Z, 0.0), (P, P)), 1, 0.2, 1.0, 0.0, (6.3, 9.1), 1.3),
    'ragged': ((37, 23), (37., 23.), ((0.0, Z), (Z, 0.5)), 1, 0.2, 1.0, 0.0, (18.5, 11.5), 4.0),
    'batch': ((20, 16), (20., 16.), ((Z, Z), (P, P)), 2, 0.2, 1.0, 0.05, (10.0, 8.0), 3.1),
    'mixed3': ((12, 10, 8), (12., 10., 8.), ((P, P), (Z, 0.2), (0.0, Z)), 1, 0.15, 1.0, 0.0, (5.5, 4.2, 3.9), 2.4),
    'aniso3': ((10, 9, 7), (5., 9., 14.), ((Z, Z), (P, P), (Z, -0.4)), 1, 0.1, 1.0, 0.2, (2.4, 0.2, 7.1), 1.9),
}


def cell_centres(res, upper):
    """Per-axis float32 cell centres: lower + linspace(0.5/n, 1 - 0.5/n, n) * size with lower = 0."""
    return [(math.linspace(0.5 / n, 1 - 0.5 / n, spatial(**{NAMES[a]: n})) * wrap(np.float32(u)) + wrap(np.float32(0.))).numpy()
            for a, (n, u) in enumerate(zip(res, upper))]


def points(axes):
    """Cell centres as a phiml tensor with a 'vector' channel (meshgrid of the per-axis centres)."""
    grids = np.meshgrid(*axes, indexing='ij')
    names = ','.join(NAMES[:len(axes)])
    return math.stack([tensor(g.astype(np.float32), spatial(names)) for g in grids], channel(vector=names))


def disc_mask(pts, centre, radius):
    return math.sum((pts - centre) ** 2, dim='vector') <= radius ** 2                # Sphere.lies_inside


def step(h_c, h_p, pts, centre, radius, dt, k_speed, k_damp, ext, dx):
    laplace = lambda x: math.laplace(x, dx=list(dx), padding=ext)
    mask = None
    if centre is not None:
        mask = disc_mask(pts, centre, radius)
        h_c, h_p = [math.where(mask, MAG * math.sin(T), f) for f in (h_c, h_p)]
    h_n = 2.0 * h_c - h_p + dt * dt * (k_speed * laplace(h_c) - k_damp * (h_c - h_p))
    return h_n, h_c, mask


def phiml_tensor(a, nb):
    names = ','.join(NAMES[:a.ndim - 1])
    return tensor(a, batch('b'), spatial(names)) if nb else tensor(a[0], spatial(names))


def notebook_centre(time, upper=12.8):
    lower, upper = (wrap(np.full(2, v, np.float32), channel(vector='x,y')) for v in (0., upper))
    centre = (lower + upper) * 0.5                                          # Box.center of Box(x=12.8, y=12.8)
    return centre + math.rotate_vector(vec(x=0, y=-12.8 / 3), time)


def step_extrapolation(e):
    """The extrapolation of h_n for h_c and h_p with extrapolation e, by the rules of field arithmetic (field (-) number keeps the
    field's extrapolation, field (-) field combines them, phi/field/_field.py:787-811; laplace: e.spatial_gradient().spatial_gradient())."""
    lap = e.spatial_gradient().spatial_gradient()
    return (e - e) + (lap - (e - e))           # 2.0 * h_c keeps e; k_speed * lap keeps lap; k_damp * (h_c - h_p) and dt * dt * (..) keep theirs


def main():
    rng = np.random.default_rng(20261018)
    out = {}
    for name, (res, upper, spec, nb, dt, ks, kd, centre, radius) in CASES.items():
        hc0 = rng.uniform(-1, 1, (nb,) + res).astype(np.float32)
        hp0 = rng.uniform(-1, 1, (nb,) + res).astype(np.float32)
        dx = tuple(float(u / n) for u, n in zip(upper, res))
        axes = cell_centres(res, upper)
        out[f'{name}/hc0'], out[f'{name}/hp0'] = hc0, hp0
        out[f'{name}/bc'] = np.array([[np.nan if s == P else (np.inf if s == Z else s) for s in ax] for ax in spec], np.float64)
        out[f'{name}/upper'] = np.array(upper, np.float64)
        out[f'{name}/params'] = np.array([dt, ks, kd, radius], np.float64)
        out[f'{name}/centres'] = np.concatenate(axes).astype(np.float32)
        names = ','.join(NAMES[:len(res)])
        c = None
        if centre is not None:
            c = wrap(np.array(centre, np.float32), channel(vector=names))
            out[f'{name}/disc'] = c.numpy('vector')
        hn, hc, mask = step(phiml_tensor(hc0, nb > 1), phiml_tensor(hp0, nb > 1), points(axes), c, radius, dt, ks, kd,
                            G.ext_from_spec(spec), dx)
        order = ','.join((['b'] if nb > 1 else []) + list(NAMES[:len(res)]))
        for key, t in (('hn', hn), ('hc', hc)):
            a = t.numpy(order)
            assert a.dtype == np.float32
            out[f'{name}/{key}'] = a if nb > 1 else a[None]
        if mask is not None:
            out[f'{name}/mask'] = mask.numpy(names)
    # the notebook: 128 x 128 in Box(x=12.8, y=12.8), ZERO_GRADIENT, h0 = 0, 16 substeps per frame
    axes = cell_centres((128, 128), (12.8, 12.8))
    pts = points(axes)
    ext = G.ext_from_spec(((Z, Z), (Z, Z)))
    h_c = h_p = tensor(np.zeros((128, 128), np.float32), spatial('x,y'))
    time, masks, centres = 0, [], []
    for s in range(300 * 16):
        centre = notebook_centre(time)
        centres.append(centre.numpy('vector'))
        if s < 32:
            h_c, h_p, mask = step(h_c, h_p, pts, centre, 1., NB_DT, 1.0, 0.0, ext, (0.1, 0.1))
            masks.append(mask.numpy('x,y'))
            if s in (15, 31):
                out[f'notebook/f{(s + 1) // 16}/hn'], out[f'notebook/f{(s + 1) // 16}/hc'] = h_c.numpy('x,y'), h_p.numpy('x,y')
        time = time + NB_DT
    out['notebook/centres'] = np.stack(centres).astype(np.float32)
    out['notebook/masks'] = np.stack(masks)
    out['notebook/axis_centres'] = np.concatenate(axes).astype(np.float32)
    out['notebook/value'] = np.float32(MAG * math.sin(T))
    for kind, e in {'zg': E.ZERO_GRADIENT, 'periodic': E.PERIODIC, 'zero': E.ZERO, 'c0.3': E.ConstantExtrapolation(0.3),
                    'c-0.7': E.ConstantExtrapolation(-0.7)}.items():
        out[f'ext/{kind}'] = np.array(repr(step_extrapolation(e)))
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'phiml_waves.npz'), **out)
    print({k: str(out[k]) for k in out if k.startswith('ext/')}, out['notebook/value'], out['notebook/masks'].sum((1, 2))[:4])


if __name__ == '__main__':
    main()
