"""
Generates tests/golden/phiml_points.npz  --  run ONLY where the reference's PhiML is reachable:

    python tests/golden/make_points_golden.py

advect.points(points, velocity, dt, integrator) for a StaggeredGrid velocity with the vendored PhiML 1.7.2, float32
(phi/physics/advect.py:20-35, 136-153).  `phi` cannot be imported (it needs a newer phiml), so its glue is restated on phiml tensors
from the cited lines:
  * the component grids: UniformGrid(res, bounds).stagger(dim, *extrapolation.valid_outer_faces(dim)) (phi/geom/_grid.py:204-209):
    unit = size / resolution along dim only, lower' = lower + unit * (-0.5 | 0.5), upper' = upper + unit * (0.5 | -0.5);
  * sample_staggered_grid (phi/field/_resample.py:276-284) -> sample_grid_at_centers (:257-258) for every component:
    grid_sample(values_c, global_to_local(p) * res' - 0.5, extrapolation[{'vector': c}]), with Box.global_to_local = (p - lower') /
    size' (phi/geom/_box.py:134-152);
  * euler: p + v0 * dt;  rk4: the four samples and p + dt * ((1 / 6.) * (v0 + 2 * (v_half + v_half2) + v_full)).
math.grid_sample, the extrapolations (valid_outer_faces, indexing by component, combine_sides with a vector constant) and all the
arithmetic are PhiML's own.

Cases: 2-D and 3-D; ZERO, ZERO_GRADIENT, PERIODIC and per-side mixes; the Lid_Driven_Cavity vector constant {'y+': vec(x=1, y=0)};
a non-zero lower corner, anisotropic cells and ragged sizes; batch 2 with per-entry and broadcast points; points on faces, on cell
centres, a few cells outside, ~10^3 cells outside, NaN and +-inf; negative dt; 1 and 4 steps of both integrators; the Streamlines
notebook's case (256 x 256, Box(x=10, y=10), ZERO boundary, the point (5, 5) and the 64 centres of an 8 x 8 grid, 50 RK4 steps of 0.1)
on a seeded divergence-free velocity (the discrete curl of a stream function that vanishes on the walls).
`int32_cast` records PhiML's float -> int32 conversion (to_int32 of floor) of NaN, +-inf and +-3e9 on this machine.
"""
import json
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402,F401  (imports phiml from /root/reference/PhiML)
from make_golden import math  # noqa: E402
from phiml.math import batch, channel, instance, spatial, vec  # noqa: E402
from phiml.math import extrapolation as E  # noqa: E402

F = np.float32
NAMES = 'xyz'
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'phiml_points.npz')


def ext_of(spec, d):
    """PhiML extrapolation of a boundary spec {'x': kind, 'y-': kind, ...}; kind = 'zg', 'periodic', a number or a vec."""
    conv = lambda k: E.ZERO_GRADIENT if k == 'zg' else (E.PERIODIC if k == 'periodic' else k)
    sides = {}
    for a in NAMES[:d]:
        if a in spec:
            sides[a] = conv(spec[a])
        else:
            sides[a] = (conv(spec[a + '-']), conv(spec[a + '+']))
    return E.combine_sides(**sides)


def plain(side):
    """A PhiML side extrapolation of one component as the library's plain spec."""
    if side == E.ZERO_GRADIENT:
        return 'zg'
    if side == E.PERIODIC:
        return 'periodic'
    return float(side.value.numpy()) if hasattr(side, 'value') else float(side)


def side_of(ext, axis, upper):
    """The extrapolation of one side of a (component's) extrapolation."""
    if isinstance(ext, E._MixedExtrapolation):
        return ext.ext[axis] if axis in ext.ext else ext.ext[axis + ('+' if upper else '-')]
    return ext


def stagger(lower, upper, res, ext, c):
    """(lower', upper', res') of component c as phiml tensors / ints (UniformGrid.stagger)."""
    d = len(res)
    lo_st, hi_st = ext.valid_outer_faces(NAMES[c])
    lower_t = math.tensor(np.asarray(lower, F), channel(vector=','.join(NAMES[:d])))
    upper_t = math.tensor(np.asarray(upper, F), channel(vector=','.join(NAMES[:d])))
    mask = math.tensor(np.array([1 if a == c else 0 for a in range(d)]), channel(vector=','.join(NAMES[:d])))
    unit = (upper_t - lower_t) / math.tensor(np.asarray(res), channel(vector=','.join(NAMES[:d]))) * mask
    lo2 = lower_t + unit * (-0.5 if lo_st else 0.5)
    up2 = upper_t + unit * (0.5 if hi_st else -0.5)
    res2 = [r + (int(lo_st) + int(hi_st) - 1 if a == c else 0) for a, r in enumerate(res)]
    return lo2, up2, res2


def sampler(values, lower, upper, res, ext):
    d = len(res)
    comps = []
    for c in range(d):
        lo2, up2, res2 = stagger(lower, upper, res, ext, c)
        vt = math.tensor(values[c], batch('b'), spatial(**dict(zip(NAMES, res2))))
        comps.append((vt, lo2, up2, math.tensor(np.asarray(res2), channel(vector=','.join(NAMES[:d]))), ext[{'vector': NAMES[c]}]))

    def sample(p):
        out = []
        for vt, lo2, up2, r2, ec in comps:
            local = (p - lo2) / (up2 - lo2) * r2 - 0.5
            out.append(math.grid_sample(vt, local, ec))
        return math.stack(out, channel(vector=','.join(NAMES[:d])))
    return sample, comps


def euler(sample, p, dt):
    return p + sample(p) * dt


def rk4(sample, p, dt):
    v0 = sample(p)
    v_half = sample(p + 0.5 * dt * v0)
    v_half2 = sample(p + 0.5 * dt * v_half)
    v_full = sample(p + dt * v_half2)
    return p + dt * ((1 / 6.) * (v0 + 2 * (v_half + v_half2) + v_full))


def test_points(rng, lower, upper, res, n_random=40):
    """World points of every kind the fixture covers, (N, d) float32."""
    d = len(res)
    lo, up = np.asarray(lower, F), np.asarray(upper, F)
    dx = (up - lo) / np.asarray(res, F)
    pts = [lo + rng.random((n_random, d)).astype(F) * (up - lo)]
    idx = rng.integers(0, np.asarray(res) + 1, (12, d))
    pts.append(lo + idx.astype(F) * dx)                                         # on faces (and cell corners)
    pts.append(lo + (rng.integers(0, np.asarray(res), (12, d)) + F(0.5)) * dx)  # on cell centres
    pts.append(lo + (rng.random((12, d)) * (np.asarray(res) + 6) - 3).astype(F) * dx)   # up to 3 cells outside
    far = lo + (rng.random((8, d)) * 2 - 0.5).astype(F) * (up - lo) * F(1000) / np.asarray(res, F).max() * np.asarray(res, F)
    pts.append(far.astype(F))                                                   # ~10^3 cells outside
    special = np.tile(((lo + up) / 2).astype(F), (6, 1))
    special[0, 0] = np.nan
    special[1, d - 1] = np.inf
    special[2, 0] = -np.inf
    special[3, :] = np.nan
    special[4, 1] = F(3e9)
    special[5, 0] = F(-3e9)
    pts.append(special)
    return np.concatenate(pts).astype(F)


def velocity_values(rng, res, ext, batch_size):
    d = len(res)
    vals = []
    for c in range(d):
        lo_st, hi_st = ext.valid_outer_faces(NAMES[c])
        shape = tuple(r + (int(lo_st) + int(hi_st) - 1 if a == c else 0) for a, r in enumerate(res))
        vals.append(rng.standard_normal((batch_size,) + shape).astype(F))
    return vals


def divergence_free_2d(n, seed):
    """u_x = d psi / dy on the x faces, u_y = -d psi / dx on the y faces, psi on the cell corners, zero on the walls: the interior
    faces of a closed (ZERO) box, (n - 1, n) and (n, n - 1)."""
    rng = np.random.default_rng(seed)
    s = np.linspace(0, 1, n + 1)
    X, Y = np.meshgrid(s, s, indexing='ij')
    psi = np.zeros_like(X)
    for _ in range(6):
        kx, ky = rng.integers(1, 5, 2)
        psi += rng.standard_normal() * np.sin(np.pi * kx * X) * np.sin(np.pi * ky * Y)
    psi *= 0.5
    h = 10.0 / n
    ux = (psi[1:-1, 1:] - psi[1:-1, :-1]) / h
    uy = -(psi[1:, 1:-1] - psi[:-1, 1:-1]) / h
    return [ux[None].astype(F), uy[None].astype(F)]


CASES = {
    # name: (resolution, lower, upper, boundary, velocity batch, points batch)
    'zero_2d': ((12, 9), (-1.5, 0.25), (4.5, 3.0), {'x': 0, 'y': 0}, 1, 1),
    'zg_2d': ((11, 7), (0., 0.), (11., 3.5), {'x': 'zg', 'y': 'zg'}, 1, 1),
    'periodic_2d': ((10, 13), (2., -1.), (7., 5.5), {'x': 'periodic', 'y': 'periodic'}, 1, 1),
    'mixed_2d': ((9, 10), (0., 0.), (4.5, 10.), {'x-': 'zg', 'x+': 0.3, 'y': 'periodic'}, 1, 1),
    'mixed2_2d': ((8, 6), (-2., 1.), (2., 4.), {'x-': -0.7, 'x+': 'zg', 'y-': 0.25, 'y+': 'zg'}, 1, 1),
    'cavity_2d': ((12, 12), (0., 0.), (1., 1.), {'x': 0, 'y-': 0, 'y+': vec(x=1, y=0)}, 1, 1),
    'batch_2d': ((10, 8), (0., 0.), (5., 4.), {'x': 'zg', 'y': 0}, 2, 2),
    'broadcast_2d': ((10, 8), (0., 0.), (5., 4.), {'x': 'periodic', 'y': 'zg'}, 2, 1),
    'zero_3d': ((7, 5, 6), (-1., 0.5, 2.), (2.5, 3., 5.), {'x': 0, 'y': 0, 'z': 0}, 1, 1),
    'zg_3d': ((6, 7, 5), (0., 0., 0.), (6., 3.5, 10.), {'x': 'zg', 'y': 'zg', 'z': 'zg'}, 1, 1),
    'periodic_3d': ((6, 5, 7), (0., 0., 0.), (3., 5., 7.), {'x': 'periodic', 'y': 'periodic', 'z': 'periodic'}, 1, 1),
    'mixed_3d': ((7, 6, 5), (1., -2., 0.), (8., 1., 2.5), {'x': 'periodic', 'y-': 0.4, 'y+': 'zg', 'z-': 'zg', 'z+': -0.2}, 2, 1),
}
RUNS = [('euler', 1, 0.35), ('rk4', 1, 0.35), ('rk4', 4, 0.2), ('euler', 3, -0.3)]


def main():
    rng = np.random.default_rng(2024)
    out = {'meta': np.array(json.dumps({'phiml': __import__('phiml').__version__, 'numpy': np.__version__, 'cases': list(CASES),
                                        'runs': RUNS}))}
    special = np.array([np.nan, np.inf, -np.inf, 3e9, -3e9, 2.5, -2.5], F)
    out['int32_cast/in'] = special
    out['int32_cast/out'] = math.to_int32(math.floor(math.tensor(special, instance('i')))).numpy('i')
    for name, (res, lower, upper, bspec, vb, pb) in CASES.items():
        d = len(res)
        ext = ext_of(bspec, d)
        vals = velocity_values(rng, res, ext, vb)
        sample, comps = sampler(vals, lower, upper, res, ext)
        pts = np.stack([test_points(rng, lower, upper, res) for _ in range(pb)])
        p0 = math.tensor(pts, batch('b'), instance('points'), channel(vector=','.join(NAMES[:d]))) if pb > 1 else \
            math.tensor(pts[0], instance('points'), channel(vector=','.join(NAMES[:d])))
        out[f'{name}/points'] = pts
        out[f'{name}/spec'] = np.array(json.dumps([[[plain(side_of(ext[{'vector': NAMES[c]}], a, u)) for u in (False, True)]
                                                    for a in NAMES[:d]] for c in range(d)]))
        out[f'{name}/bounds'] = np.array([lower, upper], F)
        for c in range(d):
            out[f'{name}/v{c}'] = vals[c]
            vt, lo2, up2, r2, _ = comps[c]
            out[f'{name}/stagger{c}'] = np.stack([lo2.numpy('vector'), (up2 - lo2).numpy('vector'), r2.numpy('vector').astype(F)])
        for integ, steps, dt in RUNS:
            p = p0
            for _ in range(steps):
                p = (euler if integ == 'euler' else rk4)(sample, p, dt)
            out[f'{name}/{integ}_{steps}_{dt}'] = p.numpy(['b', 'points', 'vector'])
    # the Streamlines notebook: 256^2, Box(x=10, y=10), ZERO, (5, 5) and the 64 centres of an 8 x 8 grid, 50 RK4 steps of 0.1
    n = 256
    ext = E.ZERO
    vals = divergence_free_2d(n, 7)
    sample, _ = sampler(vals, (0., 0.), (10., 10.), (n, n), ext)
    c8 = np.linspace(F(0.5 / 8), F(1 - 0.5 / 8), 8, dtype=F) * F(10) + F(0)        # CenteredGrid(..., x=8, y=8) axis centres
    X, Y = np.meshgrid(c8, c8, indexing='ij')
    starts = np.concatenate([np.array([[5, 5]], F), np.stack([X.ravel(), Y.ravel()], -1)]).astype(F)
    p = math.tensor(starts, instance('points'), channel(vector='x,y'))
    trj = [starts]
    for _ in range(50):
        p = rk4(sample, p, .1)
        trj.append(p.numpy(['b', 'points', 'vector'])[0])
    out['notebook/v0'], out['notebook/v1'] = vals
    out['notebook/points'] = starts[None]
    out['notebook/trajectory'] = np.stack(trj)[:, None]
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays")


if __name__ == '__main__':
    main()
