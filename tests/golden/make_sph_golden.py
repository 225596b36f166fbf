"""
Generates tests/golden/phiml_sph.npz  --  run ONLY where the reference's PhiML is reachable:

    python tests/golden/make_sph_golden.py

The SPH notebook's substep apply_bounds(sph_step(v)) (examples/particles/SPH.ipynb) with the vendored PhiML 1.7.2, float32.  `phi`
cannot be imported (it needs a newer phiml), so its glue is restated on phiml tensors from the cited lines:
  * the constants: Sphere(volume=h ** d) keeps radius_from_volume(volume) and reports volume_from_radius(radius); desired_neighbors =
    expected_neighbors(volume, h, d), s = radius_from_volume(volume desired_neighbors) (phi/geom/_sphere.py:69-90,
    phi/physics/sph.py:71-98); m = 0.01 mean(volume), P = -(45 m) / (PI h ** 6), V = (45 0.025 m) / (PI h ** 6) (the notebook);
  * neighbor_graph (phi/physics/sph.py:23-68): deltas = pairwise_differences(x, max_distance=s, format='sparse', domain=(lower,
    upper)), distances = vec_length(deltas, eps=1e-5), the poly6 kernel of evaluate_kernel (:150-160).  In this snapshot Graph has
    only (nodes, edges, boundary), so neighbor_graph's Graph(..., deltas=, distances=) does not run; the step uses those two tensors
    as sph.py states them, connectivity = tensor_like(edges, 1) and unit_deltas = safe_div(deltas, distances)
    (phi/geom/_graph.py:34-46);
  * sph_step and apply_bounds as the notebook's cells, with Field arithmetic on the particle values and positions.
pairwise_differences, the sparse sums, safe_div, clip, where and all arithmetic are PhiML's own.  The pairs: see step().

Cases: 2-D and 3-D; a jittered lattice as the notebook builds it at a small size; particles leaving a small box in a substep on one
axis and on several; pairs at distance exactly s; a pair closer than sqrt(1e-5); an isolated particle; particles starting above the
upper corner (the min(., res - 1) clamp of the top cell); 1 and 5 substeps.  Per case: the inputs and constants, the first substep's
pairs in stored order and the pairs of PhiML's sparse search, rho and F, and x and v after all substeps.
"""
import json
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402,F401  (imports the reference's PhiML)
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle_sph as O  # noqa: E402  (the stored order of the pairs)
from make_golden import math  # noqa: E402
from phiml.math import PI, channel, dual, instance, rename_dims, wrap  # noqa: E402

F = np.float32
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'phiml_sph.npz')
H = 0.8


def constants(d, h=H):
    vfr = (lambda r: 4 / 3 * PI * r ** 3) if d == 3 else (lambda r: PI * r ** 2)
    rfv = (lambda v: (.75 / PI * v) ** (1 / 3)) if d == 3 else (lambda v: math.sqrt(v / PI))
    volume = vfr(rfv(wrap(h ** d)))
    s = rfv(volume * (vfr(h) / volume))
    m = 0.01 * math.mean(volume)
    P = -(45.0 * m) / (PI * h ** 6)
    V = (45.0 * 0.025 * m) / (PI * h ** 6)
    norm = (315 / 64 / PI if d == 3 else 4 / PI) / s ** (d + 6)
    return s, m, P, V, norm


def step(x, v, d, lower, upper, h=H):
    """One apply_bounds(sph_step(v)).  Returns x, v, (rows, cols) in stored order, rho, F, and (rows, cols) of PhiML's own sparse
    search, as NumPy arrays."""
    names = 'xyz'[:d]
    s, m, P, V, norm = constants(d, h)
    xt = math.tensor(x, instance('particles'), channel(vector=','.join(names)))
    vt = math.tensor(v, instance('particles'), channel(vector=','.join(names)))
    lo = math.tensor(np.asarray(lower, F), channel(vector=','.join(names)))
    up = math.tensor(np.asarray(upper, F), channel(vector=','.join(names)))
    gravity = math.vec(**dict(zip(names, (0, 0, -0.1) if d == 3 else (0, -0.1))))
    searched = math.pairwise_differences(xt, max_distance=s, format='sparse', domain=(lo, up))
    search = searched._indices.numpy([instance(searched._indices).name, 'sparse_idx'])
    # The hash-grid search of PhiML 1.7.2 drops every pair in the (-1, ..., -1) neighbour cell (find_neighbors_sparse gathers
    # neighbor_partitions at direction - 1 = -1 for direction 0, the last partition) and stores duplicates in its place.  The step
    # therefore runs on the pairs PhiML's dense search finds with the sparse search's test, sqrt(vec_squared(delta)) < s, stored in
    # the oracle's order (tests/oracle_sph.py), and deltas = pairwise_differences(x, format=that connectivity).
    r2 = math.vec_squared(math.pairwise_differences(xt, format='dense')).numpy(['particles', '~particles'])
    keep = np.sqrt(r2) < s.numpy()
    I, J = O.pairs(x, lower, upper, s.numpy())
    assert set(zip(I.tolist(), J.tolist())) == set(zip(*np.nonzero(keep))), "oracle pairs differ from PhiML's dense search"
    n = x.shape[0]
    idx = math.tensor(np.stack([I, J], -1).astype(np.int32), instance('pairs'), channel(idx='particles,~particles'))
    conn = math.sparse_tensor(idx, math.ones(instance(pairs=len(I))), instance(particles=n) & dual(particles=n),
                              can_contain_double_entries=False, indices_sorted=False)
    deltas = math.pairwise_differences(xt, format=conn)
    distances = math.vec_length(deltas, eps=1e-5)
    kernel = norm * (s ** 2 - math.vec_squared(deltas)) ** 3
    rho = math.sum(kernel, dual) * m
    pressure = 20. * (rho - 1.)
    nb_rho = rename_dims(rho, instance, dual)
    nb_pressure = rename_dims(pressure, instance, dual)
    gaps = h - distances
    avg_pressure = (math.tensor_like(kernel, 1) * pressure + nb_pressure) / (2 * nb_rho)
    pressure_force = -math.safe_div(deltas, distances) * avg_pressure * gaps ** 2
    dv = math.pairwise_differences(vt, format=kernel)
    viscous_force = dv / nb_rho * gaps
    force = math.sum(P * pressure_force + V * viscous_force, dual)
    a = force / rho + gravity
    vt = vt + a * (0.01 * h)
    xt = xt + (0.01 * h) * vt
    clipped = math.clip(xt, lo, up)
    vt = math.where(clipped == xt, vt, vt * -0.95)
    return (clipped.numpy(['particles', 'vector']).astype(F), vt.numpy(['particles', 'vector']).astype(F), (I, J),
            rho.numpy(['particles']).astype(F), force.numpy(['particles', 'vector']).astype(F), search)


def lattice(dims, h=H, seed=0):
    rng = np.random.default_rng(seed)
    d = len(dims)
    grid = np.stack(np.meshgrid(*[np.arange(k) for k in dims], indexing='ij'), -1).reshape(-1, d).astype(F) * F(h)
    return (grid + F(0.001 * h) * rng.standard_normal(grid.shape).astype(F)).astype(F)


def special(d, seed):
    """A small box with every edge case: leaving particles, pairs at exactly s, a pair closer than sqrt(1e-5), an isolated particle
    and particles above the upper corner."""
    rng = np.random.default_rng(seed)
    s = F(constants(d)[0].numpy())
    upper = np.full(d, 4.0, F)
    x, v = [], []
    # a cluster in the middle, at rest
    c = np.full(d, 2.0, F)
    x += list(c + (rng.random((24, d)).astype(F) - F(0.5)) * F(1.6))
    v += [np.zeros(d, F)] * 24
    # a pair at distance exactly s along x and a pair closer than sqrt(1e-5), near the lower corner
    a = np.full(d, 0.125, F); b = a.copy(); b[0] = a[0] + s     # 0.125 and s share the ulp of [0.5, 1): exact
    assert b[0] - a[0] == s and np.sqrt(F(b[0] - a[0]) * F(b[0] - a[0])) == s
    x += [a, b]; v += [np.zeros(d, F)] * 2
    e = np.full(d, 0.3, F); e[0] = 3.6; e2 = e.copy(); e2[1] += F(1e-3)
    x += [e, e2]; v += [np.zeros(d, F)] * 2
    # isolated
    iso = np.full(d, 3.5, F); iso[0] = 0.2
    x.append(iso); v.append(np.zeros(d, F))
    # leaving on one axis (fast outward along y) and on several (diagonal), both corners
    w = np.full(d, 2.0, F); w[1] = 3.95; x.append(w); vv = np.zeros(d, F); vv[1] = 20.0; v.append(vv)
    x.append(np.full(d, 3.97, F)); v.append(np.full(d, 15.0, F))
    x.append(np.full(d, 0.03, F)); v.append(np.full(d, -12.0, F))
    # starting above the upper corner: the top cell clamp
    t = np.full(d, 1.0, F); t[0] = 4.5; x.append(t); v.append(np.zeros(d, F))
    t = np.full(d, 1.2, F); t[0] = 6.1; x.append(t); v.append(np.zeros(d, F))
    return np.asarray(x, F), np.asarray(v, F), np.zeros(d, F), upper


def main():
    cases = {}
    for d in (3, 2):
        dims = (5, 6, 5) if d == 3 else (10, 12)
        x = lattice(dims, seed=d)
        cases[f'lattice{d}'] = (x, np.zeros_like(x), np.zeros(d, F), np.full(d, 80., F))
        xs, vs, lo, up = special(d, seed=10 + d)
        cases[f'special{d}'] = (xs, vs, lo, up)
    out = {}
    meta = {'phiml': __import__('phiml').__version__, 'numpy': np.__version__, 'h': H, 'cases': []}
    for name, (x, v, lo, up) in cases.items():
        d = x.shape[1]
        s, m, P, V, norm = constants(d)
        for substeps in (1, 5):
            key = f'{name}_{substeps}'
            meta['cases'].append(key)
            xc, vc = x, v
            for k in range(substeps):
                xc, vc, (I, J), rho, force, search = step(xc, vc, d, lo, up)
                if k == 0:
                    out[f'{key}/rows'], out[f'{key}/cols'] = I.astype(np.int32), J.astype(np.int32)
                    out[f'{key}/search_rows'], out[f'{key}/search_cols'] = search[:, 0].astype(np.int32), search[:, 1].astype(np.int32)
                    out[f'{key}/rho'], out[f'{key}/force'] = rho, force
            out[f'{key}/x0'], out[f'{key}/v0'], out[f'{key}/lower'], out[f'{key}/upper'] = x, v, lo, up
            out[f'{key}/x'], out[f'{key}/v'] = xc, vc
            out[f'{key}/substeps'] = np.int32(substeps)
            out[f'{key}/const'] = np.array([t.numpy() for t in (s, m, P, V, norm)], F)   # s, m, P, V, norm
    out['meta'] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, len(meta['cases']), 'cases')


if __name__ == '__main__':
    main()
