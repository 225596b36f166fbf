"""
Generates tests/golden/phiml_diffuse_varying.npz  --  run ONLY where the reference's PhiML is reachable:

    python tests/golden/make_diffuse_varying_golden.py

diffuse.implicit(u, k, dt) with a spatially varying diffusivity k (phi/physics/diffuse.py:48-59, 90-95, 129-141) with the vendored
PhiML.  `phi` cannot be imported (it needs a newer phiml), so its glue is restated here on phiml tensors with phiml ops:
    w = k * (-dt)                                  amount of explicit(x, k, -dt), fp32 (diffuse.py:48)
    w takes u's extrapolation, constants included  amount.at(u), keep_boundary=False (phi/field/_resample.py:56-63)
    f = minimum(w_lo, w_hi) on every face          stagger(w, math.minimum, NONE) (phi/field/_field_math.py:535-581)
    g = (x_hi - x_lo) / dx on every face           spatial_gradient(x, boundary=NONE, at='face') (_field_math.py:229-236)
    sharpen(x) = x + sum_d (F_{i+1/2} - F_{i-1/2}) / dx_d, F = f * g   divergence, order 2 (_field_math.py:617-626)
Everything numerical - pad, minimum, slicing, tracing the affine map with jit_compile_linear and the CG of
solve_linear(Solve('CG', rtol, 1e-5, x0=y)) - is PhiML's own code (PhiML/phiml/math/_optimize.py:616-645).
Cases: 2-D zero / periodic / all-ZERO_GRADIENT / per-side mixes with non-zero constants, Heat_Flow's boundary with a bars-like
k of contrast 100, a 3-D mix, anisotropic dx, two batch entries with their own k, and back-diffusion (dt < 0) with a constant side
whose value lies below the edge coefficient, so that the boundary face takes min(w_edge, c) = c.  rtol 1e-3 and 1e-5 each.
"""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports phiml from /root/reference/PhiML)
from make_golden import math, Solve  # noqa: E402
from phiml.math import batch, spatial, tensor  # noqa: E402

NAMES = 'xyz'


def bars(res, rng, contrast=100.0, base=0.01):
    """Two axis-aligned boxes of k = base * contrast on a background of k = base (Heat_Flow's `bars + .01`)."""
    k = np.full(res, base, np.float32)
    for _ in range(2):
        lo = [int(rng.integers(0, n - 2)) for n in res]
        hi = [int(min(n, l + rng.integers(2, max(3, n // 2)))) for l, n in zip(lo, res)]
        k[tuple(slice(l, h) for l, h in zip(lo, hi))] = base * contrast
    return k


CASES = [   # name, boundary spec, resolution, dx, dt, k(rng)
    ('zero', ((0.0, 0.0), (0.0, 0.0)), (16, 12), (1.0, 1.0), 1.0, lambda r, rng: bars(r, rng)),
    ('periodic', (('periodic', 'periodic'), ('periodic', 'periodic')), (16, 12), (1.0, 1.0), 1.0, lambda r, rng: bars(r, rng)),
    ('zg', (('zg', 'zg'), ('zg', 'zg')), (16, 12), (1.0, 1.0), 1.0, lambda r, rng: bars(r, rng)),
    ('mixed', ((0.5, 'zg'), (-0.25, 0.75)), (16, 12), (1.0, 1.0), 1.0,
     lambda r, rng: rng.uniform(0.05, 1.0, r).astype(np.float32)),
    ('heat', ((1.0, 'zg'), ('periodic', 'periodic')), (20, 10), (1.0, 1.0), 1.0, lambda r, rng: bars(r, rng)),   # Heat_Flow.ipynb
    ('aniso', ((0.5, 'zg'), ('zg', -0.25)), (16, 12), (0.5, 0.25), 0.05, lambda r, rng: bars(r, rng)),
    ('mixed3', (('periodic', 'periodic'), (0.5, 'zg'), ('zg', -0.5)), (8, 6, 7), (1.0, 0.5, 1.0), 0.5, lambda r, rng: bars(r, rng)),
    ('back', ((0.01, 'zg'), ('zg', 0.0)), (16, 12), (1.0, 1.0), -0.05,
     lambda r, rng: rng.uniform(0.5, 1.0, r).astype(np.float32)),                # dt < 0: w = 0.05 k > 0.01 = c at x-
]


def sharpen(x, w, ext, dx):
    total = x
    for i, dim in enumerate(x.shape.spatial.names):
        n = x.shape.get_size(dim)
        wp = math.pad(w, {dim: (1, 1)}, ext)
        xp = math.pad(x, {dim: (1, 1)}, ext)
        f = math.minimum(wp[{dim: slice(0, n + 1)}], wp[{dim: slice(1, n + 2)}])
        grad = (xp[{dim: slice(1, n + 2)}] - xp[{dim: slice(0, n + 1)}]) / dx[i]
        flux = f * grad
        total = total + (flux[{dim: slice(1, n + 1)}] - flux[{dim: slice(0, n)}]) / dx[i]
    return total


def solve(y, w, ext, dx, rtol):
    lin = math.jit_compile_linear(sharpen, auxiliary_args='w,ext,dx')
    s = Solve('CG', rtol, 1e-5, x0=y, max_iterations=1000)
    with math.SolveTape() as tape:
        x = math.solve_linear(lin, y, s, w=w, ext=ext, dx=dx)
    return x, tape[s].iterations


def main():
    out = {}
    rng = np.random.default_rng(29)
    for name, spec, res, dx, dt, kfn in CASES:
        d = len(res)
        ext = G.ext_from_spec(spec)
        u = rng.standard_normal(res).astype(np.float32)
        k = kfn(res, rng)
        out[f'{name}/bc'] = G.spec_to_arr(spec)
        out[f'{name}/dx'] = np.array(dx)
        out[f'{name}/dt'] = np.array(dt)
        out[f'{name}/u'] = u
        out[f'{name}/k'] = k
        w = G.to_tensor(k) * (-dt)
        for rtol, tag in ((1e-3, 'r3'), (1e-5, 'r5')):
            x, it = solve(G.to_tensor(u), w, ext, dx, rtol)
            out[f'{name}/{tag}/x'] = G.npy(x, d)
            out[f'{name}/{tag}/iterations'] = np.array(int(it))
    # two batch entries with their own k.  A k with a batch dim makes the traced matrix batch-dependent, and PhiML 1.7.2 then runs
    # ONE CG over the block-diagonal system with one stopping rule ('batch/joint/...', one iteration count).  Each entry solved
    # alone ('batch/<b>/...') is what the library computes, one system per entry as for a plain-number diffusivity.
    res, dx, dt, spec = (16, 12), (1.0, 1.0), 1.0, ((1.0, 'zg'), ('periodic', 'periodic'))
    u = rng.standard_normal((2,) + res).astype(np.float32)
    k = np.stack([bars(res, rng), rng.uniform(0.05, 1.0, res).astype(np.float32)])
    out['batch/bc'] = G.spec_to_arr(spec)
    out['batch/dx'] = np.array(dx)
    out['batch/dt'] = np.array(dt)
    out['batch/u'] = u
    out['batch/k'] = k
    yb = tensor(u, batch('b'), spatial('x,y'))
    wb = tensor(k, batch('b'), spatial('x,y')) * (-dt)
    for rtol, tag in ((1e-3, 'r3'), (1e-5, 'r5')):
        x, it = solve(yb, wb, G.ext_from_spec(spec), dx, rtol)
        out[f'batch/joint/{tag}/x'] = x.numpy('b,x,y')
        out[f'batch/joint/{tag}/iterations'] = np.array(int(it.max))
        for b in range(2):
            x, it = solve(G.to_tensor(u[b]), G.to_tensor(k[b]) * (-dt), G.ext_from_spec(spec), dx, rtol)
            out[f'batch/{b}/{tag}/x'] = G.npy(x, 2)
            out[f'batch/{b}/{tag}/iterations'] = np.array(int(it))
    np.savez_compressed(os.path.join(G.OUT, 'phiml_diffuse_varying.npz'), **out)
    print(f"wrote {len(out)} arrays")
    for key in sorted(out):
        if key.endswith('iterations'):
            print(key, out[key])


if __name__ == '__main__':
    main()
