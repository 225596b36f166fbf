"""
Generates tests/golden/phiml_fp64.npz  --  run ONLY where the reference's PhiML is reachable:

    python tests/golden/make_fp64_golden.py

The reference's arithmetic layer (vendored PhiML 1.7.2, NumPy backend) under math.precision(64), the yardstick of the fp64 path
(math.set_global_precision(64), the Taylor-Green notebook).  The phi glue is restated on phiml tensors as in make_golden.py
(stagger / divergence / masked_laplace from there; the Taylor-Green step below); the numerics are PhiML's own.  Records:
  - laplace for every boundary set of make_golden.py, 2-D and 3-D, float64 inputs;
  - staggered divergence and the face gradient;
  - math.grid_sample at back-traced points (a seeded displacement of up to three cells from the cell centres);
  - solve_linear(Solve('CG', 1e-12, 1e-12)) of periodic, open and closed pressure systems in 2-D and 3-D (iteration counts and
    solutions).  Singular systems take a balanced right-hand side and rank_deficiency=0, i.e. plain CG without the random-probe
    matrix offset, as the library's pressure solve runs them;
  - one Taylor-Green step at 16^2 (diffuse.explicit -> semi_lagrangian -> make_incompressible with Solve('CG', 1e-12, 1e-12, x0=p)).
"""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports phiml from the reference tree)
from make_golden import math, to_tensor, npy, ext_from_spec, spec_to_arr, pressure_ext, remove_const, NAMES  # noqa: E402
from phiml.math import channel, instance, spatial, tensor, wrap, Solve  # noqa: E402
from phiml.math import extrapolation as E  # noqa: E402

SYSTEMS = {'periodic': 'periodic', 'closed': 0.0, 'open': 'zg'}       # velocity boundaries


def taylor_green_step(u, v, p, dt, nu, n, L):
    """One notebook step on a periodic n x n StaggeredGrid of Box(x=L, y=L): u at the x faces (i h, (j + 1/2) h), v at the y faces
    ((i + 1/2) h, j h), p at the cell centres."""
    P = E.PERIODIC
    h = L / n
    dxv = wrap((h, h), channel(vector='x,y'))
    # diffuse.explicit (phi/physics/diffuse.py:13-60): every component with its own (periodic) boundary, field + amount * laplace
    amount = nu * dt
    u = u + amount * math.laplace(u, dxv, padding=P)
    v = v + amount * math.laplace(v, dxv, padding=P)
    # semi_lagrangian (phi/physics/advect.py:156-179): the other component at the faces by shift resampling (_resample.py:341-364),
    # back-trace in world space, grid_sample on the component's own grid (lower' = -h/2 along its axis, size L, n points)
    comps = {'x': u, 'y': v}
    out = {}
    for c, t in (('x', 'y'), ('y', 'x')):
        other = comps[t]
        padded = math.pad(math.pad(other, {t: (0, 1)}, P), {c: (1, 1)}, P)
        at_faces = math.sample_subgrid(padded, wrap((0.5, 0.5), channel('vector')), spatial(**{'x': n + 1 if c == 'x' else n, 'y': n + 1 if c == 'y' else n}))
        at_faces = at_faces[{c: slice(0, n)}]
        own = comps[c]
        lower = {a: (-0.5 * h if a == c else 0.0) for a in 'xy'}
        pts = {a: lower[a] + math.linspace(0.5 / n, 1 - 0.5 / n, spatial(**{a: n})) * L for a in 'xy'}
        vel = {c: own, t: at_faces}
        lookup = {a: pts[a] - vel[a] * dt for a in 'xy'}
        coords = math.stack([(lookup[a] - lower[a]) / L * n - 0.5 for a in 'xy'], channel(vector='x,y'))
        out[c] = math.grid_sample(own, coords, P)
    u, v = out['x'], out['y']
    # make_incompressible (phi/physics/fluid.py:94-162) without the matrix offset
    vext = ext_from_spec((('periodic', 'periodic'),) * 2)
    pext = ext_from_spec(pressure_ext((('periodic', 'periodic'),) * 2))
    div = G.staggered_divergence([u, v], (h, h), vext)
    div = div - math.mean(div)
    lin = math.jit_compile_linear(G.masked_laplace, auxiliary_args='dx,pext,vext0')
    solve = Solve('CG', 1e-12, 1e-12, x0=p, max_iterations=1000, rank_deficiency=0)
    with math.SolveTape() as tape:
        p = math.solve_linear(lin, div, solve, dx=(h, h), pext=pext, vext0=vext)
    grad = G.stagger_grad(p, (h, h), pext, vext)
    return u - grad[0], v - grad[1], p, int(tape[solve].iterations)


def main():
    rng = np.random.default_rng(64)
    out = {}
    with math.precision(64):
        for name, spec in list(G.BC_SETS_2D.items()) + [(k + '3', s) for k, s in G.BC_SETS_3D.items()]:
            d = len(spec)
            shape = (7, 5) if d == 2 else (5, 4, 6)
            dx = (0.3, 2 * np.pi / 25) if d == 2 else (0.5, 0.3, 2 * np.pi / 25)
            ext = ext_from_spec(spec)
            a = rng.standard_normal(shape)
            out[f'laplace/{name}/bc'] = spec_to_arr(spec)
            out[f'laplace/{name}/dx'] = np.array(dx)
            out[f'laplace/{name}/in'] = a
            out[f'laplace/{name}/out'] = npy(math.laplace(to_tensor(a), wrap(dx, channel(vector=','.join(NAMES[:d]))), padding=ext), d)
            # grid_sample at back-traced points: cell centres displaced by up to three cells
            idx = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing='ij'), -1).reshape(-1, d)
            coords = idx + rng.uniform(-3, 3, idx.shape)
            ct = tensor(coords, instance('points'), channel(vector=','.join(NAMES[:d])))
            out[f'sample/{name}/bc'] = spec_to_arr(spec)
            out[f'sample/{name}/grid'] = a
            out[f'sample/{name}/coords'] = coords
            out[f'sample/{name}/out'] = math.grid_sample(to_tensor(a), ct, ext).numpy('points')
            # staggered divergence and face gradient
            if name.startswith('one'):
                continue
            vext = ext_from_spec(spec)
            pext = ext_from_spec(pressure_ext(spec))
            comps = []
            for c in range(d):
                lo, up = vext.valid_outer_faces(NAMES[c])
                s = list(shape); s[c] = shape[c] - 1 + int(lo) + int(up)
                comps.append(rng.standard_normal(s))
            p = rng.standard_normal(shape)
            out[f'fluid/{name}/bc'] = spec_to_arr(spec)
            out[f'fluid/{name}/dx'] = np.array(dx)
            out[f'fluid/{name}/p'] = p
            for c in range(d):
                out[f'fluid/{name}/v{c}'] = comps[c]
            out[f'fluid/{name}/div'] = npy(G.staggered_divergence([to_tensor(c) for c in comps], dx, vext), d)
            for c, g in enumerate(G.stagger_grad(to_tensor(p), dx, pext, vext)):
                out[f'fluid/{name}/grad{c}'] = npy(g, d)

        # CG through solve_linear
        for system, side in SYSTEMS.items():
            for d in (2, 3):
                spec = ((side, side),) * d
                res = (16, 12) if d == 2 else (10, 8, 7)
                dx = (0.5, 0.25) if d == 2 else (1.0, 0.5, 0.75)
                vext0 = ext_from_spec(remove_const(spec))
                pext = ext_from_spec(pressure_ext(spec))
                rhs = rng.standard_normal(res)
                if system != 'open':
                    rhs -= rhs.mean()
                lin = math.jit_compile_linear(G.masked_laplace, auxiliary_args='dx,pext,vext0')
                solve = Solve('CG', 1e-12, 1e-12, x0=to_tensor(np.zeros(res)), max_iterations=2000, rank_deficiency=0)
                with math.SolveTape() as tape:
                    x = math.solve_linear(lin, to_tensor(rhs), solve, dx=dx, pext=pext, vext0=vext0)
                key = f'cg/{system}{d}'
                out[f'{key}/bc'] = spec_to_arr(spec)
                out[f'{key}/dx'] = np.array(dx)
                out[f'{key}/rhs'] = rhs
                out[f'{key}/x'] = npy(x, d)
                out[f'{key}/iterations'] = np.array(int(tape[solve].iterations))

        # one Taylor-Green step at 16^2
        n, L, nu, dt = 16, 2 * np.pi, 0.1, 10. / 199
        h = L / n
        f, c = np.arange(n) * h, (np.arange(n) + 0.5) * h
        X, Y = np.meshgrid(f, c, indexing='ij')
        u0 = np.cos(X) * np.sin(Y)
        X, Y = np.meshgrid(c, f, indexing='ij')
        v0 = -np.sin(X) * np.cos(Y)
        X, Y = np.meshgrid(c, c, indexing='ij')
        p0 = -0.25 * (np.cos(2 * X) + np.cos(2 * Y))
        u1, v1, p1, it = taylor_green_step(to_tensor(u0), to_tensor(v0), to_tensor(p0), dt, nu, n, L)
        out.update({'tg/u0': u0, 'tg/v0': v0, 'tg/p0': p0, 'tg/u1': npy(u1, 2), 'tg/v1': npy(v1, 2), 'tg/p1': npy(p1, 2),
                    'tg/iterations': np.array(it), 'tg/params': np.array([n, L, nu, dt])})
    assert all(v.dtype != np.float32 for v in out.values())
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'phiml_fp64.npz')
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays")


if __name__ == '__main__':
    main()
