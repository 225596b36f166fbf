"""
Generates tests/golden/phiml_diffuse_implicit.npz  --  run ONLY where the reference's PhiML is reachable:

    python tests/golden/make_diffuse_implicit_golden.py

diffuse.implicit (phi/physics/diffuse.py:63-95) with the vendored PhiML: `sharpen` restated on phiml tensors exactly as
diffuse.explicit(x, diffusivity, -dt) reaches math.laplace (phi/field/_field_math.py:128: weights = diffusivity * -dt), traced by
jit_compile_linear and solved by solve_linear(Solve('CG', rtol, atol, x0=y)) - the affine system M x = y - bias
(PhiML/phiml/math/_optimize.py:616-645).  Fixtures for tests/oracle_diffuse.py (and through it the CUDA solve).
Cases: 2-D zero / periodic / per-side mixes, Heat_Flow's boundary (non-zero constant -> bias), a 3-D mix, anisotropic dx,
a/dx^2 in {0.1, 5}, rtol 1e-3 and 1e-5, and one 2-component periodic field with a channel('vector') dim, whose components
PhiML solves as separate systems.
"""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports phiml from /root/reference/PhiML)
from make_golden import math, Solve  # noqa: E402
from phiml.math import channel, spatial, tensor  # noqa: E402

CASES = [   # name, boundary spec, resolution, dx
    ('zero', ((0.0, 0.0), (0.0, 0.0)), (16, 12), (1.0, 1.0)),
    ('periodic', (('periodic', 'periodic'), ('periodic', 'periodic')), (16, 12), (1.0, 1.0)),
    ('mixed', (('zg', 0.0), (0.0, 'zg')), (16, 12), (1.0, 1.0)),
    ('heat', ((1.0, 'zg'), ('periodic', 'periodic')), (16, 12), (1.0, 1.0)),            # Heat_Flow.ipynb: {'x-': 1, 'x+': ZERO_GRADIENT, 'y': PERIODIC}
    ('aniso', ((0.5, 'zg'), ('zg', -0.25)), (16, 12), (0.5, 0.25)),
    ('mixed3', (('periodic', 'periodic'), (0.0, 'zg'), ('zg', 0.5)), (8, 6, 7), (1.0, 0.5, 1.0)),
]


def sharpen(x, dx, ext, a):
    return x + math.laplace(x, dx=dx, padding=ext, weights=-a)


def solve(y, dx, ext, a, rtol):
    lin = math.jit_compile_linear(sharpen, auxiliary_args='dx,ext,a')
    s = Solve('CG', rtol, 1e-5, x0=y, max_iterations=1000)
    with math.SolveTape() as tape:
        x = math.solve_linear(lin, y, s, dx=dx, ext=ext, a=a)
    return x, tape[s].iterations


def main():
    out = {}
    rng = np.random.default_rng(17)
    for name, spec, res, dx in CASES:
        d = len(res)
        ext = G.ext_from_spec(spec)
        u = rng.standard_normal(res).astype(np.float32)
        out[f'{name}/bc'] = G.spec_to_arr(spec)
        out[f'{name}/dx'] = np.array(dx)
        out[f'{name}/u'] = u
        for k in (0.1, 5.0):
            a = float(k * min(dx) ** 2)
            for rtol, tag in ((1e-3, 'r3'), (1e-5, 'r5')):
                x, it = solve(G.to_tensor(u), dx, ext, a, rtol)
                out[f'{name}/k{k:g}/{tag}/x'] = G.npy(x, d)
                out[f'{name}/k{k:g}/{tag}/iterations'] = np.array(int(it))
                out[f'{name}/k{k:g}/amount'] = np.array(a)
    # two components of a periodic vector field: the tracer keeps the uncoupled vector dim out of the matrix, so solve_linear runs
    # one system per component (per-component iteration counts)
    res, dx = (16, 12), (1.0, 1.0)
    u = rng.standard_normal(res + (2,)).astype(np.float32)
    y = tensor(u, spatial('x,y'), channel(vector='x,y'))
    out['vec2/u'] = u
    for rtol, tag in ((1e-3, 'r3'), (1e-5, 'r5')):
        x, it = solve(y, dx, G.ext_from_spec((('periodic', 'periodic'),) * 2), 2.0, rtol)
        out[f'vec2/{tag}/x'] = x.numpy('x,y,vector')
        out[f'vec2/{tag}/iterations'] = it.numpy('vector')
    np.savez_compressed(os.path.join(G.OUT, 'phiml_diffuse_implicit.npz'), **out)
    print(f"wrote {len(out)} arrays")


if __name__ == '__main__':
    main()
