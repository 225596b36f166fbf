"""
Generates tests/golden/phiml_julia.npz  --  run ONLY where the reference's PhiML is reachable:

    python tests/golden/make_julia_golden.py

The Julia_Set notebook (examples/grids/Julia_Set.ipynb) with the vendored PhiML 1.7.2 on its NumPy backend, float32 / complex64:

    c = 0.7885 * math.exp(1j*math.linspace(0, 2*PI, batch(time=100)))
    def julia_map(z, counter, c):
        next_z = z ** 2 + c
        counter += abs(z) < 2
        return next_z, counter
    counts = iterate(julia_map, iter_count, re + im*1j, 0, c=c)[1]        # at the cell centres (re, im)

`phi` cannot be imported (it needs a newer phiml), so the cell centres are restated on phiml tensors from the cited lines:
lower + linspace(0.5/n, 1 - 0.5/n, n) * size (UniformGrid.center, phi/geom/_grid.py:60-63, Box.local_to_global, _box.py:154-158).
julia_map, iterate, exp, linspace and the complex arithmetic are PhiML's own.  The complex64 rounding comes from NumPy's SIMD loops,
so the file records the CPU features NumPy dispatched to (`numpy/simd_found`, as np.show_runtime() lists them): on this record
abs(z) = big * sqrt(fma(r, r, 1)), and PhiML's z ** 2 = np.power(z, 2) = (a*a - b*b, a*b + b*a) without fma (tests/oracle_julia.py
reproduces every count).

Cases (`<case>/c`: complex64 constants as (re, im) float32 pairs, `<case>/centres`: n_x x then n_y y centres, `<case>/counts`: uint8
(batch, x, y), `<case>/iterations`):
  notebook   every 11th of the notebook's 100 constants at 256 x 256 in Box(-2..2, -2..2), 50 iterations
  band_*     thin boxes around |z0| = 2 (on the x axis, the y axis and the diagonal); `<case>/hypot_differs` counts the cells where a
             correctly rounded hypot in place of NumPy's abs gives another count
  iter0 / iter1 / iter50   a ragged 37 x 23 grid with three constants and 0, 1 and 50 iterations
  big_c      constants with |c| > 2, inside and beyond the kernel's early-exit bound (|re|, |im| <= 4), 50 iterations
  nonfinite  inf and NaN constants, 50 iterations
"""
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import math  # noqa: E402  (imports phiml from the reference's PhiML tree)
from phiml.math import batch, spatial, tensor, wrap  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
NB_BOX = ((-2., 2.), (-2., 2.))
CASES = {
    # name: (resolution, ((x lower, x upper), (y lower, y upper)), constants, iterations)
    'band_x': ((64, 48), ((2 - 1e-6, 2 + 1e-6), (-1e-3, 1e-3)), [0.7885 + 0j, -0.8 + 0.156j], 50),
    'band_y': ((48, 64), ((-1e-3, 1e-3), (2 - 1e-6, 2 + 1e-6)), [0.7885 + 0j, 0.285 + 0.01j], 50),
    'band_diag': ((40, 40), ((2 ** .5 - 1e-6, 2 ** .5 + 1e-6), (2 ** .5 - 1e-6, 2 ** .5 + 1e-6)), [-0.4 + 0.6j], 50),
    'iter0': ((37, 23), ((-1.7, 2.1), (-1.3, 0.9)), [0.7885 + 0j, -0.7269 + 0.1889j, 0.355 + 0.355j], 0),
    'iter1': ((37, 23), ((-1.7, 2.1), (-1.3, 0.9)), [0.7885 + 0j, -0.7269 + 0.1889j, 0.355 + 0.355j], 1),
    'iter50': ((37, 23), ((-1.7, 2.1), (-1.3, 0.9)), [0.7885 + 0j, -0.7269 + 0.1889j, 0.355 + 0.355j], 50),
    'big_c': ((48, 40), ((-2.5, 2.5), (-2., 2.)), [2.5 + 0.5j, -0.3 - 3.9j, -4.5 + 0.1j, 7 + 7j], 50),
    'nonfinite': ((24, 20), ((-2., 2.), (-2., 2.)), [complex(np.inf, 0), complex(np.nan, 0.3), complex(0.2, -np.inf)], 50),
}


def julia_map(z, counter, c):
    next_z = z ** 2 + c
    counter += abs(z) < 2
    return next_z, counter


def cell_centres(res, box):
    """Per-axis float32 cell centres: lower + linspace(0.5/n, 1 - 0.5/n, n) * size."""
    return [(math.linspace(0.5 / n, 1 - 0.5 / n, spatial(x=n)) * wrap(np.float32(u - l)) + wrap(np.float32(l))).numpy().astype(np.float32)
            for n, (l, u) in zip(res, box)]


def counts(axes, c, iterations):
    """The notebook's sampling function at the cell centres `axes`, for the phiml batch tensor c; (time, x, y) int32."""
    re, im = (tensor(g, spatial('x,y')) for g in np.meshgrid(*axes, indexing='ij'))
    cnt = math.iterate(julia_map, iterations, re + im * 1j, 0, c=c)[1]
    shape = (c.shape.get_size('time'),) + tuple(len(a) for a in axes)
    if not isinstance(cnt, math.Tensor):                  # iterations == 0: the initial counter 0
        return np.full(shape, cnt, np.int32)
    assert cnt.dtype.kind == int and cnt.dtype.bits == 32, cnt.dtype
    return np.broadcast_to(cnt.numpy('time,x,y'), shape).astype(np.int32)     # one iteration: counts of z0 only, without `time`


def hypot_counts(axes, c, iterations):
    """The same map with abs(z) replaced by the correctly rounded hypot (float64 hypot rounded to float32)."""
    a, b = (g.astype(np.float32) for g in np.meshgrid(*axes, indexing='ij'))
    z = (a + 1j * b).astype(np.complex64)[None].repeat(len(c), 0)
    cc = np.asarray(c, np.complex64)[:, None, None]
    cnt = np.zeros(z.shape, np.int32)
    with np.errstate(all='ignore'):
        for _ in range(iterations):
            cnt += np.hypot(z.real.astype(np.float64), z.imag.astype(np.float64)).astype(np.float32) < 2
            z = z ** 2 + cc
    return cnt


def pairs(c):
    return np.asarray(c, np.complex64).view(np.float32).reshape(-1, 2)


def main():
    from numpy._core._multiarray_umath import __cpu_dispatch__, __cpu_features__
    out = {'numpy/version': np.array(np.__version__), 'numpy/simd_found': np.array(' '.join(f for f in __cpu_dispatch__ if __cpu_features__[f]))}
    c_all = 0.7885 * math.exp(1j * math.linspace(0, 2 * math.PI, batch(time=100)))
    assert c_all.dtype.kind == complex and c_all.numpy().dtype == np.complex64
    out['notebook/c_all'] = pairs(c_all.numpy('time'))
    pick = list(range(0, 100, 11))
    out['notebook/pick'] = np.array(pick, np.int32)
    axes = cell_centres((256, 256), NB_BOX)
    sub = math.tensor(c_all.numpy('time')[pick], batch('time'))
    out['notebook/c'] = pairs(sub.numpy('time'))
    out['notebook/centres'] = np.concatenate(axes)
    out['notebook/counts'] = counts(axes, sub, 50).astype(np.uint8)
    out['notebook/iterations'] = np.int32(50)
    out['notebook/box'] = np.array(NB_BOX, np.float64)
    for name, (res, box, cs, iterations) in CASES.items():
        axes = cell_centres(res, box)
        c = math.tensor(np.asarray(cs, np.complex64), batch('time'))
        got = counts(axes, c, iterations)
        out[f'{name}/c'] = pairs(cs)
        out[f'{name}/centres'] = np.concatenate(axes)
        out[f'{name}/counts'] = got.astype(np.uint8)
        out[f'{name}/iterations'] = np.int32(iterations)
        out[f'{name}/box'] = np.array(box, np.float64)
        if name.startswith('band'):
            out[f'{name}/hypot_differs'] = np.int32((hypot_counts(axes, cs, iterations) != got).sum())
    np.savez_compressed(os.path.join(OUT, 'phiml_julia.npz'), **out)
    print(out['numpy/simd_found'], {k: int(v) for k, v in out.items() if k.endswith('hypot_differs')},
          {k: v.shape for k, v in out.items() if k.endswith('/counts')})


if __name__ == '__main__':
    main()
