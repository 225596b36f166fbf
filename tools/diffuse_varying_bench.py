#!/usr/bin/env python
"""Implicit diffusion with a varying diffusivity (phicuda_diffuse_implicit_varying_f32) on one GPU, next to the plain-number
diffusivity solve (phicuda_diffuse_implicit_f32) on the same grid in the same run.

    python tools/diffuse_varying_bench.py [--size 512] [--reps 3] [--iters 100]

Cases: a size^3 field with a blocky diffusivity (background 0.01, blocks of 1: contrast 100), all periodic and with a constant x-
side (x-: 1, x+: ZERO_GRADIENT, y, z periodic), dt = 1.  Every solve runs a fixed --iters CG iterations (rtol = atol = 0), so that
both operators are timed over the same work.  Per case: ms per solve and per iteration (CUDA events, median over --reps after one
warm-up solve), and the HBM rate at the stated byte count per cell and iteration: 30 B for the plain-number operator (pass A: r, d
read, d' written; pass B: d' read, r read and written, x every second iteration) and 38 B for the varying one (k read once more in
each of the two sweeps)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from phiflow_b200 import _ops as ops  # noqa: E402
from phiflow_b200._clocks import ClockSampler  # noqa: E402

PER = ('periodic', 'periodic')


def _timed(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def _random(dom, gen):
    t = dom.alloc_centered()
    idx = (slice(None),) + tuple(slice(0, dom.res[a]) for a in range(dom.dim - 1, -1, -1))
    t[idx] = torch.randn((dom.batch,) + tuple(reversed(dom.res)), generator=gen, device=dom.device)
    return t


def _blocky(dom, seed=0):
    """0.01 everywhere, 1.0 in 8 random boxes of up to a quarter of the edge length."""
    rng = np.random.default_rng(seed)
    k = torch.full_like(dom.alloc_centered(), 0.01)
    n = dom.res
    for _ in range(8):
        lo = [int(rng.integers(0, m)) for m in n]
        hi = [min(m, l + int(rng.integers(1, m // 4 + 2))) for l, m in zip(lo, n)]
        k[0, lo[2]:hi[2], lo[1]:hi[1], lo[0]:hi[0]] = 1.0
    return k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--iters', type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA device')
    dev = torch.device('cuda:0')
    gen = torch.Generator(device=dev).manual_seed(0)
    sampler = ClockSampler(0)
    sampler.start()
    out = {'cases': []}
    n, its = args.size, args.iters
    dom = ops.Domain((n,) * 3, (1.0,) * 3, 1, device=dev)
    u = _random(dom, gen)
    k = _blocky(dom)
    for name, spec in (('periodic', (PER,) * 3), ('constant x-', ((1.0, 'zg'), PER, PER))):
        for op, fn, bpc in (('varying k', lambda: ops.diffuse_implicit_varying(dom, spec, u, k, 1.0, 0.0, 0.0, its), 38.0),
                            ('scalar k', lambda: ops.diffuse_implicit(dom, spec, u, 0.5, 0.0, 0.0, its), 30.0)):
            ms = _timed(fn, args.reps)
            rec = ops.read_results(dom)
            info = ops.last_launch_info()
            it = int(rec['iterations'][0])
            out['cases'].append({'case': f'{name} {n}^3', 'operator': op, 'cg_operator': ops.last_cg_operator(), 'iterations': it,
                                 'ms_per_solve': ms, 'ms_per_iteration': ms / max(it, 1), 'passes': info['passes'],
                                 'generic': info['generic'], 'bytes_per_cell_iteration': bpc,
                                 'tbs': bpc * n ** 3 * it / (ms * 1e-3) / 1e12})
    clocks = sampler.summary()
    out.update({'gpu': clocks.get('gpu') or torch.cuda.get_device_name(0), 'power_limit_w': clocks.get('power_limit_w'),
                'sm_mhz_median': clocks.get('sm_mhz'), 'clock_reasons': clocks.get('reasons')})
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
