#!/usr/bin/env python
"""The fp64 path (math.set_global_precision(64)) on one GPU.

    python tools/fp64_bench.py [--steps 50] [--reps 5] [--out FILE]

1. The Taylor-Green notebook's size (25 x 25, periodic): microseconds per step of examples/taylor_green.py's `step` (diffuse.explicit,
   semi_lagrangian, make_incompressible with Solve('CG', 1e-12, 1e-12, x0=p)), host clock around --steps steps ending in a device
   synchronise, median over --reps; next to the same step of the float64 oracle (tests/oracle_fp64.py) on the host's cores.
2. Large grids (256^3 and 512^3, batch 1, periodic): the fp64 CG (phicuda_cg_poisson_f64) run for a fixed number of iterations,
   milliseconds per iteration (CUDA events around a 40- and a 20-iteration solve, the difference over 20 iterations, median over
   --reps) and the share of the HBM bound at 64 B/cell per iteration (3.35 TB/s); and at 512^3 the one-thread-per-sample divergence,
   grad_sub and staggered advection kernels in milliseconds per call, with the HBM rate at the bytes each must move.
Prints one JSON object with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'examples'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import oracle_np as O  # noqa: E402
from phiflow_b200 import _ops  # noqa: E402
import taylor_green as tg  # noqa: E402

HBM = 3.35e12
F64 = torch.float64


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip()


def notebook(steps, reps):
    from oracle_fp64 import taylor_green_step
    from phiflow_b200.flow import CenteredGrid, StaggeredGrid, math
    with math.precision(64):
        v0 = StaggeredGrid(tg.analytic_velocity(0.), **tg.domain())
        p0 = CenteredGrid(tg.analytic_pressure(0.), **tg.domain())
    v, p = tg.step(v0, p0, tg.DT)                       # warm-up: module loads, workspaces
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        v, p = v0, p0
        t0 = time.perf_counter()
        for _ in range(steps):
            v, p = tg.step(v, p, tg.DT)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) / steps * 1e6)
    vbc, res, dx = O.uniform_bc(2, 'periodic'), (tg.N, tg.N), (2 * np.pi / tg.N,) * 2
    vo, po = tg.analytic_velocity(0.), tg.analytic_pressure(0.)
    t0 = time.perf_counter()
    n_oracle = 10
    for _ in range(n_oracle):
        vo, po, _ = taylor_green_step(vo, po, tg.DT, tg.VISCOSITY, vbc, res, dx, (0., 0.), (2 * np.pi,) * 2)
    oracle_us = (time.perf_counter() - t0) / n_oracle * 1e6
    return {'gpu_us_per_step': float(np.median(times)), 'gpu_us_all_reps': [round(t, 1) for t in times], 'oracle_us_per_step': oracle_us}


def timed(fn, reps):
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def large(n, reps, kernels):
    res, dx = (n, n, n), (1.0, 1.0, 1.0)
    vbc = O.uniform_bc(3, 'periodic')
    dom = _ops.Domain(res, dx, 1, vbc=vbc, dtype=F64)
    g = torch.Generator(device='cuda').manual_seed(0)
    rhs = torch.randn(dom.alloc_centered().shape, generator=g, device='cuda', dtype=F64)
    x = dom.alloc_centered()
    out = {}

    def solve(k):
        prm = _ops.cg_params(vbc, rtol=0.0, atol=0.0, max_iter=k, dtype=F64)
        x.zero_()
        _ops.cg_poisson(dom, vbc, rhs, x, prm)
    solve(20)
    t20, t40 = timed(lambda: solve(20), reps), timed(lambda: solve(40), reps)
    assert int(_ops.read_results(dom)['iterations'][0]) == 40
    per_it = float(np.median([(b - a) / 20 for a, b in zip(t20, t40)]))
    cells = n ** 3
    out['cg_ms_per_iteration'] = per_it
    out['cg_hbm_share_64B_per_cell'] = 64 * cells / (per_it * 1e-3) / HBM
    if kernels:
        v = [torch.randn(dom.alloc_faces()[0].shape, generator=g, device='cuda', dtype=F64) for _ in range(3)]
        div = dom.alloc_centered()
        vout = dom.alloc_faces()
        calls = 5
        for name, fn, nbytes in [
                ('divergence', lambda: _ops.divergence(dom, vbc, v, out=div), 4 * 8 * cells),            # 3 components read, div written
                ('grad_sub', lambda: _ops.grad_sub(dom, vbc, v, x), 7 * 8 * cells),                     # p, 3 read + 3 written
                ('advect_staggered', lambda: _ops.advect_staggered(dom, vbc, v, vbc, v, 0.5, out=vout), 6 * 8 * cells)]:
            fn()
            ts = timed(lambda: [fn() for _ in range(calls)], reps)
            ms = float(np.median(ts)) / calls
            out[f'{name}_ms'] = ms
            out[f'{name}_TBps_at_{nbytes // cells}B_per_cell'] = nbytes / (ms * 1e-3) / 1e12
    del dom
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fp64_bench measures the GPU; there is nothing to measure without one"
    result = {'card': card(), 'notebook_25x25': notebook(args.steps, args.reps),
              'grid_256': large(256, args.reps, False), 'grid_512': large(512, args.reps, True)}
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(text + '\n')


if __name__ == '__main__':
    main()
