#!/usr/bin/env python
"""CG-adaptive with obstacles (k_cg_ring<..., ADAPT, CgOp::Masked>) next to plain CG with obstacles on the same system, one GPU.

    python tools/cg_adaptive_masked_bench.py [--reps 3] [--iters 200] [--steps 20]

Solver timing: every solve runs a fixed --iters iterations (rtol = atol = 0) from x0 = 0, CG and CG-adaptive alternating, median of
--reps after one warm-up solve each (CUDA events).  Workloads: the Wake_Flow geometry (examples/wake_flow.py) at 512 x 256 x 64 and
Batched_Smoke (examples/batched_smoke_obstacle.py) at 2048^2, batch 3.  The HBM rate is computed from byte counts per cell and
iteration that are EXPECTED, not measured: 38 B for masked CG (30 B of the two-sweep CG plus the mask's 4 B in each sweep) and 42 B
for masked CG-adaptive (34 B of CG-adaptive plus the mask's 4 B in each of the two sweeps).
Stopping rules: iterations per step of --steps warm-started Batched_Smoke steps at 256^2 under Solve('CG') and Solve() (= CG-adaptive).
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from phiflow_b200 import _ops as ops, _lib  # noqa: E402
from phiflow_b200._clocks import ClockSampler  # noqa: E402
import phiflow_b200.flow as flow  # noqa: E402

BYTES = {'CG': 38.0, 'CG-adaptive': 42.0}


def _solve_fn(dom, vbc, y, acc, method, iters):
    prm = ops.cg_params(vbc, rtol=0.0, atol=0.0, max_iter=iters, method=method)
    ws, res = dom.workspace()
    x = dom.alloc_centered()

    def fn():
        x.zero_()
        _lib.check(_lib.load().phicuda_cg_poisson_masked_f32(C.byref(dom.grid), C.byref(ops.make_vbc(vbc, dom.dim)), ops._ptr(y), ops._ptr(x),
                                                             ops._ptr(acc), C.byref(prm), ops._ptr(res), ops._ptr(ws), C.c_size_t(ws.numel()),
                                                             ops._stream()))
    return fn


def _time(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def solver_case(name, res, batch, bounds, vspec, obstacle, reps, iters):
    v = flow.StaggeredGrid(0, vspec, bounds, batch, **dict(zip('xyz', res)))
    accessible, _ = flow._obstacle_masks(v, obstacle)
    dom = v.dom
    gen = torch.Generator(device='cuda').manual_seed(0)
    y = dom.alloc_centered()
    idx = (slice(None),) + tuple(slice(0, dom.res[a]) for a in range(dom.dim - 1, -1, -1))
    y[idx] = torch.randn((batch,) + tuple(reversed(res)), generator=gen, device='cuda')
    y *= accessible
    vbc = v.vspec
    fns = {m: _solve_fn(dom, vbc, y, accessible, m, iters) for m in ('CG', 'CG-adaptive')}
    times, rows = {m: [] for m in fns}, []
    for m, fn in fns.items():
        fn()
    for _ in range(reps):
        for m, fn in fns.items():                       # alternating
            times[m].append(_time(fn))
    cells = int(np.prod(res)) * batch
    for m in fns:
        fns[m]()
        torch.cuda.synchronize()
        info, it = ops.last_launch_info(), int(ops.read_results(dom)['iterations'].max())
        ms = float(np.median(times[m])) / max(it, 1)
        rows.append({'case': name, 'method': m, 'iterations': it, 'ms_per_iteration': ms, 'masked': info['masked'], 'adaptive': info['adaptive'],
                     'TY': info['TY'], 'stages': info['stages'], 'expected_bytes_per_cell_iteration': BYTES[m],
                     'tbs_at_expected_bytes': BYTES[m] * cells / (ms * 1e-3) / 1e12})
    return rows


def smoke_iterations(res, steps):
    domain = flow.Box(x=100, y=100)
    obstacle = flow.Box(x=(35, 65), y=(50, 70))
    masks = np.stack([r * flow.resample(flow.Sphere(x=cx, y=9.5, radius=5), to=flow.CenteredGrid(0, flow.ZERO_GRADIENT, domain, x=res, y=res),
                                        soft=True).numpy() for r, cx in zip((.1, .2, .3), (40, 50, 60))])
    out = {}
    for label, make in (("Solve('CG')", lambda p: flow.Solve('CG', 1e-5, 1e-5, x0=p)), ('Solve()', lambda p: flow.Solve(x0=p))):
        v = flow.StaggeredGrid(0, 0, domain, batch=3, x=res, y=res)
        s = flow.CenteredGrid(0, flow.ZERO_GRADIENT, domain, batch=3, x=res, y=res)
        inflow = flow.CenteredGrid(masks, flow.ZERO_GRADIENT, domain, batch=3, x=res, y=res)
        p, its = None, []
        with flow.SolveTape() as tape:
            for _ in range(steps):
                s = flow.advect.mac_cormack(s, v, 1.) + inflow
                v = flow.advect.semi_lagrangian(v, v, 1.) + flow.resample(s * (0, 0.1), to=v) * 1.
                v, p = flow.fluid.make_incompressible(v, obstacle, make(p))
        its = [r[1].iterations.tolist() for r in tape.records]
        out[label] = its
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--steps', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA device')
    sampler = ClockSampler(0)
    sampler.start()
    cyl = flow.geom.infinite_cylinder(x=20, y=50, radius=10, inf_dim='z')
    wake = {'x-': flow.vec(x=2, y=0, z=0), 'x+': flow.ZERO_GRADIENT, 'y': flow.PERIODIC, 'z': flow.PERIODIC}
    rows = solver_case('Wake_Flow 512x256x64', (512, 256, 64), 1, flow.Box(x=200, y=100, z=5), wake, cyl, args.reps, args.iters)
    rows += solver_case('Batched_Smoke 2048^2 x3', (2048, 2048), 3, flow.Box(x=100, y=100), 0, flow.Box(x=(35, 65), y=(50, 70)),
                        args.reps, args.iters)
    its = smoke_iterations(256, args.steps)
    clocks = sampler.summary()
    out = {'gpu': clocks.get('gpu') or torch.cuda.get_device_name(0), 'power_limit_w': clocks.get('power_limit_w'),
           'sm_mhz_median': clocks.get('sm_mhz'), 'clock_reasons': clocks.get('reasons'), 'solver': rows,
           'batched_smoke_256_iterations_per_step': its}
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
