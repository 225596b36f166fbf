#!/usr/bin/env python
"""advect.points (phicuda_advect_points_f32, kernel k_advect_points) on one GPU.

    python tools/points_bench.py [--reps 5] [--out FILE]

Times, with CUDA events (median over --reps after a warm-up), RK4 trajectories of seeded points in a seeded random StaggeredGrid velocity
(ZERO_GRADIENT sides, Box of 1 per cell):
  notebook  the Streamlines notebook's size: 64 points, 50 steps of 0.1 in 256 x 256
  2d        2^22 tracers, 100 steps in 2048 x 2048
  3d        2^22 tracers, 100 steps in 256 x 256 x 256
each as ONE fused launch of all steps (what `streamlines` runs) and as `steps` launches of one step (what `iterate` over advect.points
runs, without its host copies).  Both write the final positions only; the two results are compared bit for bit.  Rates are
point-steps per second.  Prints one JSON object with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from phiflow_b200 import _ops  # noqa: E402

SIZES = {'notebook': ((256, 256), 64, 50), '2d': ((2048, 2048), 1 << 22, 100), '3d': ((256, 256, 256), 1 << 22, 100)}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def bench(name, res, n, steps, reps, dt=0.1):
    d = len(res)
    spec = (('zg', 'zg'),) * d
    dom = _ops.Domain(res, (1.0,) * d, 1, vbc=spec)
    rng = np.random.default_rng(1)
    v = [t.normal_(generator=torch.Generator(device='cuda').manual_seed(c)) for c, t in enumerate(dom.alloc_faces())]
    upper = tuple(float(r) for r in res)
    pts = torch.from_numpy((rng.random((1, n, d)) * np.asarray(upper)).astype(np.float32)).cuda()
    out1, outk = torch.empty_like(pts), torch.empty_like(pts)

    def fused():
        _ops.advect_points(dom, spec, v, (0.,) * d, upper, pts, dt, 'rk4', steps, out=out1)

    def per_step():
        _ops.advect_points(dom, spec, v, (0.,) * d, upper, pts, dt, 'rk4', 1, out=outk)
        for _ in range(steps - 1):
            _ops.advect_points(dom, spec, v, (0.,) * d, upper, outk, dt, 'rk4', 1, out=outk)

    t_fused, t_steps = timed(fused, reps), timed(per_step, reps)
    torch.cuda.synchronize()
    return {'size': name, 'res': list(res), 'points': n, 'steps': steps, 'fused_ms': round(t_fused, 4), 'per_step_launches_ms': round(t_steps, 4),
            'fused_point_steps_per_s': n * steps / (t_fused * 1e-3), 'per_step_point_steps_per_s': n * steps / (t_steps * 1e-3),
            'speedup': round(t_steps / t_fused, 3), 'same_bits': bool(torch.equal(out1, outk))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    _ops.require_cuda()
    rows = [bench(k, *SIZES[k], args.reps) for k in SIZES]
    result = {'card': card(), 'rows': rows}
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
