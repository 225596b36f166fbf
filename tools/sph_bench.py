#!/usr/bin/env python
"""SPH (phicuda_sph_f32, kernel k_sph) on one GPU.

    python tools/sph_bench.py [--reps 5] [--substeps 40] [--out FILE]

Times, with CUDA events (median over --reps after a warm-up), `substeps` substeps of the SPH notebook's dam break:
  notebook  the notebook's 25 x 100 x 25 = 62 500 particles on its jittered lattice in Box(x=80, y=80, z=80)
  1m        2^20 particles: a 64 x 256 x 64 jittered lattice of the same spacing in Box(x=80, y=240, z=80)
each as ONE fused launch of all substeps (what sph_step(..., substeps=40) runs per frame) and as `substeps` launches of one substep
(what iterate(..., substeps=40) over sph_step runs, without its host copies).  The two results are compared bit for bit.  Rates are
substeps per second.  Prints one JSON object with the card's name and power limit, read in the same run."""
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

SIZES = {'notebook': ((25, 100, 25), (80., 80., 80.)), '1m': ((64, 256, 64), (80., 240., 80.))}
H = 0.8


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


def lattice(dims, seed=0):
    grid = np.stack(np.meshgrid(*[np.arange(k) for k in dims], indexing='ij'), -1).reshape(-1, 3).astype(np.float32) * np.float32(H)
    return (grid + np.float32(0.001 * H) * np.random.default_rng(seed).standard_normal(grid.shape).astype(np.float32)).astype(np.float32)


def bench(name, dims, upper, substeps, reps):
    volume = np.float32(4 / 3 * np.pi) * np.power(np.power(np.float32(.75 / np.pi) * np.asarray(H ** 3, np.float32), 1 / 3), 3)
    prm = _ops.sph_params((0., 0., 0.), upper, H, np.float32(0.01) * volume, 0.01 * H, (0., 0., -0.1))
    x = torch.from_numpy(lattice(dims)).cuda()
    v = torch.zeros_like(x)
    out = {}

    def fused():
        out['fused'] = _ops.sph(x, v, prm, substeps)

    def per_substep():
        xs, vs = x, v
        for _ in range(substeps):
            xs, vs = _ops.sph(xs, vs, prm, 1)
        out['split'] = (xs, vs)

    t_fused, t_split = timed(fused, reps), timed(per_substep, reps)
    torch.cuda.synchronize()
    same = all(torch.equal(a, b) for a, b in zip(out['fused'], out['split']))
    return {'size': name, 'particles': int(x.shape[0]), 'substeps': substeps, 'fused_ms': round(t_fused, 4),
            'per_substep_launches_ms': round(t_split, 4), 'fused_substeps_per_s': round(substeps / (t_fused * 1e-3), 1),
            'per_substep_substeps_per_s': round(substeps / (t_split * 1e-3), 1), 'speedup': round(t_split / t_fused, 3),
            'grid_ctas': _ops.last_launch_info()['grid_ctas'], 'same_bits': same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--substeps', type=int, default=40)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    _ops.require_cuda()
    rows = [bench(k, *SIZES[k], args.substeps, args.reps) for k in SIZES]
    result = {'card': card(), 'rows': rows}
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
