#!/usr/bin/env python
"""One-sweep against two-sweep CG on the bench's 512^3 plume state (one GPU).

    python tools/cg_passes_bench.py [--size 512] [--rounds 5] [--warmup 3]

The plume of bench.py is advanced `--warmup` steps; then, `--rounds` times, each form (PHICUDA_CG_PASSES unset = one sweep per
iteration where it applies, =2 = two sweeps) runs the next plume step from the same saved state, in alternating order.  Reported per
form: the pressure solve's time (CUDA events recorded by the library around the solve), its iterations, and the achieved HBM rate
for the algorithmic byte counts of one_sweep_bytes (one-sweep) and cells * (30 it + 32) (two-sweep, the count bench.py reports)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from phiflow_b200 import _ops as ops  # noqa: E402
from phiflow_b200._clocks import ClockSampler  # noqa: E402


def one_sweep_bytes(cells, it):
    """Bytes of a one-sweep solve of `it` iterations: d_k, d_{k-1} read and d_{k+1} written (12 B/cell per iteration), the x read
    and write of every third sweep (8 B/cell), the steps still owed after the loop (it % 3 = 1: x and d_k, 12 B/cell; = 2: x, d_k
    and d_{k-1}, 16 B/cell), set-up passes 32 + the q_0 sweep 8.  Counts the cadence without the small-beta guard, which makes a
    sweep apply two steps early; it does not trigger on the plume's solves."""
    it = np.asarray(it, np.int64)
    return cells * (12.0 * it + 8.0 * (it // 3) + np.choose(it % 3, [0.0, 12.0, 16.0]) + 40.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA device')
    dev = torch.device('cuda:0')
    n = args.size
    cells = float(n) ** 3
    sim = bench.PlumeSim(n, dev)
    _, res_dev = sim.dom.workspace()
    for _ in range(args.warmup):
        sim.step()
    torch.cuda.synchronize()
    snap = ([t.clone() for t in sim.v], sim.s.clone(), sim.p.clone())
    sampler = ClockSampler(0)
    sampler.start()
    runs = {1: [], 2: []}
    for rnd in range(args.rounds):
        for passes in ((1, 2) if rnd % 2 == 0 else (2, 1)):
            for c in range(3):
                sim.v[c].copy_(snap[0][c])
            sim.s.copy_(snap[1])
            sim.p.copy_(snap[2])
            if passes == 2:
                os.environ['PHICUDA_CG_PASSES'] = '2'
            else:
                os.environ.pop('PHICUDA_CG_PASSES', None)
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s0.record()
            sim.ops.plume_step(sim.dom, sim.vbc, sim.sbc, sim.v, sim.s, sim.p, sim.inflow, bench.DT, bench.INFLOW_RATE, bench.BUOYANCY,
                               sim.prm, cg_events=ev)
            s1.record()
            torch.cuda.synchronize()
            info = ops.last_launch_info()
            assert info['passes'] == passes, info
            runs[passes].append({'cg_ms': ev[0].elapsed_time(ev[1]), 'step_ms': s0.elapsed_time(s1), 'iterations': int(res_dev[0].item()),
                                 'TY': info['TY'], 'stages': info['stages'], 'split': info['split'], 'grid_ctas': info['grid_ctas']})
    os.environ.pop('PHICUDA_CG_PASSES', None)
    clocks = sampler.summary()
    out = {'grid': n, 'rounds': args.rounds, 'gpu': clocks.get('gpu') or torch.cuda.get_device_name(0),
           'power_limit_w': clocks.get('power_limit_w'), 'sm_mhz_median': clocks.get('sm_mhz'), 'clock_reasons': clocks.get('reasons')}
    for passes, rs in runs.items():
        ms = np.array([r['cg_ms'] for r in rs])
        it = np.array([r['iterations'] for r in rs], float)
        t = ms * 1e-3
        out[f'{passes}_sweep'] = {
            'cg_ms_per_solve': {'median': float(np.median(ms)), 'min': float(ms.min()), 'max': float(ms.max())},
            'step_ms_median': float(np.median([r['step_ms'] for r in rs])),
            'iterations': sorted(set(int(i) for i in it)),
            'ms_per_iteration': float(np.median(ms / it)),
            'gbs_one_sweep_bytes': float(np.median(one_sweep_bytes(cells, it) / t / 1e9)),
            'gbs_at_30B': float(np.median(cells * (30.0 * it + 32.0) / t / 1e9)),
            'ring': {k: rs[0][k] for k in ('TY', 'stages', 'split', 'grid_ctas')}}
    out['speedup_cg_median'] = out['2_sweep']['cg_ms_per_solve']['median'] / out['1_sweep']['cg_ms_per_solve']['median']
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
