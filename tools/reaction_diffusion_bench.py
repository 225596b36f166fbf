#!/usr/bin/env python
"""Reaction-diffusion (phicuda_reaction_diffusion_f32) on one GPU.

    python tools/reaction_diffusion_bench.py [--frames 50] [--reps 5] [--out FILE]

1. The notebook's size (100 x 100, batch 3, maze parameters, ZERO boundary): microseconds per frame of 20 substeps, the fused call
   (flow.reaction_diffusion(..., substeps=20): one launch) against the notebook's own cell on the mirror's field arithmetic (20 cells of
   about 20 launches each), host clock around --frames frames ending in a device synchronise, median over --reps.
2. Large grids (4096^2 and 512^3, batch 1, periodic): milliseconds per substep of a 20-substep call through the C ABI (in place, no
   copies; CUDA events, median over --reps after a warm-up call) and the HBM rate at 16 B/cell per substep (u, v read, u', v' written).
Prints one JSON object with the card's name and power limit."""
import argparse
import ctypes as C
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
from phiflow_b200 import _lib, _ops  # noqa: E402
import phiflow_b200.flow as flow  # noqa: E402
import reaction_diffusion as ex  # noqa: E402

MAZE = ex.PARAMS['maze']


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout
        return q.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name()


def notebook(frames, reps):
    u0 = ex.initial_state()
    out = {}
    for name, fn in (('fused', lambda u, v: flow.reaction_diffusion(u, v, dt=.5, substeps=20, **MAZE)),
                     ('mirror_ops', lambda u, v: ex.iterate(ex.reaction_diffusion_cell, 1, u, v, dt=.5, substeps=20, f_kwargs=MAZE))):
        u, v = fn(u0, u0)                      # warm-up
        times = []
        for _ in range(reps):
            u, v = u0, u0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(frames):
                u, v = fn(u, v)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) / frames * 1e6)
        out[name] = float(np.median(times))
    return {'us_per_frame_fused': out['fused'], 'us_per_frame_mirror_ops': out['mirror_ops'],
            'speedup': out['mirror_ops'] / out['fused']}


def large(res, reps, substeps=20):
    dom = _ops.Domain(res, (1.0,) * len(res), 1)
    gen = torch.Generator(device='cuda').manual_seed(0)
    u = torch.rand(dom._shape(dom.cext), generator=gen, device='cuda')
    v = torch.rand(dom._shape(dom.cext), generator=gen, device='cuda') * 0.4
    lib = _lib.load()
    n = lib.phicuda_reaction_diffusion_scratch_bytes(C.byref(dom.grid))
    scratch = torch.empty(n // 4, dtype=torch.float32, device='cuda')
    vbc = _ops.make_vbc((('periodic', 'periodic'),) * len(res), 2)

    def call():
        _lib.check(lib.phicuda_reaction_diffusion_f32(C.byref(dom.grid), C.byref(vbc), _ops._ptr(u), _ops._ptr(v), MAZE['du'], MAZE['dv'],
                                                      MAZE['f'], MAZE['k'], 0.5, substeps, _ops._ptr(scratch), n, _ops._stream()))
    call()
    info = _ops.last_launch_info()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / substeps)
    ms = float(np.median(times))
    cells = float(np.prod(res))
    return {'res': list(res), 'ms_per_substep': ms, 'TBps_at_16B_per_cell': 16 * cells / (ms * 1e-3) / 1e12,
            'generic': info['generic'], 'TY': info['TY'], 'stages': info['stages'], 'grid_ctas': info['grid_ctas']}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=50)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    _ops.require_cuda()
    res = {'card': card(), 'notebook_100x100_batch3': notebook(a.frames, a.reps),
           'large': [large((4096, 4096), a.reps), large((512, 512, 512), a.reps)]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
