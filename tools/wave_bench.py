#!/usr/bin/env python
"""The wave step (phicuda_wave_f32) on one GPU.

    python tools/wave_bench.py [--frames 50] [--reps 5] [--out FILE]

1. The notebook's size (128 x 128, ZERO_GRADIENT, the moving disc): microseconds per frame of 16 substeps, the fused call
   (examples/waves.py `frame`: one launch, the 16 discs evaluated on the host) against the notebook's own cell on the mirror's field
   arithmetic (`--cell`: 16 cells of about a dozen launches and a host-built mask each), host clock around --frames frames ending in
   a device synchronise, median over --reps.
2. Large grids (4096^2 and 512^3, batch 1, periodic, a disc in every substep): milliseconds per substep of a 16-substep call through
   the C ABI (in place; CUDA events, median over --reps after a warm-up call) and the HBM rate at 12 B/cell per substep (h_c and h_p
   read, h_n written).  An even substep count, so the odd-count copy does not enter.
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
import waves as ex  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout
        return q.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name()


def notebook(frames, reps):
    h0 = ex.initial_state()
    out = {}
    for name, fn in (('fused', ex.frame), ('cell', lambda h, p, t: ex.iterate(ex.step, 1, h, p, t, substeps=ex.SUBSTEPS))):
        fn(h0, h0, 0)                          # warm-up
        times = []
        for _ in range(reps):
            state = (h0, h0, 0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(frames):
                state = fn(*state)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) / frames * 1e6)
        out[name] = float(np.median(times))
    return {'us_per_frame_fused': out['fused'], 'us_per_frame_cell': out['cell'], 'speedup': out['cell'] / out['fused']}


def large(res, reps, substeps=16):
    dom = _ops.Domain(res, (1.0,) * len(res), 1)
    gen = torch.Generator(device='cuda').manual_seed(0)
    hc = torch.rand(dom._shape(dom.cext), generator=gen, device='cuda')
    hp = torch.rand(dom._shape(dom.cext), generator=gen, device='cuda')
    lib = _lib.load()
    n = lib.phicuda_wave_scratch_bytes(C.byref(dom.grid), substeps)
    scratch = torch.empty(n // 4 + 1, dtype=torch.float32, device='cuda')
    bc = _ops.make_bc((('periodic', 'periodic'),) * len(res))
    table = (_lib.PhiWaveDisc * substeps)()
    for s, t in enumerate(table):
        t.present, t.value = 1, -0.5
        for a, r in enumerate(res):
            t.center[a] = r / 2 + r / 4 * np.cos(0.3 * s + a)
    centres = np.concatenate([np.arange(r, dtype=np.float32) + np.float32(0.5) for r in res])
    cp = centres.ctypes.data_as(C.POINTER(C.c_float))

    def call():
        _lib.check(lib.phicuda_wave_f32(C.byref(dom.grid), C.byref(bc), _ops._ptr(hc), _ops._ptr(hp), 1e-3, 1.0, 0.0, table, 64.0, cp,
                                        substeps, _ops._ptr(scratch), 4 * scratch.numel(), _ops._stream()))
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
    return {'res': list(res), 'ms_per_substep': ms, 'TBps_at_12B_per_cell': 12 * cells / (ms * 1e-3) / 1e12,
            'generic': info['generic'], 'TY': info['TY'], 'stages': info['stages'], 'grid_ctas': info['grid_ctas']}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=50)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    _ops.require_cuda()
    res = {'card': card(), 'notebook_128x128': notebook(a.frames, a.reps),
           'large': [large((4096, 4096), a.reps), large((512, 512, 512), a.reps)]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
