#!/usr/bin/env python
"""The Julia counts (phicuda_julia_f32, kernel k_julia) on one GPU.

    python tools/julia_bench.py [--reps 5] [--spot 4096] [--out FILE]

Times the kernel with CUDA events around one call through the C ABI (the host-to-device copy of the constants and centres included,
median over --reps after a warm-up call) at two sizes, both in Box(-2..2, -2..2) with 50 iterations and the notebook's constants
0.7885 exp(i t), t evenly spaced over [0, 2 pi]:
  notebook   256 x 256 x 100 constants
  large      4096 x 4096 x 128 constants (batch x cells = 2^31)
  wide       4096 x 4096 x 136 constants: count offsets beyond 2^31 (64-bit indexing)
Rates are in cell-iterations per second: batch x cells x iterations over the kernel time, counting the iterations that the early exit
skips as done.  The counts of the large and wide runs are checked against tests/oracle_julia.py at --spot seeded cells each, a
quarter of them in the last batch entries.  Prints one JSON object with the card's name and power limit and the k_julia row of
tools/sass_counts.py (static FP32 instruction count)."""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from phiflow_b200 import _lib, _ops  # noqa: E402
from oracle_julia import abs32, square_plus  # noqa: E402

ITERATIONS = 50


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def sass_row():
    """k_julia's row of tools/sass_counts.py as {column: count}."""
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'sass_counts.py')], capture_output=True, text=True)
    if out.returncode != 0:
        return {'error': out.stderr.strip()[-200:]}
    lines = out.stdout.splitlines()
    head = re.findall(r'\S+', lines[0])
    cols = head[1:head.index('kernel')]
    row = next(line for line in lines if line.rstrip().endswith('k_julia'))
    return dict(zip(cols, (int(v) for v in row.split()[:len(cols)])))


def setup(n, batch):
    dom = _ops.Domain((n, n), (4.0 / n,) * 2, batch)
    c = (np.float32(0.7885) * np.exp(1j * np.linspace(np.float32(0), np.float32(2 * np.pi), batch, dtype=np.float32))).astype(np.complex64)
    axis = np.linspace(np.float32(0.5 / n), np.float32(1 - 0.5 / n), n, dtype=np.float32) * np.float32(4) + np.float32(-2)
    return dom, c, np.concatenate([axis, axis])


def run(n, batch, reps):
    dom, c, centres = setup(n, batch)
    counts = torch.empty(dom._shape(dom.cext), dtype=torch.int32, device='cuda')
    lib = _lib.load()
    need = lib.phicuda_julia_scratch_bytes(C.byref(dom.grid))
    scratch = torch.empty(need, dtype=torch.uint8, device='cuda')
    pairs = c.view(np.float32)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))

    def call():
        _lib.check(lib.phicuda_julia_f32(C.byref(dom.grid), fp(centres), fp(pairs), ITERATIONS, _ops._ptr(counts), _ops._ptr(scratch),
                                         C.c_size_t(need), _ops._stream()))
    call()
    assert _ops.last_launch_info()['kernel'] == _lib.KERNEL_JULIA
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = float(np.median(times))
    work = float(batch) * n * n * ITERATIONS
    out = {'res': [n, n], 'batch': batch, 'iterations': ITERATIONS, 'ms': ms, 'ms_all': times, 'cell_iterations_per_s': work / (ms * 1e-3),
           'mean_count': float(counts[:, :, :n].float().mean())}
    return out, dom, c, centres, counts


def spot_check(dom, c, centres, counts, k, seed=0):
    """Counts at k seeded cells against the oracle, a quarter of them in the last batch entries; returns the number of mismatches."""
    n, batch = dom.res[0], dom.batch
    rng = np.random.default_rng(seed)
    b = np.concatenate([rng.integers(0, batch, k - k // 4), rng.integers(batch - max(batch // 8, 1), batch, k // 4)])
    x, y = rng.integers(0, n, k), rng.integers(0, n, k)
    a, im = centres[x].copy(), centres[n + y].copy()
    cr, ci = c.real[b].astype(np.float32), c.imag[b].astype(np.float32)
    want = np.zeros(k, np.int32)
    for _ in range(ITERATIONS):
        want += abs32(a, im) < np.float32(2)
        a, im = square_plus(a, im, cr, ci)
    flat = counts.view(-1)
    idx = torch.from_numpy((b.astype(np.int64) * dom.cext[1] + y) * dom.cext[0] + x).to(counts.device)
    got = flat[idx].cpu().numpy()
    return int((got != want).sum()), int((b.astype(np.int64) * dom.cext[1] * dom.cext[0] >= 2 ** 31).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--spot', type=int, default=4096)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    _ops.require_cuda()
    res = {'card': card()}
    res['notebook'], *_ = run(256, 100, a.reps)
    for name, batch in (('large', 128), ('wide', 136)):
        out, dom, c, centres, counts = run(4096, batch, a.reps)
        out['spot_mismatches'], out['spot_cells_beyond_2^31'] = spot_check(dom, c, centres, counts, a.spot)
        out['spot_cells'] = a.spot
        res[name] = out
        del counts
        torch.cuda.empty_cache()
    res['sass_k_julia'] = sass_row()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
