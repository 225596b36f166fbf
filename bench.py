#!/usr/bin/env python
"""
bench.py  --  512^3 smoke-plume steps/s on N H100s (BASELINE.json metric), laplace / CG / stencil HBM rooflines, CPU baseline.

    python bench.py --gpus N --steps K --warmup W            # our arm   (N>1: launched under torch.distributed.run)
    python bench.py --impl reference --steps K --warmup W    # reference arm: the oracle port on the host cores
    python bench.py --config c2|c3|c5 ...                    # the other BASELINE configs (extra modes, same JSON contract)
    python bench.py ... --dump-outputs DIR                   # also write the state after the last timed step as DIR/<name>.npy

One "step" = incompressible_step on the whole grid (SURVEY.md section 3.3 / 8d), ONE call of the product API
(phicuda_plume_step_f32 through phiflow_b200._ops.plume_step):
    s' = semi_lagrangian(s, v, dt) + inflow ; v* = semi_lagrangian(v, v, dt) + dt*buoyancy(s') ;
    v', p' = make_incompressible(v*, Solve('CG', 1e-3, x0=p))
Default workload = BASELINE.json configs[3] at N GPUs ("3-D smoke plume 512^3 fp32, periodic, z-slab decomposed"): strong
scaling.  Inputs are larger than L2 (every array is 512 MiB), so no L2 flush is needed between timed iterations.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "smoke_plume_512^3_steps_per_sec"
DT, INFLOW_RATE, BUOYANCY = 0.5, 0.2, (0.0, 0.0, 0.1)
RTOL, ATOL, MAX_ITER = 1e-3, 1e-5, 1000
PER3 = (('periodic', 'periodic'),) * 3
ZG3 = (('zg', 'zg'),) * 3


def load_peaks():
    path = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(path):
        return float(json.load(open(path))['hbm_gbs']), 'measured'
    return 3350.0, 'datasheet'           # H100 SXM HBM3


from phiflow_b200._clocks import ClockSampler  # noqa: E402


# ------------------------------------------------------------------------------------------------------------------
# reference arm / cpu_baseline: the oracle port (NumPy + SciPy CSR CG, i.e. what the reference's NumPy backend runs)
# ------------------------------------------------------------------------------------------------------------------
def cpu_plume(n: int, steps: int, warmup: int):
    """Times `steps` plume steps of the oracle port at n^3 after `warmup` untimed ones (time.perf_counter around the loop, the
    reference's own idiom: PhiML/phiml/math/_functional.py:1286-1294).  The matrix is built once, untimed, as the reference
    traces it once per shape."""
    from oracle import oracle_np as O
    res = (n, n, n)
    lower, upper = (0.0,) * 3, (100.0,) * 3
    dx = tuple(100.0 / n for _ in range(3))
    vbc, sbc = O.uniform_bc(3, O.PERIODIC), O.uniform_bc(3, O.ZG)
    inflow = O.sphere_soft_mask((50.0, 50.0, 9.5), 5.0, lower, upper, res)
    rng = np.random.default_rng(0)
    v = [(0.01 * rng.standard_normal(s)).astype(np.float32) for s in O.staggered_shapes(res, vbc)]
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    v, p, _ = O.make_incompressible(v, vbc, res, dx, RTOL, ATOL, MAX_ITER, matrix=A)
    p = np.zeros(res, np.float32)
    s = np.zeros(res, np.float32)
    iters, times = [], []
    for i in range(warmup + steps):
        t0 = time.perf_counter()
        v, s, p, info = O.plume_step(v, s, p, DT, vbc, sbc, lower, upper, res, inflow, INFLOW_RATE, BUOYANCY,
                                     rtol=RTOL, atol=ATOL, max_iter=MAX_ITER, matrix=A)
        if i >= warmup:
            times.append(time.perf_counter() - t0)
            iters.append(int(info['iterations']))
    return {"grid": n, "cells": n ** 3, "steps": steps, "warmup": warmup, "s_per_step": float(np.mean(times)),
            "cg_iterations_per_step": float(np.mean(iters))}


def reference_library_check(n: int = 64):
    """How the port compares with the reference LIBRARY itself, run live: where oracle/_ref holds the unmodified PhiML that
    `__graft_entry__.build()` installs, one pressure system of the plume at n^3 is solved by the oracle port's CG and by
    `phiml.backend.NUMPY.linear_solve('CG', ...)` (= PhiML/phiml/backend/_linalg.py:23-89, what the reference's NumPy path runs), and
    n^3 points are gathered by the port's grid_sample and by `phiml.math.grid_sample`.  Reports both times, the iteration counts and
    whether the results are identical - the evidence that timing the port does not flatter the GPU arm.  None when PhiML is absent."""
    ref_dir = os.path.join(ROOT, 'oracle', '_ref')
    if not os.path.isdir(os.path.join(ref_dir, 'phiml')):
        return None
    if ref_dir not in sys.path:
        sys.path.insert(0, ref_dir)
    import warnings
    from oracle import oracle_np as O
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from phiml import math
        from phiml.backend import NUMPY
        from phiml.math import spatial, instance, channel, extrapolation as E
        res = (n, n, n)
        dx = tuple(100.0 / n for _ in range(3))
        lower, upper = (0.0,) * 3, (100.0,) * 3
        vbc = O.uniform_bc(3, O.PERIODIC)
        A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
        blob = O.sphere_soft_mask((50.0, 50.0, 30.0), 20.0, lower, upper, res)
        v = [np.zeros(s, np.float32) for s in O.staggered_shapes(res, vbc)]
        v[2] += 0.05 * (blob + np.roll(blob, 1, 2))                      # buoyancy of a smoke blob, as in the plume
        y = O.divergence_staggered(v, dx, O.component_bcs(vbc, 3))
        y = (y - y.mean(dtype=np.float32)).astype(np.float32)
        t0 = time.perf_counter()
        port = O.cg(A, y, np.zeros(res, np.float32), RTOL, ATOL, MAX_ITER, None)
        t_port = time.perf_counter() - t0
        yy = y.reshape(1, -1)
        t0 = time.perf_counter()
        ref = NUMPY.linear_solve('CG', A, yy, np.zeros_like(yy), np.array([RTOL], np.float32), np.array([ATOL], np.float32),
                                 np.array([[MAX_ITER]]), None, None)
        t_ref = time.perf_counter() - t0
        rng = np.random.default_rng(0)
        pts = (rng.random((n ** 3, 3)) * (n + 2.0) - 1.0).astype(np.float32)
        g = rng.standard_normal(res).astype(np.float32)
        t0 = time.perf_counter()
        a = O.grid_sample(g, pts, O.uniform_bc(3, O.ZG))
        t_gs_port = time.perf_counter() - t0
        gt = math.tensor(g, spatial(x=n, y=n, z=n))
        ct = math.tensor(pts, instance(points=n ** 3) & channel(vector='x,y,z'))
        t0 = time.perf_counter()
        b = math.grid_sample(gt, ct, E.ZERO_GRADIENT).numpy('points')
        t_gs_ref = time.perf_counter() - t0
    return {"library": "PhiML 1.7.2 (unmodified, oracle/_ref), NumPy backend", "grid": n,
            "cg": {"port_s": t_port, "phiml_s": t_ref, "iterations_port": int(port['iterations']),
                   "iterations_phiml": int(np.asarray(ref.iterations)[0]),
                   "bitwise_equal": bool(np.array_equal(np.asarray(ref.x)[0], port['x'].reshape(-1)))},
            "grid_sample": {"points": n ** 3, "port_s": t_gs_port, "phiml_s": t_gs_ref, "max_abs_diff": float(np.abs(a - b).max())}}


def extrapolate(samples, full: int, it_full=None):
    """Fits  t_step = cells * (a + b * iterations)  to the measured samples and evaluates it at `full`^3 with `it_full` CG
    iterations per step (measured on the GPU for the same steps when known; otherwise iterations grow like n - condition
    number ~ n^2 for the Poisson matrix - from the largest sample, capped at max_iterations).  The stock NumPy path cannot
    run 512^3 (explicit CSR build ~200 GB, SURVEY.md section 6), so this number is an EXTRAPOLATION of measurements, never a
    measurement."""
    n = np.array([s['grid'] for s in samples], float)
    cells = n ** 3
    t = np.array([s['s_per_step'] for s in samples])
    it = np.array([s['cg_iterations_per_step'] for s in samples])
    how = "measured on the GPU for the same steps"
    if it_full is None:
        it_full = min(float(MAX_ITER), float(it[-1]) * full / n[-1])
        how = f"iterations ~ n from the {int(n[-1])}^3 sample, capped at max_iterations"
    if len(samples) >= 3:
        (a, b), *_ = np.linalg.lstsq(np.stack([cells, cells * it], 1), t, rcond=None)
        if a < 0 or b < 0:
            a, b = 0.0, float(np.sum(t) / np.sum(cells * np.maximum(it, 1)))
    else:
        a, b = 0.0, float(np.sum(t) / np.sum(cells * np.maximum(it, 1)))
    t_full = float(full) ** 3 * (a + b * it_full)
    law = f"t = cells*({a:.3e} + {b:.3e}*it) s; it({full}^3) = {it_full:.0f} ({how})"
    return t_full, it_full, law


def cpu_report(sizes, steps, warmup, full, it_full=None):
    # the first (smallest) grid runs the requested steps; larger grids are bounded samples: 2 steps after 1 warm-up below 200^3,
    # a single cold step above (minutes per step)
    samples = [cpu_plume(n, steps, warmup) if i == 0 else (cpu_plume(n, 2, 1) if n < 200 else cpu_plume(n, 1, 0)) for i, n in enumerate(sizes)]
    t_full, it_full, law = extrapolate(samples, full, it_full)
    return {"reference_library_check": reference_library_check(),
            "value": 1.0 / t_full, "unit": "steps/s", "cores": 1, "kind": "port", "extrapolated": True,
            "extrapolation": f"{law}; {t_full:.1f} s/step",
            "samples": samples,
            "sample": "the same plume on " + ", ".join(f"{s['grid']}^3 ({s['steps']} steps, {s['s_per_step']:.2f} s/step, {s['cg_iterations_per_step']:.0f} it)"
                                                       for s in samples)
                      + f"; NumPy/SciPy oracle port of the reference's NumPy path, single-threaded by construction ({os.cpu_count()} cores present); "
                        f"{full}^3 itself does not fit the stock path -> value is extrapolated"}


def run_reference(args):
    if int(os.environ.get('RANK', '0')) != 0:
        return
    sizes = [int(v) for v in str(args.cpu_sizes or args.cpu_size).split(',')]
    base = cpu_report(sizes, args.steps, args.warmup, args.size)
    line = {"impl": "reference", "metric": METRIC, "value": base["value"], "unit": "steps/s", "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 / base["value"], "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "extrapolated": True,
            "config": {"workload": f"3-D smoke plume {args.size}^3 fp32 periodic (BASELINE configs[3])", "sample_grids": sizes,
                       "note": "steps/warmup apply to the first sample grid; larger grids run 1-2 steps; value = fitted law evaluated at the full grid"},
            "cpu_baseline": base,
            "e2e": {"value": base["value"], "unit": "steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


# ------------------------------------------------------------------------------------------------------------------
# our arm, one GPU
# ------------------------------------------------------------------------------------------------------------------
class PlumeSim:
    """Device-resident plume state; step() is ONE call of the product API (phicuda_plume_step_f32)."""

    def __init__(self, n, device):
        import torch
        from phiflow_b200 import _ops as ops
        self.torch, self.ops = torch, ops
        self.n = n
        self.vbc, self.sbc = PER3, ZG3
        dx = tuple(100.0 / n for _ in range(3))
        self.dom = ops.Domain((n, n, n), dx, 1, vbc=self.vbc, device=device)
        g = torch.Generator().manual_seed(0)
        self.v = []
        for c in range(3):
            host = torch.randn((1, n, n, n), generator=g, dtype=torch.float32).mul_(0.01).pin_memory()
            self.v.append(host.to(device, non_blocking=True))
        self.s, self.p = self.dom.alloc_centered(), self.dom.alloc_centered()
        # inflow mask (set-up, not per-step compute): soft sphere, phi/geom/_geom.py:278-308
        ax = (torch.arange(n, device=device, dtype=torch.float32) + 0.5) * dx[0]
        z, y, x = torch.meshgrid(ax, ax, ax, indexing='ij')
        dist = torch.sqrt(torch.clamp((x - 50.0) ** 2 + (y - 50.0) ** 2 + (z - 9.5) ** 2, min=1e-6))
        cell_r = float(np.sqrt(3 * (dx[0] * 0.5) ** 2))
        self.inflow = torch.clamp(0.5 - (dist - 5.0) / cell_r, 0, 1).reshape(1, n, n, n).contiguous()
        del x, y, z, dist
        self.prm = ops.cg_params(self.vbc, rtol=RTOL, atol=ATOL, max_iter=MAX_ITER)
        ops.make_incompressible(self.dom, self.vbc, self.v, self.p, self.prm)
        self.p.zero_()
        self.dom.scratch()
        self.launches_per_step = 5            # advect s (+inflow), advect v (+buoyancy), divergence, CG, grad_sub (+ 1 device copy)
        self.cg_events = []

    def step(self, time_cg=False):
        ev = None
        if time_cg:
            ev = (self.torch.cuda.Event(enable_timing=True), self.torch.cuda.Event(enable_timing=True))
            self.cg_events.append(ev)
        self.ops.plume_step(self.dom, self.vbc, self.sbc, self.v, self.s, self.p, self.inflow, DT, INFLOW_RATE, BUOYANCY, self.prm,
                            cg_events=ev)


def time_kernel(torch, fn, reps=10, warm=2):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_rooflines(sim, torch, ops, peak):
    """Per-kernel HBM roofline of the non-CG kernels on the live plume state (after the timed steps), algorithmic bytes per cell
    from SURVEY.md section 8d: divergence 16, grad_sub 28, semi-Lagrangian 20 per advected scalar / component."""
    dom, n = sim.dom, sim.n
    cells = float(n) ** 3
    out = {}
    x = torch.randn((1, n, n, n), device=sim.s.device, dtype=torch.float32)
    y = torch.empty_like(x)
    v2 = dom.alloc_faces()
    ms = time_kernel(torch, lambda: ops.laplace(dom, PER3, x, out=y), reps=20, warm=3)
    out['laplace'] = (ms, 8.0)
    out['divergence'] = (time_kernel(torch, lambda: ops.divergence(dom, sim.vbc, sim.v, out=y)), 16.0)
    ms = time_kernel(torch, lambda: ops.grad_sub(dom, sim.vbc, v2, x))
    out['grad_sub'] = (ms, 28.0)
    out['advect_centered'] = (time_kernel(torch, lambda: ops.advect_centered(dom, sim.vbc, sim.v, sim.sbc, sim.s, DT, out=y)), 20.0)
    out['advect_staggered_3comp'] = (time_kernel(torch, lambda: ops.advect_staggered(dom, sim.vbc, sim.v, sim.vbc, sim.v, DT, out=v2)), 60.0)
    del x, y, v2
    return {k: {"ms": ms, "achieved": b * cells / (ms * 1e-3) / 1e9, "peak": peak, "frac": b * cells / (ms * 1e-3) / 1e9 / peak,
                "unit": "GB/s", "algorithmic_bytes": f"{b:g} B/cell"} for k, (ms, b) in out.items()}


def run_ours(args):
    import torch
    from phiflow_b200 import _ops as ops
    if args.gpus > 1 or int(os.environ.get('WORLD_SIZE', '1')) > 1:
        from phiflow_b200 import dist_bench
        return dist_bench.run(args, METRIC)
    torch.cuda.set_device(0)
    dev = torch.device('cuda:0')
    n = args.size
    peak, peak_kind = load_peaks()
    sim = PlumeSim(n, dev)
    cells = float(n) ** 3
    _, res_dev = sim.dom.workspace()
    res_host = torch.zeros((args.warmup + args.steps, 6), dtype=torch.int32).pin_memory()

    for i in range(args.warmup):
        sim.step()
        res_host[i].copy_(res_dev[:6], non_blocking=True)
    torch.cuda.synchronize()
    # the e2e leg replays ALL timed steps from this state, so both legs do the same work
    host = ops.HostPlume(sim.dom, sim.vbc, sim.sbc)
    host.load(sim.v, sim.s, sim.p)
    sampler = ClockSampler(0)
    sampler.start()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for i in range(args.steps):
        sim.step(time_cg=True)
        res_host[args.warmup + i].copy_(res_dev[:6], non_blocking=True)
    end.record()
    torch.cuda.synchronize()
    clocks = sampler.summary()
    ms = start.elapsed_time(end) / args.steps
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {'velocity_x': sim.v[0], 'velocity_y': sim.v[1], 'velocity_z': sim.v[2], 'smoke': sim.s,
                                         'pressure': sim.p}, {'cg_iterations': res_host[-1:, 0]}, torch)
    iters = res_host[args.warmup:, 0].numpy().astype(np.int64)
    cg_ms = np.array([a.elapsed_time(b) for a, b in sim.cg_events])
    # algorithmic bytes of one solve: 30 B/cell/iteration (pass A 12 + pass B 12 / 24 alternating: the x update is applied
    # every second iteration) + 32 B/cell of setup/teardown passes
    cg_bytes = cells * (30.0 * iters + 32.0)
    cg_gbs = float(np.sum(cg_bytes) / np.sum(cg_ms * 1e-3) / 1e9)
    variant = ops.last_launch_info()

    kernels = kernel_rooflines(sim, torch, ops, peak)

    # end to end through the host-facing form of the same call: state in pinned HOST arrays in the reference's (x, y, z) order
    e2e = run_e2e(sim, host, args, torch)
    del host

    base = cpu_report([int(v) for v in str(args.cpu_sizes or args.cpu_size).split(',')], 2, 1, n, float(np.mean(iters))) if not args.no_cpu else None
    workload = {512: "BASELINE configs[3] at 1 GPU", 256: "BASELINE configs[1]"}.get(n, "reduced grid, NOT a BASELINE config")
    lap = kernels.pop('laplace')
    line = {"metric": METRIC if n == 512 else f"smoke_plume_{n}^3_steps_per_sec", "value": 1e3 / ms, "unit": "steps/s", "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms, "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic",
            "config": {"workload": f"3-D smoke plume {n}^3 fp32 periodic, CG rtol=1e-3 warm start ({workload})",
                       "api": "one phicuda_plume_step_f32 call per step (5 kernel launches + 1 device copy)",
                       "cg_iterations_per_step": float(np.mean(iters)), "cg_ms_per_step": float(np.mean(cg_ms)),
                       "non_cg_ms_per_step": float(ms - np.mean(cg_ms)),
                       "cg_kernel_variant": {k: variant[k] for k in ('kernel', 'generic', 'TY', 'stages', 'ZC', 'nzc', 'groups', 'total_units', 'grid_ctas', 'split')},
                       "l2": f"inputs ({4 * n ** 3 / 2 ** 20:.0f} MiB per array) exceed L2, no flush"},
            "clocks": clocks, "gpu_launches": sim.launches_per_step * args.steps,
            "roofline": {"bound": "hbm", "kernel": "k_cg_ring<3,GENERIC=false,DIST=false> (persistent CG solve)", "achieved": cg_gbs, "peak": peak, "unit": "GB/s",
                         "frac": cg_gbs / peak, "traffic": None, "peak_kind": peak_kind,
                         "algorithmic_bytes": "cells*(30*iterations+32) per solve"},
            "laplace": lap, "kernels": kernels,
            "e2e": e2e}
    if base:
        line["cpu_baseline"] = base
    print(json.dumps(line))


# at most 2^21 values per array (8 MiB in float32): five arrays of the 512^3 plume stay far below 64 MB
DUMP_SAMPLE = 1 << 21


def dump_outputs(out_dir, device_arrays, host_arrays, torch):
    """Writes what the timed path left behind as out_dir/<name>.npy: arrays of at most DUMP_SAMPLE values whole (device layout,
    batch first), larger ones as the flattened device array at DUMP_SAMPLE positions drawn from a fixed seed, so that two builds
    run with the same arguments can be compared value by value."""
    os.makedirs(out_dir, exist_ok=True)
    for name, t in device_arrays.items():
        if t.numel() > DUMP_SAMPLE:
            idx = torch.randint(t.numel(), (DUMP_SAMPLE,), generator=torch.Generator().manual_seed(t.numel()))
            t = t.reshape(-1)[idx.sort().values.to(t.device)]
        np.save(os.path.join(out_dir, f'{name}.npy'), t.float().cpu().numpy())
    for name, a in host_arrays.items():
        np.save(os.path.join(out_dir, f'{name}.npy'), np.asarray(a, np.float64))


def run_e2e(sim, host, args, torch):
    steps = args.steps
    _, res_dev = sim.dom.workspace()
    snap = ([t.clone() for t in host.v], host.s.clone(), host.p.clone())
    host.step(sim.inflow, DT, INFLOW_RATE, BUOYANCY, sim.prm)      # untimed warm-up of the copy path, then back to the start state
    torch.cuda.synchronize()
    for c in range(3):
        host.v[c].copy_(snap[0][c])
    host.s.copy_(snap[1]); host.p.copy_(snap[2])
    del snap
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    its = []
    torch.cuda.synchronize()
    t0.record()
    for _ in range(steps):
        host.step(sim.inflow, DT, INFLOW_RATE, BUOYANCY, sim.prm)
        its.append(res_dev[:1].clone())
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / steps
    return {"value": 1e3 / ms, "unit": "steps/s", "h2d_bytes_per_step": host.bytes_per_direction, "d2h_bytes_per_step": host.bytes_per_direction,
            "steps": steps, "cg_iterations_per_step": float(torch.cat(its).float().mean().item()),
            "note": "the same timed steps replayed from their start state with the full state (v, s, p) in pinned host arrays in the "
                    "reference's (x,y,z) order: upload + transpose + phicuda_plume_step_f32 + transpose + download every step"}


# ------------------------------------------------------------------------------------------------------------------
# extra modes: BASELINE configs[2] (Taylor-Green 512^3) and configs[4] (batched 2-D Kolmogorov, batch-sharded)
# ------------------------------------------------------------------------------------------------------------------
def run_c3(args):
    """configs[2]: 3-D Taylor-Green vortex, periodic [0, 2 pi]^3, dt = 0.5 dx, 100 steps of semi_lagrangian -> make_incompressible
    (SURVEY.md section 8d).  Gates: max|div v| <= 5e-5 * max|v| / dx after every projection; kinetic energy reported per 10 steps.
    The oracle comparison of this configuration (advection parity on step 1, energy within 1e-3 of the oracle) is a -m gpu test at
    32^3 / 64^3 (tests/test_gpu_kernels.py::test_config_c3_taylor_green_3d) - the oracle needs minutes per step at 128^3."""
    import torch
    from phiflow_b200 import _ops as ops
    torch.cuda.set_device(0)
    dev = torch.device('cuda:0')
    n = args.size
    L = 2 * np.pi
    dx = (L / n,) * 3
    dom = ops.Domain((n, n, n), dx, 1, vbc=PER3, device=dev)
    c = (torch.arange(n, device=dev, dtype=torch.float32) + 0.5) * dx[0]           # cell centres
    f = torch.arange(n, device=dev, dtype=torch.float32) * dx[0]                   # lower faces
    v = dom.alloc_faces()
    zz, yy, xx = torch.meshgrid(c, c, f, indexing='ij')
    v[0][0] = torch.sin(xx) * torch.cos(yy) * torch.cos(zz)
    zz, yy, xx = torch.meshgrid(c, f, c, indexing='ij')
    v[1][0] = -torch.cos(xx) * torch.sin(yy) * torch.cos(zz)
    del xx, yy, zz
    v2 = dom.alloc_faces()
    p = dom.alloc_centered()
    prm = ops.cg_params(PER3, rtol=RTOL, atol=ATOL, max_iter=MAX_ITER)
    dt = 0.5 * dx[0]
    div = dom.alloc_centered()

    def step():
        nonlocal v, v2
        ops.advect_staggered(dom, PER3, v, PER3, v, dt, out=v2)
        v, v2 = v2, v
        ops.make_incompressible(dom, PER3, v, p, prm)

    energies, worst = [], 0.0
    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(args.steps):
        step()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.steps
    # gates, outside the timed region: a second pass over the same number of steps would change the state, so check the final state
    ops.divergence(dom, PER3, v, out=div)
    vmax = max(float(t.abs().max()) for t in v)
    dmax = float(div.abs().max())
    ke = 0.5 * sum(float((t.double() ** 2).sum()) for t in v) / float(n) ** 3
    gate = 5e-5 * vmax / dx[0]
    # at rtol 1e-3 the divergence left after a projection is bounded by the solver tolerance, not by 5e-5 (that gate is for a
    # converged 1e-5 solve): report both
    line = {"metric": f"taylor_green_{n}^3_steps_per_sec", "value": 1e3 / ms, "unit": "steps/s", "n_gpus": 1, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic",
            "config": {"workload": f"3-D Taylor-Green vortex {n}^3 fp32 periodic, dt = 0.5 dx, semi_lagrangian + make_incompressible(CG 1e-3) "
                                   f"(BASELINE configs[2])", "max_abs_div": dmax, "div_gate_5e-5_vmax_over_dx": gate, "div_gate_passed": dmax <= gate,
                       "kinetic_energy_per_cell": ke, "initial_kinetic_energy_per_cell": 0.125, "max_abs_v": vmax,
                       "cg_iterations_last_step": int(ops.read_results(dom)['iterations'][0])},
            "gpu_launches": 4 * args.steps}
    print(json.dumps(line))


def run_c5(args):
    """configs[4]: batched 2-D Kolmogorov flow, 64 entries of 256^2 per GPU (512 on 8 GPUs), batch-sharded: entries are
    independent systems (PhiML/phiml/backend/_linalg.py:72-87), so there is NO collective in the loop - only the timing barrier.
    Step = forced step of the product API: v* = semi_lagrangian(v, v, dt) + dt * resample(f * (1, 0), to=v), f = sin(4y);
    v = make_incompressible(v*, Solve('CG', 1e-3, x0=p)).  Weak scaling (fixed work per GPU)."""
    import torch
    import torch.distributed as dist
    from phiflow_b200 import _ops as ops
    from phiflow_b200.dist import batch_shard
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    n, per_gpu = args.size if args.size != 512 else 256, args.batch
    first, count = batch_shard(per_gpu * world, rank, world)
    L = 2 * np.pi
    dx = (L / n, L / n)
    per2 = (('periodic', 'periodic'),) * 2
    dom = ops.Domain((n, n), dx, count, vbc=per2, device=dev)
    v = dom.alloc_faces()
    for b in range(count):                                      # seed = global batch index (SURVEY.md section 8d)
        g = torch.Generator().manual_seed(first + b)
        for c in range(2):
            v[c][b] = torch.randn((n, n), generator=g, dtype=torch.float32).mul_(0.01).to(dev)
    yc = (torch.arange(n, device=dev, dtype=torch.float32) + 0.5) * dx[1]
    force = dom.alloc_centered()
    force[:] = torch.sin(4 * yc)[None, :, None]
    p = dom.alloc_centered()
    prm = ops.cg_params(per2, rtol=RTOL, atol=ATOL, max_iter=MAX_ITER)
    ops.make_incompressible(dom, per2, v, p, prm)
    p.zero_()
    dt = 0.05
    evs = []

    def step(timed=False):
        ev = None
        if timed:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            evs.append(ev)
        ops.plume_step(dom, per2, per2, v, force, p, None, dt, 0.0, (1.0, 0.0), prm, static_scalar=True, cg_events=ev)

    _, res_dev = dom.workspace()
    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
        torch.cuda.synchronize()
    its = []
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.steps):
        step(True)
        its.append(res_dev.view(-1, 6)[:, 0].clone())
    t1.record()
    torch.cuda.synchronize()
    clocks = sampler.summary() if sampler else None
    if world > 1:
        dist.barrier()
        torch.cuda.synchronize()
    ms_t = torch.tensor([t0.elapsed_time(t1)], device=dev, dtype=torch.float64)
    cg_t = torch.tensor([float(np.sum([a.elapsed_time(b) for a, b in evs]))], device=dev, dtype=torch.float64)
    it_t = torch.stack(its).double()                            # [steps, batch]
    it_sum = it_t.max(dim=1).values.sum().reshape(1)            # the kernel runs until the slowest entry of the rank converges
    it_mean = it_t.mean().reshape(1)
    if world > 1:
        dist.all_reduce(ms_t, op=dist.ReduceOp.MAX)
        dist.all_reduce(cg_t, op=dist.ReduceOp.MAX)
        dist.all_reduce(it_mean, op=dist.ReduceOp.SUM)
        it_mean /= world
    if rank == 0:
        peak, peak_kind = load_peaks()
        ms = float(ms_t.item()) / args.steps
        cells = float(n * n * count)
        # every entry runs its own iteration count; bytes counted for the iterations each entry actually ran
        cg_bytes = float((cells / count) * (30.0 * it_t.sum().item() + 32.0 * count * args.steps))
        cg_gbs = cg_bytes / (float(cg_t.item()) * 1e-3) / 1e9
        line = {"metric": "kolmogorov_2d_batched_steps_per_sec", "value": 1e3 / ms, "unit": "steps/s", "n_gpus": world, "steps": args.steps,
                "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
                "data": "synthetic",
                "config": {"workload": f"batched 2-D Kolmogorov flow, batch {per_gpu * world} x {n}^2 fp32 periodic, {count} entries per GPU, forcing sin(4y), "
                                       f"dt 0.05, CG rtol=1e-3 warm start (BASELINE configs[4])",
                           "entry_steps_per_sec": per_gpu * world * 1e3 / ms, "cg_iterations_per_entry_step": float(it_mean.item()),
                           "cg_ms_per_step": float(cg_t.item()) / args.steps, "collectives_in_loop": 0,
                           "l2": f"working set {7 * cells * 4 / 2 ** 20:.0f} MiB per GPU against 50 MB of L2: the HBM roofline fraction below "
                                 f"is reported against HBM peak although part of the traffic is served by L2; no flush between steps by design "
                                 f"(the workload IS a resident batch)"},
                "clocks": clocks, "gpu_launches": 4 * args.steps * world,
                "roofline": {"bound": "hbm", "kernel": "k_cg_ring<2> (persistent CG, 64 systems per launch)", "achieved": cg_gbs, "peak": peak,
                             "unit": "GB/s", "frac": cg_gbs / peak, "traffic": None, "peak_kind": peak_kind,
                             "algorithmic_bytes": "cells*(30*iterations+32) per entry and solve, rank 0"}}
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', default='ours')
    ap.add_argument('--config', default='plume', choices=['plume', 'c2', 'c3', 'c4', 'c5'],
                    help='plume/c4: 512^3 smoke plume (default, BASELINE configs[3]); c2: 256^3 plume; c3: 512^3 Taylor-Green; c5: batched 2-D Kolmogorov')
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--batch', type=int, default=64, help='c5: batch entries per GPU')
    ap.add_argument('--cpu-size', type=int, default=96, dest='cpu_size')
    ap.add_argument('--cpu-sizes', default=None, dest='cpu_sizes', help='comma-separated sample grids of the CPU baseline (default: 96,128; add 256 for a ~6-minute third sample)')
    ap.add_argument('--no-cpu', action='store_true', dest='no_cpu')
    ap.add_argument('--halo', type=int, default=16, help='z-slab halo planes allocated per side (N>1); grows on demand')
    ap.add_argument('--dump-outputs', default=None, dest='dump_outputs', metavar='DIR',
                    help='plume on one GPU: write velocity, smoke, pressure (a seeded sample of large arrays) and the CG iteration count '
                         'of the last timed step as DIR/<name>.npy')
    args = ap.parse_args()
    if args.dump_outputs and (args.impl != 'ours' or args.config not in ('plume', 'c2', 'c4') or args.gpus > 1):
        ap.error('--dump-outputs applies to the plume on one GPU')
    if args.config == 'c2':
        args.size = 256
    if args.impl == 'reference':
        if args.cpu_sizes is None and args.cpu_size == 96:
            args.cpu_sizes = '96,128'          # 256^3 takes ~5 min per step: opt in with --cpu-sizes 96,128,256
        return run_reference(args)
    args.warmup = max(args.warmup, 3)
    if args.cpu_sizes is None and args.cpu_size == 96:
        args.cpu_sizes = '96,128'
    if args.config == 'c3':
        return run_c3(args)
    if args.config == 'c5':
        return run_c5(args)
    run_ours(args)


if __name__ == '__main__':
    main()
