#!/usr/bin/env python
"""The notebook step with static obstacles: ONE call (fluid.incompressible_step(..., obstacles=)) next to the sequenced mirror cells
(advect -> + inflow -> resample(s * b, to=v) -> semi_lagrangian -> + buoyancy -> make_incompressible(v, obstacle, Solve(x0=p))), one GPU.

    python tools/plume_obstacle_bench.py [--steps 10] [--warmup 3] [--rounds 3] [--only NAME]

Arms, alternated round by round in one process from the same state:
  one_call        fluid.incompressible_step(..., obstacles=geometry): phicuda_plume_step_masked_f32
  sequenced       the mirror cells as examples/batched_smoke_obstacle.py writes them; the obstacle masks come from the memo
  sequenced_raster the same with the memo emptied before every step: make_incompressible rasterises the geometry on the host every
                  step, as it did before the memo
ms/step: host clock around each step, which ends in a device synchronise (the mirror reads the solve records to raise NotConverged).
CG ms: CUDA events the library records around the pressure solve of the one-call step (PhiPlumeParams cg events), the same solve in
every arm (fused == sequenced bit for bit); non-CG ms = ms/step - CG ms.  Solves run with suppress=(NotConverged,): a step's cost,
not a convergence test.  Workloads: Batched_Smoke 256^2 batch 3, Fluid_Logo 128^2 and 1024^2, the Wake_Flow geometry 512 x 256 x 64
(the one-call arm advects a zero smoke field there; the notebook has none).
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from phiflow_b200 import _ops as ops  # noqa: E402
from phiflow_b200._clocks import ClockSampler  # noqa: E402
import phiflow_b200.flow as F  # noqa: E402


def batched_smoke(res=256):
    dom = F.Box(x=100, y=100)
    masks = np.stack([r * F.resample(F.Sphere(x=cx, y=9.5, radius=5), to=F.CenteredGrid(0, F.ZERO_GRADIENT, dom, x=res, y=res), soft=True).numpy()
                      for r, cx in zip((.1, .2, .3), (40, 50, 60))])
    return dict(v=F.StaggeredGrid(0, 0, dom, batch=3, x=res, y=res), s=F.CenteredGrid(0, F.ZERO_GRADIENT, dom, batch=3, x=res, y=res),
                inflow=F.CenteredGrid(masks, F.ZERO_GRADIENT, dom, batch=3, x=res, y=res), obstacle=F.Box(x=(35, 65), y=(50, 70)),
                buoyancy=(0, 0.1), solve=lambda p: F.Solve(x0=p, suppress=(F.NotConverged,)), advection='mac_cormack')


def fluid_logo(res):
    domain = dict(x=res, y=res, bounds=F.Box(x=100, y=100))
    geometry = F.union([F.Box(x=(15 + x * 7, 15 + (x + 1) * 7), y=(41, 83)) for x in range(1, 10, 2)]
                       + [F.Box(x=(43, 50), y=(41, 48)), F.Box(x=(15, 43), y=(83, 90)), F.Box(x=(50, 85), y=(83, 90))])
    inflow = F.CenteredGrid(F.Box(x=(14, 21), y=(6, 10)), F.ZERO_GRADIENT, **domain) + \
        F.CenteredGrid(F.Box(x=(81, 88), y=(6, 10)), F.ZERO_GRADIENT, **domain) * 0.9 + \
        F.CenteredGrid(F.Box(x=(44, 47), y=(49, 51)), F.ZERO_GRADIENT, **domain) * 0.4
    return dict(v=F.StaggeredGrid(0, 0, **domain), s=F.CenteredGrid(0, F.ZERO_GRADIENT, **domain), inflow=inflow, obstacle=geometry,
                buoyancy=(0, 0.1), solve=lambda p: F.Solve('CG-adaptive', 1e-5, x0=p, suppress=(F.NotConverged,)), advection='semi_lagrangian')


def wake_flow():
    b = {'x-': F.vec(x=2, y=0, z=0), 'x+': F.ZERO_GRADIENT, 'y': F.PERIODIC, 'z': F.PERIODIC}
    g = dict(x=512, y=256, z=64, bounds=F.Box(x=200, y=100, z=5))
    return dict(v=F.StaggeredGrid((8., 0, 0), b, **g), s=F.CenteredGrid(0, F.ZERO_GRADIENT, **g), inflow=None,
                obstacle=F.geom.infinite_cylinder(x=20, y=50, radius=10, inf_dim='z'), buoyancy=(0, 0, 0),
                solve=lambda p: F.Solve(x0=p, suppress=(F.NotConverged,)), advection=None)


WORKLOADS = {'batched_smoke_256x3': batched_smoke, 'fluid_logo_128': lambda: fluid_logo(128), 'fluid_logo_1024': lambda: fluid_logo(1024),
             'wake_flow_512x256x64': wake_flow}


def one_call(w, v, s, p):
    return F.fluid.incompressible_step(v, s, p, 1.0, inflow=w['inflow'], inflow_rate=1.0, buoyancy=w['buoyancy'], solve=w['solve'](p),
                                       smoke_advection=w['advection'] or 'semi_lagrangian', obstacles=w['obstacle'])


def sequenced(w, v, s, p, raster=False):
    if raster:
        F._MASKS.clear()
    if w['advection'] is not None:
        adv = F.advect.mac_cormack if w['advection'] == 'mac_cormack' else F.advect.semi_lagrangian
        s = adv(s, v, 1.0) + w['inflow']
        buoy = F.resample(s * w['buoyancy'], to=v)
        v = F.advect.semi_lagrangian(v, v, 1.0) + buoy * 1.0
    else:
        v = F.advect.semi_lagrangian(v, v, 1.0)
    v, p = F.fluid.make_incompressible(v, w['obstacle'], w['solve'](p))
    return v, s, p


def cg_ms(w, v, s, p, n):
    """CG time of the one-call step from the library's events, n steps from the given state."""
    kw = {}
    kw['accessible'], kw['factors'] = F._obstacle_masks_cached(v, w['obstacle'])
    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
    vd, sd, pd = [c.clone() for c in v.data], s.data.clone(), (p.data.clone() if p is not None else v.dom.alloc_centered())
    prm = F._cg_params(v, w['solve'](None))
    out = []
    for _ in range(n):
        ops.plume_step(v.dom, v.vspec, s.spec, vd, sd, pd, w['inflow'].data if w['inflow'] is not None else None, 1.0, 1.0, w['buoyancy'],
                       prm, mac_cormack=w['advection'] == 'mac_cormack', cg_events=ev, **kw)
        torch.cuda.synchronize()
        out.append(ev[0].elapsed_time(ev[1]))
    return out, ops.read_results(v.dom)['iterations'].tolist()


def run(name, steps, warmup, rounds):
    w = WORKLOADS[name]()
    v, s, p = w['v'], w['s'], None
    for _ in range(warmup):                           # a developed flow, and every shape warmed in every arm
        v, s, p = one_call(w, v, s, p)
        sequenced(w, v, s, p)
        sequenced(w, v, s, p, raster=True)
    arms = {'one_call': lambda st: one_call(w, *st), 'sequenced': lambda st: sequenced(w, *st),
            'sequenced_raster': lambda st: sequenced(w, *st, raster=True)}
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            st = (v, s, p)
            torch.cuda.synchronize()
            for _ in range(steps):
                t0 = time.perf_counter()
                st = fn(st)
                torch.cuda.synchronize()
                times[k].append(1e3 * (time.perf_counter() - t0))
    cg, its = cg_ms(w, v, s, p, steps)
    cg_med = float(np.median(cg))
    row = {'workload': name, 'steps_per_arm': steps * rounds, 'cg_ms_median': round(cg_med, 3), 'cg_iterations_last': its}
    for k, ts in times.items():
        med = float(np.median(ts))
        row[k] = {'ms_per_step_median': round(med, 3), 'ms_per_step_min': round(float(np.min(ts)), 3), 'non_cg_ms': round(med - cg_med, 3)}
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--only', default=None, choices=sorted(WORKLOADS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA device')
    sampler = ClockSampler(0)
    sampler.start()
    rows = [run(n, args.steps, args.warmup, args.rounds) for n in WORKLOADS if args.only in (None, n)]
    clocks = sampler.summary()
    print(json.dumps({'gpu': clocks.get('gpu') or torch.cuda.get_device_name(0), 'power_limit_w': clocks.get('power_limit_w'),
                      'sm_mhz_median': clocks.get('sm_mhz'), 'clock_reasons': clocks.get('reasons'), 'rows': rows}, indent=1))


if __name__ == '__main__':
    main()
