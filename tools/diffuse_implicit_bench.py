#!/usr/bin/env python
"""Implicit diffusion (phicuda_diffuse_implicit_f32) on one GPU, next to the two-sweep pressure CG of the same run.

    python tools/diffuse_implicit_bench.py [--size 512] [--stag-size 256] [--reps 3]

Cases: a size^3 periodic scalar field and a size^3 field with Heat_Flow-like boundaries (x-: 1, x+: ZERO_GRADIENT, y, z periodic) at
a/dx^2 in {0.25, 4, 64}, and a stag-size^3 periodic StaggeredGrid (3 components, each its own system).  Per case: CG iterations,
ms per solve and per iteration (CUDA events, median over --reps after one warm-up solve), and the HBM rate for the byte count of
the two-sweep CG, 30 B/cell per iteration (pass A: r, d read, d' written; pass B: d' read, r read and written, x updated every
second iteration).  The reference point is the pressure CG of the same size with PHICUDA_CG_PASSES=2, 100 iterations at rtol 0."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from phiflow_b200 import _ops as ops  # noqa: E402
from phiflow_b200._clocks import ClockSampler  # noqa: E402

PER = ('periodic', 'periodic')


def _timed(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def _random(dom, gen):
    t = dom.alloc_centered()
    idx = (slice(None),) + tuple(slice(0, dom.res[a]) for a in range(dom.dim - 1, -1, -1))
    t[idx] = torch.randn((dom.batch,) + tuple(reversed(dom.res)), generator=gen, device=dom.device)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--stag-size', type=int, default=256)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA device')
    dev = torch.device('cuda:0')
    gen = torch.Generator(device=dev).manual_seed(0)
    sampler = ClockSampler(0)
    sampler.start()
    out = {'cases': []}
    n = args.size
    dom = ops.Domain((n,) * 3, (1.0,) * 3, 1, device=dev)
    u = _random(dom, gen)
    for name, spec in (('periodic', (PER,) * 3), ('heat_flow', ((1.0, 'zg'), PER, PER))):
        for k in (0.25, 4.0, 64.0):
            ms = _timed(lambda: ops.diffuse_implicit(dom, spec, u, k, 1e-5, 1e-5, 1000), args.reps)
            rec = ops.read_results(dom)
            info = ops.last_launch_info()
            it = int(rec['iterations'][0])
            out['cases'].append({'case': f'{name} {n}^3', 'a_dx2': k, 'iterations': it, 'converged': bool(rec['converged'][0]),
                                 'ms_per_solve': ms, 'ms_per_iteration': ms / max(it, 1), 'passes': info['passes'],
                                 'generic': info['generic'], 'tbs_at_30B': 30.0 * n ** 3 * it / (ms * 1e-3) / 1e12})
    del u
    m = args.stag_size
    sdom = ops.Domain((m,) * 3, (1.0,) * 3, 1, vbc=(PER,) * 3, device=dev)
    comps = [_random(sdom, gen) for _ in range(3)]
    for k in (0.25, 4.0, 64.0):
        ms = _timed(lambda: ops.diffuse_implicit(sdom, (PER,) * 3, comps, k, 1e-5, 1e-5, 1000), args.reps)
        rec = ops.read_results(sdom, 3)
        its = [int(i) for i in rec['iterations']]
        out['cases'].append({'case': f'staggered periodic {m}^3 x 3', 'a_dx2': k, 'iterations': its, 'converged': bool(rec['converged'].all()),
                             'ms_per_solve': ms, 'ms_per_iteration': ms / max(max(its), 1),
                             'tbs_at_30B': 30.0 * m ** 3 * sum(its) / (ms * 1e-3) / 1e12})
    del comps
    # two-sweep pressure CG on the same grid size, fixed 100 iterations
    vbc = (PER,) * 3
    pdom = ops.Domain((n,) * 3, (1.0,) * 3, 1, vbc=vbc, device=dev)
    rhs = _random(pdom, gen)
    rhs -= rhs[:, :, :, :n].mean()
    x = pdom.alloc_centered()
    prm = ops.cg_params(vbc, rtol=0.0, atol=0.0, max_iter=100)
    os.environ['PHICUDA_CG_PASSES'] = '2'
    ms = _timed(lambda: ops.cg_poisson(pdom, vbc, rhs, x.zero_(), prm), args.reps)
    os.environ.pop('PHICUDA_CG_PASSES', None)
    it = int(ops.read_results(pdom)['iterations'][0])
    out['pressure_cg_two_sweep'] = {'case': f'periodic {n}^3', 'iterations': it, 'ms_per_solve': ms, 'ms_per_iteration': ms / it,
                                    'passes': ops.last_launch_info()['passes'], 'tbs_at_30B': 30.0 * n ** 3 * it / (ms * 1e-3) / 1e12}
    clocks = sampler.summary()
    out.update({'gpu': clocks.get('gpu') or torch.cuda.get_device_name(0), 'power_limit_w': clocks.get('power_limit_w'),
                'sm_mhz_median': clocks.get('sm_mhz'), 'clock_reasons': clocks.get('reasons')})
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
