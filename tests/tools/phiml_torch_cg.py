"""
The GPU path a PhiFlow user has today, timed beside ours (SURVEY.md section 8(d): "also report, labelled separately, the reference
torch-CUDA backend on the same GPU for C2"): the pressure solve of the 256^3 periodic plume (98 % of a step) through

  (a) `phiml.backend.torch.TORCH.linear_solve('CG', csr, ...)`  - the UNMODIFIED PhiML 1.7.2 from oracle/_ref; with
      matrix_offset=None this is its best case, the fused `torch_sparse_cg` loop (cuSPARSE SpMM + torch reductions, one host sync
      per iteration for the `while` condition; PhiML/phiml/backend/torch/_torch_backend.py:857-872, 1264-1292);
  (b) the same call with the `matrix_offset` the reference sets on periodic / closed domains (phi/physics/fluid.py:145-148) ->
      generic `_linalg.cg` on torch tensors (_torch_backend.py:858-860), optional (--with-offset);
  (c) `phicuda_cg_poisson_f32` (persistent TMA-ring kernel), same right-hand side, same tolerances, x0 = 0.

`phi` itself cannot be imported (needs phiml >= 1.14), so the whole step of the reference cannot be run on the GPU; the solve is
the part that can, and it is the part that matters.  Timing: CUDA events, 1 warm-up + `--reps` solves each, device synchronised on
both sides.  Prints one JSON line (committed as profiles/r2_phiml_torch_cg.json).

    python tests/tools/phiml_torch_cg.py [--n 256] [--reps 3] [--with-offset] [--no-ours]
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, 'oracle', '_ref')


def timed(fn, reps, cuda):
    fn()                                                       # warm-up (cuSPARSE buffers, lazy module loads)
    times = []
    for _ in range(reps):
        if cuda:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            out = fn()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) * 1e-3)
        else:
            t0 = time.perf_counter()
            out = fn()
            times.append(time.perf_counter() - t0)
    return out, float(np.median(times)), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=256)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--rtol', type=float, default=1e-3)
    ap.add_argument('--atol', type=float, default=1e-5)
    ap.add_argument('--with-offset', action='store_true')
    ap.add_argument('--no-ours', action='store_true', help='reference side only (dry run on a CPU box)')
    args = ap.parse_args()
    if not os.path.isdir(os.path.join(REF, 'phiml')):
        print(json.dumps({"unavailable": "PhiML not installed under oracle/_ref (run __graft_entry__.build() where the reference's PhiML tree exists, oracle/ref_build.py)"}))
        return
    sys.path.insert(0, REF)
    from oracle import oracle_np as O
    cuda = torch.cuda.is_available()
    dev = 'cuda' if cuda else 'cpu'
    n = args.n
    res, dx = (n, n, n), (100.0 / n,) * 3
    lower, upper = (0.0,) * 3, (100.0,) * 3
    vbc = O.uniform_bc(3, O.PERIODIC)
    t0 = time.perf_counter()
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))                    # == the matrix phiml traces (tests/golden)
    t_matrix = time.perf_counter() - t0
    # right-hand side: divergence of the buoyancy kick of a smoke blob + the seeded noise of the bench's initial velocity
    blob = O.sphere_soft_mask((50.0, 50.0, 30.0), 20.0, lower, upper, res)
    rng = np.random.default_rng(0)
    v = [(0.01 * rng.standard_normal(s)).astype(np.float32) for s in O.staggered_shapes(res, vbc)]
    v[2] += 0.05 * (blob + np.roll(blob, 1, 2))
    y = O.divergence_staggered(v, dx, O.component_bcs(vbc, 3))
    y = (y - y.mean(dtype=np.float32)).astype(np.float32)
    out = {"workload": f"pressure solve of the {n}^3 periodic plume (BASELINE configs[2] = c2 when n = 256): CG, rtol {args.rtol}, atol {args.atol}, x0 = 0",
           "cells": n ** 3, "matrix_build_s_scipy": t_matrix, "device": torch.cuda.get_device_name(0) if cuda else 'cpu',
           "timing": f"CUDA events, median of {args.reps} after 1 warm-up" if cuda else "perf_counter (CPU dry run)"}
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from phiml.backend.torch import TORCH
        import phiml
        lin = torch.sparse_csr_tensor(torch.from_numpy(A.indptr.astype(np.int64)), torch.from_numpy(A.indices.astype(np.int64)),
                                      torch.from_numpy(A.data.astype(np.float32)), size=A.shape).to(dev)
        yt = torch.from_numpy(y.reshape(1, -1)).to(dev)
        x0 = torch.zeros_like(yt)
        tol = (torch.tensor([args.rtol], dtype=torch.float32, device=dev), torch.tensor([args.atol], dtype=torch.float32, device=dev), np.array([[1000]]))

        def ref_solve(offset=None):
            return TORCH.linear_solve('CG', lin, yt, x0, tol[0], tol[1], tol[2], None, offset)
        r, t_ref, all_ref = timed(ref_solve, args.reps, cuda)
        it_ref = int(np.asarray(r.iterations.cpu())[0])
        out["phiml_torch"] = {"library": f"PhiML {phiml.__version__} TorchBackend (unmodified, oracle/_ref), torch {torch.__version__}", "method": r.method,
                              "s_per_solve": t_ref, "all_s": all_ref, "iterations": it_ref, "us_per_iteration": 1e6 * t_ref / max(it_ref, 1),
                              "converged": bool(np.asarray(r.converged.cpu())[0])}
        x_ref = r.x[0].float().cpu().numpy()
        print(json.dumps(out), file=sys.stderr, flush=True)            # partial results survive a later failure
        if args.with_offset:
            offset = O.estimate_matrix_offset(A, n ** 3, np.random.default_rng(0))
            off_t = torch.tensor([offset], dtype=torch.float32, device=dev)
            r2, t2, all2 = timed(lambda: ref_solve(off_t), max(1, args.reps - 1), cuda)
            it2 = int(np.asarray(r2.iterations if isinstance(r2.iterations, np.ndarray) else r2.iterations.cpu()).ravel()[0])
            out["phiml_torch_with_matrix_offset"] = {"method": r2.method, "s_per_solve": t2, "all_s": all2, "iterations": it2,
                                                     "us_per_iteration": 1e6 * t2 / max(it2, 1), "matrix_offset": float(offset)}
    print(json.dumps(out), file=sys.stderr, flush=True)
    if not args.no_ours:
        from phiflow_b200 import _ops as ops
        dom = ops.Domain(res, dx, 1, vbc=vbc)
        rhs = dom.centered_from_numpy(y)
        x = dom.alloc_centered()
        prm = ops.cg_params(vbc, rtol=args.rtol, atol=args.atol, max_iter=1000, balance=False)

        def our_solve():
            x.zero_()
            ops.cg_poisson(dom, vbc, rhs, x, prm)
        _, t_our, all_our = timed(our_solve, args.reps, True)
        info = ops.read_results(dom)
        it_our = int(info['iterations'][0])
        got = dom.centered_to_numpy(x).reshape(-1)
        xr = x_ref - x_ref.mean()
        li = ops.last_launch_info()
        out["phicuda"] = {"s_per_solve": t_our, "all_s": all_our, "iterations": it_our, "us_per_iteration": 1e6 * t_our / max(it_our, 1),
                          "converged": bool(info['converged'][0]), "kernel_variant": li, "includes": "x.zero_() (one memset) per solve",
                          "gbps_at_30B_per_cell_iteration": 30.0 * n ** 3 * it_our / t_our / 1e9}
        out["solutions_max_abs_diff_over_scale"] = float(np.abs((got - got.mean()) - xr).max() / max(np.abs(xr).max(), 1e-30))
        out["speedup_per_solve"] = t_ref / t_our
        out["speedup_per_iteration"] = (t_ref / max(it_ref, 1)) / (t_our / max(it_our, 1))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
