"""
The one-sweep CG (pass F in ring_kernels.cu) does not store the residual: each pass recovers r_k = d_k - beta_k d_{k-1} from the two
staged directions.  Its rounding error is relative to the current |r_k|, so the gap between the recurrence residual (which drives the
stopping rule) and the true residual y - A x must stay as small as with the stored residual of the two-sweep kernel, also over a
long solve that runs into fp32's attainable accuracy.

Reference semantics: PhiML/phiml/backend/_linalg.py:52-90 (CG); the true residual uses oracle/oracle_np.py's laplace in float64.
"""
import numpy as np
import pytest
import torch

from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from phiflow_b200 import _ops as ops
    from test_gpu_cg_fused import PER3, solve


def test_fused_true_residual_long_solve():
    """128^3 periodic, smooth zero-mean right-hand side as in the plume, rtol 1e-6, atol 0 (about 320 iterations): both forms
    converge with the same iteration count, and the one-sweep form's true residual is at most twice the two-sweep form's."""
    n = 128
    res = (n, n, n)
    dx = (100.0 / n,) * 3
    rng = np.random.default_rng(0)
    y = rng.standard_normal(res).astype(np.float32)
    for _ in range(3):
        y = ((y + np.roll(y, 1, 0) + np.roll(y, 1, 1) + np.roll(y, 1, 2)) / 4).astype(np.float32)
    y = (y - y.mean(dtype=np.float64)).astype(np.float32)
    dom = ops.Domain(res, dx, 1, vbc=PER3)
    prm = ops.cg_params(PER3, rtol=1e-6, atol=0.0, max_iter=5000)
    x1, i1, _ = solve(dom, PER3, y[None], prm, 1)
    x2, i2, _ = solve(dom, PER3, y[None], prm, 2)
    for info in (i1, i2):
        assert info['converged'][0] == 1 and info['diverged'][0] == 0, info
    n1, n2 = int(i1['iterations'][0]), int(i2['iterations'][0])
    assert abs(n1 - n2) <= max(2, n2 // 100), (n1, n2)
    y64 = y.astype(np.float64)
    rel = {}
    with O.precision(64):
        for passes, x in ((1, x1), (2, x2)):
            r = y64 - O.laplace(x[0].astype(np.float64), dx, O.pressure_bc(PER3))
            rel[passes] = float(np.sqrt(np.sum(r * r) / np.sum(y64 * y64)))
    assert rel[1] <= 2.0 * rel[2], (rel, n1, n2)
