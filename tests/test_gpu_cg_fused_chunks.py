"""
Pass F, the one-sweep CG iteration (ring_kernels.cu), with x read straight from global memory one plane ahead (x does not travel
through the ring), on z chunks that do not divide nz, several units per CTA and both tail-split modes.  Every case asserts through
last_launch_info() that the one-sweep form ran (passes == 1) and on which tile (TY).

Reference semantics: PhiML/phiml/backend/_linalg.py:52-90 (CG); oracle = oracle/oracle_np.py (pinned by tests/golden).
"""
import numpy as np
import pytest
import torch

from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from phiflow_b200 import _ops as ops
    from test_gpu_cg_fused import DX, PER3, env, solve

# shape -> (z chunks forced with PHICUDA_RING_NZC so that the chunk does not divide nz, TY)
SHAPES = {(256, 64, 40): (3, 8), (512, 64, 24): (5, 4)}


def assert_tile(ty, **kw):
    info = ops.last_launch_info()
    assert info['passes'] == 1 and info['TY'] == ty, info
    for k, v in kw.items():
        assert info[k] == v, info
    return info


@pytest.mark.parametrize('res', list(SHAPES))
def test_truncated_iterates(res):
    """Exactly k iterations (odd and even k: the x update of every second pass and the step owed after the last one), with z chunks
    that do not divide nz, against the two-sweep kernel and against the oracle's CG."""
    nzc, ty = SHAPES[res]
    rng = np.random.default_rng(51)
    rhs = rng.standard_normal((1,) + res).astype(np.float32)
    A = O.poisson_matrix(res, DX, O.pressure_bc(PER3))
    y = rhs[0] - rhs[0].mean()
    with env(PHICUDA_RING_NZC=nzc, PHICUDA_RING_SPLIT=0):
        dom = ops.Domain(res, DX, 1, vbc=PER3)
        for k in (1, 2, 3, 4, 7):
            prm = ops.cg_params(PER3, rtol=1e-12, atol=0.0, max_iter=k)
            got, info, _ = solve(dom, PER3, rhs, prm, 1)
            li = assert_tile(ty)
            assert li['nzc'] > 1 and res[2] % li['ZC'] != 0, li
            two, _, _ = solve(dom, PER3, rhs, prm, 2)
            ref = O.cg(A, y, np.zeros(res, np.float32), 1e-12, 0.0, k, None)
            assert info['iterations'][0] == k == ref['iterations']
            xr = ref['x'].reshape(res)
            xr = xr - xr.mean()
            scale = max(1.0, np.abs(xr).max())
            np.testing.assert_allclose(got[0], xr, rtol=0, atol=2e-5 * scale)
            np.testing.assert_allclose(got[0], two[0], rtol=0, atol=2e-5 * scale)


@pytest.mark.parametrize('res', list(SHAPES))
@pytest.mark.parametrize('rtol', [1e-3, 1e-5])
def test_converged_against_two_sweep(res, rtol):
    """Converged solves: the two-sweep kernel's iteration counts and solutions."""
    rng = np.random.default_rng(52)
    rhs = rng.standard_normal((2,) + res).astype(np.float32)
    rhs[1] *= 4.0
    dom = ops.Domain(res, DX, 2, vbc=PER3)
    prm = ops.cg_params(PER3, rtol=rtol, atol=1e-5, max_iter=5000)
    x1, i1, _ = solve(dom, PER3, rhs, prm, 1)
    assert_tile(SHAPES[res][1])
    x2, i2, _ = solve(dom, PER3, rhs, prm, 2)
    for b in range(2):
        n1, n2 = int(i1['iterations'][b]), int(i2['iterations'][b])
        assert i1['converged'][b] == 1 and abs(n1 - n2) <= max(2, n2 // 100), (n1, n2)
        np.testing.assert_allclose(x1[b], x2[b], rtol=0, atol=20 * rtol * np.abs(x2[b]).max())


def test_units_and_tail_split():
    """Several units per CTA (PHICUDA_RING_NZC) and both tail-split modes give the same iterates."""
    res = (256, 128, 48)
    rng = np.random.default_rng(53)
    rhs = rng.standard_normal((1,) + res).astype(np.float32)
    dom = ops.Domain(res, DX, 1, vbc=PER3)
    for k in (3, 4):
        prm = ops.cg_params(PER3, rtol=1e-12, atol=0.0, max_iter=k)
        outs = {}
        for split, nzc in ((0, 16), (1, None)):
            with env(PHICUDA_RING_SPLIT=split, PHICUDA_RING_NZC=nzc):
                got, _, _ = solve(dom, PER3, rhs, prm, 1)
                li = assert_tile(8, split=split)
                if split == 0:
                    assert li['total_units'] >= li['grid_ctas'] + 64, li
            outs[split] = got[0]
        scale = max(1.0, np.abs(outs[0]).max())
        np.testing.assert_allclose(outs[1], outs[0], rtol=0, atol=1e-6 * scale)

