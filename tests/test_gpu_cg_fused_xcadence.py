"""
x cadence of the one-sweep CG (pass F in ring_kernels.cu): x is updated every third iteration with a d_{k-2} rebuilt from the staged
directions, a sweep whose beta_k is below FUSED_XBETA_MIN applies its two owed steps at once instead, and an entry that stops owing
zero, one or two steps gets them after the loop.  Right-hand sides made of m Fourier modes of the periodic Laplacian with distinct
eigenvalues are solved exactly by CG in m iterations, which fixes where each entry stops and makes beta small or zero on purpose.

Reference semantics: PhiML/phiml/backend/_linalg.py:52-90 (CG); oracle = oracle/oracle_np.py (pinned by tests/golden).
"""
import numpy as np
import pytest
import torch

from oracle import oracle_np as O
from test_gpu_cg_fused import DX, MULTI, PER3, assert_passes, env, solve

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from phiflow_b200 import _ops as ops

XBETA_MIN = 1e-2          # FUSED_XBETA_MIN in ring_kernels.cu


def wavenumbers(res, m):
    """The first m wavenumbers along y: high enough that A is applied to them with fp32 rounding far below the tolerance (the
    diagonal 2 (1/dx^2 + 1/dy^2 + 1/dz^2) cancels to a small eigenvalue for the lowest modes), all with distinct eigenvalues."""
    return [j * res[1] // 16 for j in (4, 2, 6, 3, 5)[:m]]


def modes(res, weights):
    """sum_j w_j cos(2 pi k_j y / ny): one Fourier mode of the periodic Laplacian per weight."""
    y = np.arange(res[1], dtype=np.float64)[None, :, None]
    f = sum(w * np.cos(2 * np.pi * k * y / res[1]) for k, w in zip(wavenumbers(res, len(weights)), weights))
    return np.broadcast_to(f, res).astype(np.float32)


def spectral_betas(res, weights):
    """beta_1, beta_2, ... of CG in exact arithmetic on the modes' right-hand side (CG on the diagonal system of its eigenvalues)."""
    lam = np.array([(2 - 2 * np.cos(2 * np.pi * k / res[1])) / DX[1] ** 2 for k in wavenumbers(res, len(weights))])
    r = np.array(weights, np.float64)
    d, rs, betas = r.copy(), r @ r, []
    for _ in range(len(weights) - 1):
        q = lam * d
        a = rs / (d @ q)
        r = r - a * q
        rs_new = r @ r
        betas.append(rs_new / rs)
        d, rs = r + betas[-1] * d, rs_new
    return betas


def check_against_oracle(res, rhs, got, info, rtol, max_iter, iterations=True):
    A = O.poisson_matrix(res, DX, O.pressure_bc(PER3))
    for b in range(rhs.shape[0]):
        y = rhs[b] - rhs[b].mean()
        ref = O.cg(A, y, np.zeros(res, np.float32), rtol, 0.0, max_iter, None)
        if iterations:
            assert info['iterations'][b] == ref['iterations'], (b, info['iterations'], ref['iterations'])
        xr = ref['x'].reshape(res)
        xr = xr - xr.mean()
        np.testing.assert_allclose(got[b], xr, rtol=0, atol=2e-5 * max(1.0, np.abs(xr).max()), err_msg=f'entry {b}')


@pytest.mark.parametrize('k', [5, 6, 8, 9])
def test_xcadence_truncated_owed(k):
    """k iterations of a random entry (owing k mod 3 steps when it stops) beside entries of 3, 4 and 5 modes, which converge at
    iterations 3, 4 and 5 and stop owing 0, 1 and 2 steps."""
    res = (256, 16, 12)
    rng = np.random.default_rng(45)
    rhs = np.stack([rng.standard_normal(res).astype(np.float32)] + [modes(res, [1.0, 0.7, 0.5, 0.4, 0.3][:m]) for m in (3, 4, 5)])
    dom = ops.Domain(res, DX, rhs.shape[0], vbc=PER3)
    prm = ops.cg_params(PER3, rtol=1e-5, atol=0.0, max_iter=k)
    got, info, _ = solve(dom, PER3, rhs, prm, 1)
    assert [int(i) for i in info['iterations']] == [k, 3, 4, 5], info['iterations']
    check_against_oracle(res, rhs, got, info, 1e-5, k)


@pytest.mark.parametrize('split,nzc', [(None, None), (0, 16), (1, None)])
def test_xcadence_small_beta_guard(split, nzc):
    """beta_1 = 0 (one mode: exact in one iteration), beta_2 = 0 (two modes) and beta_1 below the guard's threshold (three modes
    weighted 1, 1e-2, 1e-4), run on past the exact solution; the same per-entry x mode on every CTA with several units per CTA
    and with the tail split."""
    res = MULTI
    weights = ([1.0], [1.0, 0.5], [1.0, 1e-2, 1e-4])
    assert spectral_betas(res, weights[2])[0] < XBETA_MIN
    rhs = np.stack([modes(res, w) for w in weights])
    max_iter = 8
    prm = ops.cg_params(PER3, rtol=1e-12, atol=0.0, max_iter=max_iter)
    # the tail split spreads one entry over all CTAs: there every case is a solve of its own
    parts = [rhs[b:b + 1] for b in range(len(weights))] if split == 1 else [rhs]
    for part in parts:
        with env(PHICUDA_RING_SPLIT=split, PHICUDA_RING_NZC=nzc):
            dom = ops.Domain(res, DX, part.shape[0], vbc=PER3)
            got, info, _ = solve(dom, PER3, part, prm, 1)
            assert_passes(1, multi_unit=split == 0, split=split)
        # past the exact solution the residual is rounding noise, on which the oracle and the kernel may stop at different iterations
        check_against_oracle(res, part, got, info, 1e-12, max_iter, iterations=False)
