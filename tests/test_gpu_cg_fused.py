"""
The one-sweep CG of the TMA ring (k_cg_ring<3, FUSED=true>, pass F in ring_kernels.cu): beta is computed one iteration ahead so that
each iteration makes one sweep over the grid instead of two.  It is selected for 3-D, branch-free tilings with periodic y and z on
one GPU; PHICUDA_CG_PASSES=2 forces the two-sweep kernel.  Every case asserts through phicuda_last_cg_passes which form ran.

Reference semantics: PhiML/phiml/backend/_linalg.py:52-90 (CG); oracle = oracle/oracle_np.py (pinned by tests/golden).
"""
import os

import numpy as np
import pytest
import torch

from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from phiflow_b200 import _ops as ops
    from phiflow_b200 import _lib

PER3 = (('periodic', 'periodic'),) * 3
PER_ZGX = ((0.0, 0.0), ('periodic', 'periodic'), ('periodic', 'periodic'))     # closed in x: zero-gradient pressure, handled in-line
FAST_SHAPES = [(256, 16, 12), (512, 8, 8), (256, 128, 48)]
MULTI = (256, 128, 48)
DX = (0.5, 0.25, 2.0)


class env:
    def __init__(self, **kv):
        self.kv = {k: (None if v is None else str(v)) for k, v in kv.items()}

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kv}
        for k, v in self.kv.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def assert_passes(passes, multi_unit=False, split=None):
    info = ops.last_launch_info()
    assert info['kernel'] == _lib.KERNEL_CG_RING and info['generic'] == 0, info
    assert info['passes'] == passes, info
    if multi_unit:
        assert info['total_units'] >= info['grid_ctas'] + 64, info
    if split is not None:
        assert info['split'] == split, info
    return info


def solve(dom, vbc, rhs, prm, passes):
    with env(PHICUDA_CG_PASSES=None if passes == 1 else 2):
        x = dom.centered_to_numpy(ops.cg_poisson(dom, vbc, dom.centered_from_numpy(rhs), None, prm), squeeze=False)
        info = assert_passes(passes)
    return x, ops.read_results(dom), info


@pytest.mark.parametrize('res', FAST_SHAPES)
@pytest.mark.parametrize('vname', ['periodic', 'zg_x'])
def test_fused_truncated_iterates(res, vname):
    """Exactly k iterations for odd and even k (x updated every second sweep, three direction buffers) against the oracle."""
    vbc = {'periodic': PER3, 'zg_x': PER_ZGX}[vname]
    rng = np.random.default_rng(41)
    batch = 2
    rhs = rng.standard_normal((batch,) + res).astype(np.float32)
    rhs[1] *= 3.0
    A = O.poisson_matrix(res, DX, O.pressure_bc(vbc))
    with env(PHICUDA_RING_NZC=16 if res == MULTI else None):
        dom = ops.Domain(res, DX, batch, vbc=vbc)
        for k in (1, 2, 3, 4, 7, 50):
            prm = ops.cg_params(vbc, rtol=1e-12, atol=0.0, max_iter=k)
            got, info, _ = solve(dom, vbc, rhs, prm, 1)
            if res == MULTI:
                assert_passes(1, multi_unit=True)
            for b in range(batch):
                y = rhs[b] - rhs[b].mean()
                ref = O.cg(A, y, np.zeros(res, np.float32), 1e-12, 0.0, k, None)
                assert info['iterations'][b] == k == ref['iterations'] and info['converged'][b] == 0
                xr = ref['x'].reshape(res)
                xr = xr - xr.mean()
                np.testing.assert_allclose(got[b], xr, rtol=0, atol=2e-5 * max(1.0, np.abs(xr).max()))


@pytest.mark.parametrize('res', FAST_SHAPES)
@pytest.mark.parametrize('rtol', [1e-3, 1e-5])
def test_fused_against_two_pass(res, rtol):
    """Same right-hand sides through both forms: the iteration counts and the solutions agree."""
    rng = np.random.default_rng(42)
    batch = 2
    rhs = rng.standard_normal((batch,) + res).astype(np.float32)
    rhs[1] *= 5.0
    dom = ops.Domain(res, DX, batch, vbc=PER3)
    prm = ops.cg_params(PER3, rtol=rtol, atol=1e-5, max_iter=5000)
    x1, i1, _ = solve(dom, PER3, rhs, prm, 1)
    x2, i2, _ = solve(dom, PER3, rhs, prm, 2)
    for b in range(batch):
        assert i1['converged'][b] == 1 and i1['diverged'][b] == 0
        n1, n2 = int(i1['iterations'][b]), int(i2['iterations'][b])
        assert abs(n1 - n2) <= max(2, n2 // 100), (n1, n2)
        np.testing.assert_allclose(x1[b], x2[b], rtol=0, atol=20 * rtol * np.abs(x2[b]).max())


def test_fused_tail_split_and_units():
    """Tail split on and off (with several z chunks per tile when off) give the same iterates and agree with the oracle."""
    res = MULTI
    rng = np.random.default_rng(43)
    rhs = rng.standard_normal((1,) + res).astype(np.float32)
    A = O.poisson_matrix(res, DX, O.pressure_bc(PER3))
    y = rhs[0] - rhs[0].mean()
    dom = ops.Domain(res, DX, 1, vbc=PER3)
    for k in (3, 4):
        prm = ops.cg_params(PER3, rtol=1e-12, atol=0.0, max_iter=k)
        outs = {}
        for split, nzc in ((0, 16), (1, None)):
            with env(PHICUDA_RING_SPLIT=split, PHICUDA_RING_NZC=nzc):
                got, _, _ = solve(dom, PER3, rhs, prm, 1)
                assert_passes(1, multi_unit=split == 0, split=split)
            outs[split] = got[0]
        ref = O.cg(A, y, np.zeros(res, np.float32), 1e-12, 0.0, k, None)['x'].reshape(res)
        ref = ref - ref.mean()
        for split in (0, 1):
            np.testing.assert_allclose(outs[split], ref, rtol=0, atol=2e-5 * max(1.0, np.abs(ref).max()))
        np.testing.assert_allclose(outs[1], outs[0], rtol=0, atol=1e-6 * max(1.0, np.abs(ref).max()))
    with env(PHICUDA_RING_SPLIT=1):
        prm = ops.cg_params(PER3, rtol=1e-3, atol=1e-5, max_iter=5000)
        got, info, _ = solve(dom, PER3, rhs, prm, 1)
    ref = O.cg(A, y, np.zeros(res, np.float32), 1e-3, 1e-5, 5000, None)
    assert info['converged'][0] == 1 and abs(int(info['iterations'][0]) - ref['iterations']) <= max(2, ref['iterations'] // 10)
    xr = ref['x'].reshape(res)
    xr = xr - xr.mean()
    np.testing.assert_allclose(got[0], xr, rtol=0, atol=20e-3 * np.abs(xr).max())


def test_fused_batch_entries_stop_at_different_iterations():
    """Entries that converge early are frozen (their x keeps the step they owe) while the others go on: entry 1 is scaled so far
    down that the absolute tolerance stops it early, entry 2 is smooth."""
    res = (256, 16, 12)
    rng = np.random.default_rng(44)
    batch = 3
    rtol, atol = 1e-3, 1e-5
    A = O.poisson_matrix(res, DX, O.pressure_bc(PER3))
    rhs = rng.standard_normal((batch,) + res).astype(np.float32)
    rhs[1] *= 2e-5
    for _ in range(4):
        rhs[2] = sum(np.roll(rhs[2], s, a) for a in range(3) for s in (-1, 1)) / 6.0
    dom = ops.Domain(res, DX, batch, vbc=PER3)
    prm = ops.cg_params(PER3, rtol=rtol, atol=atol, max_iter=5000)
    got, info, _ = solve(dom, PER3, rhs, prm, 1)
    its = [int(i) for i in info['iterations']]
    assert len(set(its)) > 1, its
    for b in range(batch):
        y = rhs[b] - rhs[b].mean()
        ref = O.cg(A, y, np.zeros(res, np.float32), rtol, atol, 5000, None)
        assert ref['converged'] and info['converged'][b] == 1
        assert abs(its[b] - ref['iterations']) <= max(2, ref['iterations'] // 10), (its, ref['iterations'])
        xr = ref['x'].reshape(res)
        xr = xr - xr.mean()
        rel = max(rtol, atol / float(np.sqrt(np.sum(y.astype(np.float64) ** 2))))
        np.testing.assert_allclose(got[b], xr, rtol=0, atol=20 * rel * np.abs(xr).max())


def test_fused_plume_sequence():
    """Five steps of the benchmarked plume step (ops.plume_step) on the one-sweep solver, against the oracle."""
    from test_gpu_variants import _plume_parity
    _plume_parity((256, 32, 24), 5, expect_fast=True)
    assert ops.last_launch_info()['passes'] == 1


def test_fused_512_bench_state():
    """The bench's 512^3 plume (seeded state, 3 steps) through both forms: the same iteration counts and fields."""
    import bench
    dev = torch.device('cuda:0')
    out = {}
    for passes in (1, 2):
        with env(PHICUDA_CG_PASSES=None if passes == 1 else 2):
            sim = bench.PlumeSim(512, dev)
            _, res_dev = sim.dom.workspace()
            its = []
            for _ in range(3):
                sim.step()
                its.append(int(res_dev[0].item()))
            assert_passes(passes)
            out[passes] = (its, [t.clone() for t in sim.v], sim.p.clone(), sim.s.clone())
            del sim
            torch.cuda.empty_cache()
    (i1, v1, p1, s1), (i2, v2, p2, s2) = out[1], out[2]
    for a, b in zip(i1, i2):
        assert abs(a - b) <= max(2, b // 100), (i1, i2)
    for a, b in list(zip(v1, v2)) + [(p1, p2), (s1, s2)]:
        scale = float(b.abs().max())
        assert float((a - b).abs().max()) <= 1e-2 * max(scale, 1e-6), (float((a - b).abs().max()), scale)
