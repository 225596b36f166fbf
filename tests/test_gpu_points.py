"""
advect.points on the GPU (phicuda_advect_points_f32, k_advect_points, DESIGN.md row N11): PhiML's positions
(tests/golden/phiml_points.npz) bit for bit, with and without a trajectory; the kernel's restatement (tests/oracle_points.py) where
the fixture has no case; streamlines == iterate over advect.points; the launch record; broadcasting both ways; in-place output;
trajectory offsets beyond 2^31 elements; refused calls that leave the outputs untouched; examples/streamlines.py at the notebook's size.
"""
import os
import sys

import numpy as np
import pytest
import torch

from oracle_points import advect_points as oracle_advect_points
from phiflow_b200 import _lib, _ops
from test_points_host import GOLD, ROOT, cases, golden_case, runs, same

pytestmark = pytest.mark.gpu


def _setup(g, name):
    spec, vel, pts, (lower, upper), res = golden_case(g, name)
    d = len(res)
    vb = vel[0][0].shape[0]
    dx = tuple((u - l) / n for l, u, n in zip(lower, upper, res))
    vspec = [tuple(tuple(s) for s in comp) for comp in spec]
    dom = _ops.Domain(res, dx, vb, vbc=list(vspec))
    v = dom.faces_from_numpy([vel[c][0] for c in range(d)], list(vspec))
    return dom, list(vspec), v, vel, pts, lower, upper


@pytest.mark.parametrize('name', cases())
def test_fixture_bit_for_bit(name):
    g = np.load(GOLD)
    dom, vspec, v, vel, pts, lower, upper = _setup(g, name)
    p = torch.from_numpy(pts).cuda()
    for integ, steps, dt in runs():
        expected = g[f'{name}/{integ}_{steps}_{dt}']
        out = _ops.advect_points(dom, vspec, v, lower, upper, p, dt, integ, steps)
        assert same(out.cpu().numpy(), expected), (integ, steps, dt)
        assert _ops.last_launch_info()['kernel'] == _lib.KERNEL_POINTS
        out2, trj = _ops.advect_points(dom, vspec, v, lower, upper, p, dt, integ, steps, trajectory=True)
        trj = trj.cpu().numpy()
        assert same(out2.cpu().numpy(), expected) and same(trj[-1], expected)
        assert same(trj, oracle_advect_points(vel, pts, dt, integ, steps, trajectory=True)[1])
        assert same(trj[0], np.broadcast_to(pts, trj[0].shape))
    assert same(p.cpu().numpy(), pts)                                  # the input is not modified


def test_notebook_bit_for_bit():
    g = np.load(GOLD)
    spec = ((0.0, 0.0), (0.0, 0.0))
    dom = _ops.Domain((256, 256), (10 / 256, 10 / 256), 1, vbc=spec)
    v = dom.faces_from_numpy([g['notebook/v0'][0], g['notebook/v1'][0]], spec)
    p = torch.from_numpy(g['notebook/points']).cuda()
    out, trj = _ops.advect_points(dom, spec, v, (0., 0.), (10., 10.), p, 0.1, 'rk4', 50, trajectory=True)
    assert same(trj.cpu().numpy(), g['notebook/trajectory']) and same(out.cpu().numpy(), g['notebook/trajectory'][-1])


def test_points_batch_over_a_batch_one_velocity():
    """Points of batch 2 in a velocity of batch 1 (the other broadcast than the fixture's `broadcast_2d`), against the oracle."""
    g = np.load(GOLD)
    dom, vspec, v, vel, pts, lower, upper = _setup(g, 'mixed2_2d')
    pts2 = np.stack([pts[0], pts[0][::-1] * np.float32(0.9)])
    out = _ops.advect_points(dom, vspec, v, lower, upper, torch.from_numpy(pts2).cuda(), 0.3, 'rk4', 3)
    assert same(out.cpu().numpy(), oracle_advect_points(vel, pts2, 0.3, 'rk4', 3))


def test_in_place():
    g = np.load(GOLD)
    dom, vspec, v, vel, pts, lower, upper = _setup(g, 'zero_3d')
    p = torch.from_numpy(pts).cuda()
    out = _ops.advect_points(dom, vspec, v, lower, upper, p, 0.2, 'rk4', 4, out=p)
    assert out.data_ptr() == p.data_ptr() and same(p.cpu().numpy(), g['zero_3d/rk4_4_0.2'])


def test_refused_calls_leave_outputs_untouched():
    g = np.load(GOLD)
    dom, vspec, v, vel, pts, lower, upper = _setup(g, 'zg_2d')
    p = torch.from_numpy(pts).cuda()
    out = torch.full_like(p, 7.0)
    lib = _lib.load()
    m = _ops.point_map(lower, upper, dom.res, vspec)
    for steps, integ in ((0, 1), (2, 5)):
        code = lib.phicuda_advect_points_f32(_ops.C.byref(dom.grid), _ops.C.byref(_ops.make_vbc(vspec, 2)), _ops._f3(v), _ops.C.byref(m),
                                             _ops._ptr(p), p.shape[1], 1, 0.1, integ, steps, _ops._ptr(out), None, _ops._stream())
        assert code == _lib.ERR_INVALID
    m.res[0][0] += 1
    code = lib.phicuda_advect_points_f32(_ops.C.byref(dom.grid), _ops.C.byref(_ops.make_vbc(vspec, 2)), _ops._f3(v), _ops.C.byref(m),
                                         _ops._ptr(p), p.shape[1], 1, 0.1, 1, 2, _ops._ptr(out), None, _ops._stream())
    assert code == _lib.ERR_INVALID
    torch.cuda.synchronize()
    assert torch.all(out == 7.0)


def test_trajectory_offsets_beyond_2_31():
    """(steps + 1) x points x 2 > 2^31 floats (~9 GB): the last entries, at offsets beyond 2^31, match the oracle at seeded points."""
    free, _ = torch.cuda.mem_get_info()
    n, steps = (1 << 22) + 4096, 256
    need = (steps + 2) * n * 2 * 4
    if free < need + (2 << 30):
        pytest.skip(f"needs {need / 2**30:.1f} GiB free, {free / 2**30:.1f} GiB are")
    g = np.load(GOLD)
    dom, vspec, v, vel, _, lower, upper = _setup(g, 'periodic_2d')
    rng = np.random.default_rng(5)
    pts = (np.asarray(lower, np.float32) + rng.random((1, n, 2)).astype(np.float32) * (np.asarray(upper, np.float32) - np.asarray(lower, np.float32))).astype(np.float32)
    out, trj = _ops.advect_points(dom, vspec, v, lower, upper, torch.from_numpy(pts).cuda(), 0.05, 'euler', steps, trajectory=True)
    assert trj.numel() > 2 ** 31
    pick = np.concatenate([rng.integers(0, n, 48), [n - 1]])
    ref = oracle_advect_points(vel, pts[:, pick], 0.05, 'euler', steps, trajectory=True)[1]
    got = trj[:, :, torch.from_numpy(pick).cuda()].cpu().numpy()
    assert same(got, ref) and same(out[:, torch.from_numpy(pick).cuda()].cpu().numpy(), ref[-1])
    del trj, out
    torch.cuda.empty_cache()


def test_example_at_notebook_size():
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    import streamlines as ex
    x_trj, s_trj, distance = ex.run(256)
    assert x_trj.shape == (51, 2) and s_trj.shape == (51, 64, 2) and np.all(np.isfinite(s_trj)) and np.all(distance > 0)
