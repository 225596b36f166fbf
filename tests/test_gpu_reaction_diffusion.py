"""
Reaction-diffusion (the Reaction_Diffusion notebook's Gray-Scott step) on the H100: phicuda_reaction_diffusion_f32 against the
oracle (tests/oracle_reaction_diffusion.py), its variants bit for bit, its refusals, and the mirror's flow.reaction_diffusion.

Error bound of one substep, derived from the operations (not fitted): the laplace of the library differs from the oracle's only in
multiplying by fl(1 / fl(dx^2)) instead of dividing by fl(dx^2), at most 4 eps * S per cell with S = sum_d (|l| + |r| + 2 |c|) / dx_d^2
(`lap_scale`); the epilogue's eight roundings are the oracle's own, so their part is 4 eps * (|u| + dt (|du lap| + |uvv| + |f (1 - u)|)).
With dx = 1 both laplaces are the same operations, and the library's substep is the float32 oracle's bit for bit.
"""
import os
import sys

import numpy as np
import pytest

from oracle import oracle_np as O
from oracle_reaction_diffusion import laplace as lap_oracle, reaction_diffusion as rd_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'phiml_reaction_diffusion.npz')
EPS = float(np.finfo(np.float32).eps)
MAZE = dict(du=0.19, dv=0.05, f=0.06, k=0.062)
P, Z = 'periodic', 'zg'


def _spec(arr):
    return tuple(tuple('periodic' if np.isnan(s) else ('zg' if np.isinf(s) else float(s)) for s in ax) for ax in arr)


def golden_case(g, name):
    prm = g[f'{name}/params']
    return (g[f'{name}/u0'], g[f'{name}/v0'], _spec(g[f'{name}/bc']), tuple(g[f'{name}/dx']),
            dict(du=prm[0], dv=prm[1], f=prm[2], k=prm[3]), float(prm[4]))


def lap_scale(x, dx, bc):
    s = None
    for a in range(x.ndim):
        p = O.pad_axis(np.abs(x.astype(np.float64)), a, 1, 1, bc[a])
        n = x.shape[a]
        t = (np.take(p, np.arange(0, n), axis=a) + np.take(p, np.arange(2, n + 2), axis=a) + 2 * np.abs(x)) / dx[a] ** 2
        s = t if s is None else s + t
    return s


def step_bound(u, v, bc, dx, prm, dt):
    """Per-cell bound on |library - float32 oracle| for ONE substep from (u, v) (module docstring)."""
    u64, v64 = u.astype(np.float64), v.astype(np.float64)
    lu, lv = lap_oracle(u, dx, bc, np.float64), lap_oracle(v, dx, bc, np.float64)
    uvv = np.abs(u64 * v64 * v64)
    bu = dt * prm['du'] * 4 * EPS * lap_scale(u, dx, bc) + 4 * EPS * (np.abs(u64) + dt * (np.abs(prm['du'] * lu) + uvv + np.abs(prm['f'] * (1 - u64))))
    bv = dt * prm['dv'] * 4 * EPS * lap_scale(v, dx, bc) + 4 * EPS * (np.abs(v64) + dt * (np.abs(prm['dv'] * lv) + uvv + np.abs((prm['f'] + prm['k']) * v64)))
    return bu, bv


def gpu_run(u0, v0, bc, dx, prm, dt, substeps, calls=1):
    """u0, v0: (batch, x, y[, z]).  Returns (u, v) after `calls` calls of `substeps` each, and the launch info of the last call."""
    from phiflow_b200 import _ops
    dom = _ops.Domain(u0.shape[1:], dx, u0.shape[0])
    u, v = dom.centered_from_numpy(u0), dom.centered_from_numpy(v0)
    for _ in range(calls):
        u, v = _ops.reaction_diffusion(dom, bc, u, v, prm['du'], prm['dv'], prm['f'], prm['k'], dt, substeps)
    return dom.centered_to_numpy(u, squeeze=False), dom.centered_to_numpy(v, squeeze=False), _ops.last_launch_info()


def rand_state(shape, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.3, 1.0, shape).astype(np.float32), rng.uniform(0.0, 0.4, shape).astype(np.float32)


# ---- one substep against the oracle ------------------------------------------------------------------------------------------------
CASES = ['zero', 'periodic', 'zg', 'mixed', 'mixed3', 'aniso', 'ragged', 'batch']


@pytest.mark.gpu
@pytest.mark.parametrize('name', CASES)
def test_one_substep_against_oracle(name):
    u0, v0, bc, dx, prm, dt = golden_case(np.load(GOLD), name)
    u, v, info = gpu_run(u0, v0, bc, dx, prm, dt, 1)
    from phiflow_b200 import _lib
    assert info['kernel'] == _lib.KERNEL_RD_RING and info['generic'] == 1       # constant sides / 100-wide lines: per-tile handling
    for b in range(u0.shape[0]):
        ou, ov = rd_oracle(u0[b], v0[b], bc, dx, dt=dt, **prm)
        bu, bv = step_bound(u0[b], v0[b], bc, dx, prm, dt)
        assert np.all(np.abs(u[b] - ou) <= bu) and np.all(np.abs(v[b] - ov) <= bv)
        if all(d == 1.0 for d in dx):
            assert np.array_equal(u[b], ou) and np.array_equal(v[b], ov)


BRANCH_FREE = [((128, 64), ((P, P), (P, P))), ((256, 32), ((Z, Z), (P, P))), ((128, 32, 16), ((P, P), (Z, Z), (P, P))),
               ((128, 16, 12), ((Z, Z), (P, P), (Z, Z)))]


@pytest.mark.gpu
@pytest.mark.parametrize('res,bc', BRANCH_FREE)
def test_branch_free_variant_against_oracle(res, bc):
    u0, v0 = rand_state((2,) + res, 1)
    dx = (1.0,) * len(res)
    u, v, info = gpu_run(u0, v0, bc, dx, MAZE, 0.5, 1)
    assert info['generic'] == 0
    for b in range(2):
        ou, ov = rd_oracle(u0[b], v0[b], bc, dx, dt=0.5, **MAZE)
        assert np.array_equal(u[b], ou) and np.array_equal(v[b], ov)


# ---- substeps and variants, bit for bit ----------------------------------------------------------------------------------------------
SHAPES = [((128, 64), ((P, P), (P, P))), ((100, 60), ((0.0, 0.0), (0.0, 0.0))), ((37, 23), ((0.0, Z), (Z, 0.0))),
          ((64, 24, 20), ((P, P), (Z, 0.0), (0.0, Z))), ((128, 32, 24), ((P, P), (P, P), (P, P)))]


@pytest.mark.gpu
@pytest.mark.parametrize('res,bc', SHAPES)
@pytest.mark.parametrize('K', [3, 4])
def test_k_substeps_equal_k_calls(res, bc, K):
    u0, v0 = rand_state((2,) + res, 2)
    dx = (1.0,) * len(res)
    one = gpu_run(u0, v0, bc, dx, MAZE, 0.5, K)
    many = gpu_run(u0, v0, bc, dx, MAZE, 0.5, 1, calls=K)
    assert np.array_equal(one[0], many[0]) and np.array_equal(one[1], many[1])


@pytest.mark.gpu
@pytest.mark.parametrize('res,bc,knobs', [
    ((128, 96), ((P, P), (P, P)), [{}, {'PHICUDA_RING_TY': '5'}, {'PHICUDA_RING_TY': '2'}, {'PHICUDA_RING_TY': '32'}]),
    ((100, 50), ((0.0, 0.0), (0.0, 0.0)), [{}, {'PHICUDA_RING_TY': '3'}, {'PHICUDA_RING_TY': '8'}]),
    ((128, 32, 24), ((P, P), (P, P), (P, P)), [{}, {'PHICUDA_RING_TY': '3'}, {'PHICUDA_RING_NZC': '1'}, {'PHICUDA_RING_NZC': '5'},
                                              {'PHICUDA_RING_TY': '1', 'PHICUDA_RING_NZC': '3'}]),
    ((60, 20, 10), ((0.0, Z), (Z, 0.0), (P, P)), [{}, {'PHICUDA_RING_TY': '3'}, {'PHICUDA_RING_NZC': '1'}]),
])
def test_identical_across_tilings_and_variants(res, bc, knobs, monkeypatch):
    u0, v0 = rand_state((2,) + res, 3)
    dx = (1.0,) * len(res)
    outs, variants = [], set()
    for kn in knobs:
        for key in ('PHICUDA_RING_TY', 'PHICUDA_RING_NZC'):
            monkeypatch.delenv(key, raising=False)
        for key, val in kn.items():
            monkeypatch.setenv(key, val)
        u, v, info = gpu_run(u0, v0, bc, dx, MAZE, 0.5, 5)
        outs.append((u, v))
        variants.add((info['generic'], info['TY'], info['nzc']))
    assert len(variants) == len(knobs)                       # every knob setting picked a different tiling or variant
    for u, v in outs[1:]:
        assert np.array_equal(u, outs[0][0]) and np.array_equal(v, outs[0][1])


# ---- the notebook's size -------------------------------------------------------------------------------------------------------------
NOTEBOOK_FRAMES = 5          # horizon: 5 frames of 20 substeps = 100 substeps


@pytest.mark.gpu
@pytest.mark.parametrize('pset', ['maze', 'coral', 'dots'])
def test_notebook_size_against_float64(pset):
    """100 x 100, batch 3 (u: the example's smooth noise and two constants, v: uniform noise), 20 substeps per call, over 100 substeps: the library's distance from
    the float64 oracle is at most 2x the float32 oracle's own distance from it (plus 1e-6 for where the latter is ~0), and the
    library equals the float32 oracle bit for bit (dx = 1)."""
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    try:
        import reaction_diffusion as ex
    finally:
        sys.path.remove(os.path.join(ROOT, 'examples'))
    prm = ex.PARAMS[pset]
    u0 = np.stack([ex.smooth_noise() * .2 + .1, np.full((100, 100), 0.5, np.float32), np.full((100, 100), 0.25, np.float32)])
    v0 = rand_state((3, 100, 100), 4)[1]
    bc = ((0.0, 0.0), (0.0, 0.0))
    u, v, info = gpu_run(u0, v0, bc, (1.0, 1.0), prm, 0.5, 20, calls=NOTEBOOK_FRAMES)
    assert info['total_units'] > 0
    for b in range(3):
        o32 = rd_oracle(u0[b], v0[b], bc, (1.0, 1.0), dt=0.5, substeps=20 * NOTEBOOK_FRAMES, **prm)
        o64 = rd_oracle(u0[b], v0[b], bc, (1.0, 1.0), dt=0.5, substeps=20 * NOTEBOOK_FRAMES, dtype=np.float64, **prm)
        for lib, r32, r64 in ((u[b], o32[0], o64[0]), (v[b], o32[1], o64[1])):
            assert np.abs(lib - r64).max() <= 2 * np.abs(r32 - r64).max() + 1e-6
            assert np.array_equal(lib, r32)


# ---- other checks --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_zero_substeps_refusals_and_inputs():
    import torch
    from phiflow_b200 import _lib, _ops
    u0, v0 = rand_state((2, 64, 32), 5)
    dom = _ops.Domain((64, 32), (1.0, 1.0), 2)
    u, v = dom.centered_from_numpy(u0), dom.centered_from_numpy(v0)
    uc, vc = u.clone(), v.clone()
    un, vn = _ops.reaction_diffusion(dom, ((P, P), (P, P)), u, v, 0.19, 0.05, 0.06, 0.062, 0.5, 0)
    assert torch.equal(un, u) and torch.equal(vn, v)
    un, vn = _ops.reaction_diffusion(dom, ((P, P), (P, P)), u, v, 0.19, 0.05, 0.06, 0.062, 0.5, 3)
    assert torch.equal(u, uc) and torch.equal(v, vc) and not torch.equal(un, u)              # inputs not modified
    same = _ops.reaction_diffusion(dom, ((P, P), (P, P)), u, u, 0.19, 0.05, 0.06, 0.062, 0.5, 3)    # u is v
    assert torch.equal(u, uc)
    ref = gpu_run(u0, u0, ((P, P), (P, P)), (1.0, 1.0), MAZE, 0.5, 3)
    assert np.array_equal(dom.centered_to_numpy(same[0], squeeze=False), ref[0])
    # refusals through the C ABI with real device arrays leave them untouched
    lib = _lib.load()
    scratch = torch.empty(lib.phicuda_reaction_diffusion_scratch_bytes(C_ref(dom.grid)) // 4, dtype=torch.float32, device='cuda')
    for spec in ([((0.3, 0.3), (P, P))] * 2, [((Z, Z), (P, P)), ((P, P), (P, P))]):
        rc = lib.phicuda_reaction_diffusion_f32(C_ref(dom.grid), C_ref(_ops.make_vbc(spec, 2)), _ops._ptr(u), _ops._ptr(v), 0.19, 0.05, 0.06,
                                                0.062, 0.5, 3, _ops._ptr(scratch), scratch.numel() * 4, _ops._stream())
        assert rc == _lib.ERR_UNSUPPORTED
    rc = lib.phicuda_reaction_diffusion_f32(C_ref(dom.grid), C_ref(_ops.make_vbc(((P, P), (P, P)), 2)), _ops._ptr(u), _ops._ptr(v), 0.19, 0.05,
                                            0.06, 0.062, 0.5, -1, _ops._ptr(scratch), scratch.numel() * 4, _ops._stream())
    assert rc == _lib.ERR_INVALID
    torch.cuda.synchronize()
    assert torch.equal(u, uc) and torch.equal(v, vc)


def C_ref(x):
    import ctypes
    return ctypes.byref(x)


@pytest.mark.gpu
@pytest.mark.parametrize('res,widest', [((4096, 2), 4096), ((2420, 2, 4), 2420)])
def test_ring_width_limit(res, widest):
    """The widest line runs; one float4 group more is refused with the limit in the message."""
    from phiflow_b200 import _lib
    u0, v0 = rand_state((1,) + res, 6)
    dx = (1.0,) * len(res)
    bc = ((P, P),) * len(res)
    u, v, info = gpu_run(u0, v0, bc, dx, MAZE, 0.5, 2)
    ou, ov = rd_oracle(u0[0], v0[0], bc, dx, dt=0.5, substeps=2, **MAZE)
    assert np.array_equal(u[0], ou) and np.array_equal(v[0], ov)
    wider = (widest + 4,) + res[1:]
    u0, v0 = rand_state((1,) + wider, 6)
    with pytest.raises(_lib.Unsupported, match=f'at most {widest} cells'):
        gpu_run(u0, v0, bc, dx, MAZE, 0.5, 2)


# ---- the mirror ----------------------------------------------------------------------------------------------------------------------
def check_mirror(flow):
    """flow.reaction_diffusion against the notebook's cell on mirror ops (examples/reaction_diffusion.py), one call of 20 substeps vs
    20 cells, on the example's initial state (u0 as both u and v) - within 20 one-substep bounds of the final state; the inputs stay
    as they were; boundaries outside the scope raise NotImplementedError."""
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    try:
        import importlib
        import reaction_diffusion as ex
        importlib.reload(ex)
    finally:
        sys.path.remove(os.path.join(ROOT, 'examples'))
    u0 = ex.initial_state()
    before = u0.numpy().copy()
    fu, fv = flow.reaction_diffusion(u0, u0, dt=.5, substeps=20, **ex.PARAMS['maze'])
    cu, cv = u0, u0
    for _ in range(20):
        cu, cv = ex.reaction_diffusion_cell(cu, cv, dt=.5, **ex.PARAMS['maze'])
    assert np.array_equal(u0.numpy(), before)
    for e in range(3):
        bu, bv = step_bound(cu.numpy()[e], cv.numpy()[e], u0.spec, u0.dx, ex.PARAMS['maze'], 0.5)
        assert np.all(np.abs(fu.numpy()[e] - cu.numpy()[e]) <= 20 * bu) and np.all(np.abs(fv.numpy()[e] - cv.numpy()[e]) <= 20 * bv)
    assert fu.boundary == u0.boundary
    with pytest.raises(NotImplementedError, match='2c - c'):
        flow.reaction_diffusion(u0.with_extrapolation(flow.ONE), u0.with_extrapolation(flow.ONE), 0.19, 0.05, 0.06, 0.062, 0.5)
    with pytest.raises(NotImplementedError):
        flow.reaction_diffusion(u0.with_extrapolation(flow.PERIODIC), u0, 0.19, 0.05, 0.06, 0.062, 0.5)


def run_example(frames=3):
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    try:
        import importlib
        import reaction_diffusion as ex
        importlib.reload(ex)
        return {name: ex.run(name, frames) for name in ex.PARAMS}
    finally:
        sys.path.remove(os.path.join(ROOT, 'examples'))


def check_example(frames=3):
    out = run_example(frames)
    for name, (u, v) in out.items():
        assert u.shape == (frames + 1, 3, 100, 100) and v.shape == u.shape
        assert np.isfinite(u).all() and np.isfinite(v).all()
        assert not np.array_equal(u[-1], u[0])


@pytest.mark.gpu
def test_mirror():
    import phiflow_b200.flow as flow
    check_mirror(flow)


@pytest.mark.gpu
def test_example():
    check_example()
