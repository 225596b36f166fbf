"""
The wave step (the Waves notebook) on the H100: phicuda_wave_f32 against the oracle (tests/oracle_waves.py), its variants and
substeps bit for bit, its stamp, its refusals, and the mirror's flow.wave_step against the notebook's cell.

Error bound of one substep, derived from the operations (not fitted): the library's laplace differs from the oracle's only in
multiplying by fl(1 / fl(dx^2)) instead of dividing by fl(dx^2), at most 4 eps * S per cell with S = sum_d (|l| + |r| + 2 |c|) / dx_d^2
(`lap_scale` of tests/test_gpu_reaction_diffusion.py), scaled by dd * |k_speed| in h_n; the rounding of the five operations after
the laplace can move by one ulp each where their input moved, at most 4 eps * (|2 c - p| + dd (|k_speed lap| + |k_damp (c - p)|)).
The stamp is a selection and the disc test uses the same float32 operations as the oracle, so it adds nothing.  With dx = 1 both
laplaces are the same operations, and the library's substep is the float32 oracle's bit for bit.
"""
import os
import sys

import numpy as np
import pytest

from oracle_reaction_diffusion import laplace as lap_oracle
from oracle_waves import disc_mask, split_centres, wave as wave_oracle
from test_gpu_reaction_diffusion import lap_scale

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'phiml_waves.npz')
EPS = float(np.finfo(np.float32).eps)
P, Z = 'periodic', 'zg'
VALUE = np.float32(-0.5)
FIXED_POINT_CASES = ['zg', 'periodic', 'zero', 'aniso', 'batch']          # the fixture's cases without a non-zero constant


def _spec(arr):
    return tuple(tuple('periodic' if np.isnan(s) else ('zg' if np.isinf(s) else float(s)) for s in ax) for ax in arr)


def golden_case(g, name):
    """(hc0, hp0, bc, dx, dt, k_speed, k_damp, radius, centre or None, per-axis centres) of a fixture case."""
    hc0 = g[f'{name}/hc0']
    res = hc0.shape[1:]
    dx = tuple(float(u / n) for u, n in zip(g[f'{name}/upper'], res))
    dt, ks, kd, r = (float(x) for x in g[f'{name}/params'])
    centre = g[f'{name}/disc'] if f'{name}/disc' in g else None
    return hc0, g[f'{name}/hp0'], _spec(g[f'{name}/bc']), dx, dt, ks, kd, r, centre, g[f'{name}/centres']


def step_bound(hc, hp, bc, dx, dd, ks, kd):
    """Per-cell bound on |library - float32 oracle| for ONE substep from the stamped (hc, hp) (module docstring)."""
    c, p = hc.astype(np.float64), hp.astype(np.float64)
    lap = lap_oracle(hc, dx, bc, np.float64)
    return dd * abs(ks) * 4 * EPS * lap_scale(hc, dx, bc) + 4 * EPS * (np.abs(2 * c - p) + dd * (np.abs(ks * lap) + np.abs(kd * (c - p))))


def unit_centres(res):
    """Cell centres of a grid with dx = 1: 0.5, 1.5, ... along each axis."""
    return np.concatenate([np.arange(n, dtype=np.float32) + np.float32(0.5) for n in res])


def moving_discs(res, substeps, r=2.5, seed=0):
    """One disc per substep at seeded positions inside the grid, the odd ones absent when substeps > 2 (a gap in the source)."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(substeps):
        c = np.array([rng.uniform(0, n) for n in res], np.float32)
        out.append(None if (substeps > 2 and s % 3 == 2) else (c, VALUE))
    return out, np.float32(r * r)


def gpu_run(hc0, hp0, bc, dx, dd, ks, kd, discs, r2, centres, substeps, calls=1):
    """hc0, hp0: (batch, x, y[, z]).  Returns (h_c, h_p) after `calls` calls of `substeps` each (discs: calls * substeps entries),
    and the launch info of the last call."""
    from phiflow_b200 import _ops
    dom = _ops.Domain(hc0.shape[1:], dx, hc0.shape[0])
    hc, hp = dom.centered_from_numpy(hc0), dom.centered_from_numpy(hp0)
    for k in range(calls):
        hc, hp = _ops.wave(dom, bc, hc, hp, dd, ks, kd, discs[k * substeps:(k + 1) * substeps], r2, centres, substeps)
    return dom.centered_to_numpy(hc, squeeze=False), dom.centered_to_numpy(hp, squeeze=False), _ops.last_launch_info()


def oracle_run(hc0, hp0, bc, dx, dd, ks, kd, discs, r2, centres, dtype=np.float32):
    axes = split_centres(centres, hc0.shape)
    x, y = hc0, hp0
    for d in discs:
        m = disc_mask(axes, d[0], r2) if d is not None else None
        x, y = wave_oracle(x, y, bc, dx, dd, ks, kd, [m], d[1] if d is not None else 0.0, dtype=dtype)
    return x, y


def rand_state(shape, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-1, 1, shape).astype(np.float32), rng.uniform(-1, 1, shape).astype(np.float32)


# ---- one substep against the oracle ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('name', FIXED_POINT_CASES)
def test_one_substep_against_oracle(name):
    from phiflow_b200 import _lib
    hc0, hp0, bc, dx, dt, ks, kd, r, centre, centres = golden_case(np.load(GOLD), name)
    dd = np.float32(dt * dt)
    discs = [(centre, VALUE) if centre is not None else None]
    r2 = np.float32(r * r)
    hc, hp, info = gpu_run(hc0, hp0, bc, dx, dd, ks, kd, discs, r2, centres, 1)
    assert info['kernel'] == _lib.KERNEL_WAVE_RING
    axes = split_centres(centres, hc0.shape[1:])
    for b in range(hc0.shape[0]):
        on, oc = oracle_run(hc0[b], hp0[b], bc, dx, dd, ks, kd, discs, r2, centres)
        m = disc_mask(axes, centre, r2) if centre is not None else np.zeros(hc0.shape[1:], bool)
        bound = step_bound(np.where(m, VALUE, hc0[b]), np.where(m, VALUE, hp0[b]), bc, dx, dd, ks, kd)
        assert np.array_equal(hp[b], oc)                                       # the stamped h_c, exactly
        assert np.all(np.abs(hc[b] - on) <= bound)
        if all(d == 1.0 for d in dx):
            assert np.array_equal(hc[b], on)


# ---- substeps and variants, bit for bit ----------------------------------------------------------------------------------------------
SHAPES = [((128, 64), ((P, P), (P, P))), ((100, 60), ((Z, Z), (0.0, 0.0))), ((37, 23), ((0.0, Z), (Z, Z))),
          ((64, 24, 20), ((P, P), (Z, 0.0), (0.0, Z))), ((128, 32, 24), ((P, P), (P, P), (Z, Z)))]


@pytest.mark.gpu
@pytest.mark.parametrize('res,bc', SHAPES)
@pytest.mark.parametrize('K', [1, 2, 3, 4])
def test_k_substeps_equal_k_calls_and_oracle(res, bc, K):
    """K substeps in one call = K calls of one substep, bit for bit, for both parities; both equal the float32 oracle (dx = 1)."""
    hc0, hp0 = rand_state((2,) + res, K)
    dx = (1.0,) * len(res)
    discs, r2 = moving_discs(res, K, seed=K)
    centres = unit_centres(res)
    one = gpu_run(hc0, hp0, bc, dx, 0.2, 1.0, 0.1, discs, r2, centres, K)
    many = gpu_run(hc0, hp0, bc, dx, 0.2, 1.0, 0.1, discs, r2, centres, 1, calls=K)
    assert np.array_equal(one[0], many[0]) and np.array_equal(one[1], many[1])
    for b in range(2):
        oc, op = oracle_run(hc0[b], hp0[b], bc, dx, 0.2, 1.0, 0.1, discs, r2, centres)
        assert np.array_equal(one[0][b], oc) and np.array_equal(one[1][b], op)


@pytest.mark.gpu
@pytest.mark.parametrize('res,bc,knobs', [
    ((128, 96), ((P, P), (P, P)), [{}, {'PHICUDA_RING_TY': '5'}, {'PHICUDA_RING_TY': '2'}, {'PHICUDA_RING_TY': '32'}]),
    ((100, 50), ((Z, Z), (0.0, 0.0)), [{}, {'PHICUDA_RING_TY': '3'}, {'PHICUDA_RING_TY': '8'}]),
    ((128, 32, 24), ((P, P), (P, P), (P, P)), [{}, {'PHICUDA_RING_TY': '3'}, {'PHICUDA_RING_NZC': '1'}, {'PHICUDA_RING_NZC': '5'},
                                              {'PHICUDA_RING_TY': '1', 'PHICUDA_RING_NZC': '3'}]),
    ((60, 20, 10), ((0.0, Z), (Z, 0.0), (P, P)), [{}, {'PHICUDA_RING_TY': '3'}, {'PHICUDA_RING_NZC': '1'}]),
])
def test_identical_across_tilings_and_variants(res, bc, knobs, monkeypatch):
    """Every tiling and both the generic and the branch-free variant (phicuda_last_launch_info) give the same bits."""
    hc0, hp0 = rand_state((2,) + res, 3)
    dx = (1.0,) * len(res)
    discs, r2 = moving_discs(res, 5, r=6.0, seed=3)
    outs, variants = [], set()
    for kn in knobs:
        for key in ('PHICUDA_RING_TY', 'PHICUDA_RING_NZC'):
            monkeypatch.delenv(key, raising=False)
        for key, val in kn.items():
            monkeypatch.setenv(key, val)
        hc, hp, info = gpu_run(hc0, hp0, bc, dx, 0.2, 1.0, 0.0, discs, r2, unit_centres(res), 5)
        outs.append((hc, hp))
        variants.add((info['generic'], info['TY'], info['nzc']))
    assert len(variants) == len(knobs)
    if bc[0][0] == P:
        assert {v[0] for v in variants} == {0, 1}                    # both variants ran
    for hc, hp in outs[1:]:
        assert np.array_equal(hc, outs[0][0]) and np.array_equal(hp, outs[0][1])


@pytest.mark.gpu
@pytest.mark.parametrize('res,bc,centre', [((64, 48), ((Z, Z), (Z, Z)), (0.3, 20.0)), ((128, 64), ((P, P), (P, P)), (127.9, 63.8)),
                                           ((40, 30, 20), ((Z, Z), (P, P), (0.0, 0.0)), (20.0, 0.2, 19.5))])
def test_stamp_exactly_where_the_mask_is_set(res, bc, centre):
    """After one substep the returned previous state is value exactly on the oracle's mask (a disc over a wall / corner) and the
    caller's h_c everywhere else."""
    hc0, hp0 = rand_state((1,) + res, 7)
    r2 = np.float32(4.7 ** 2)
    centres = unit_centres(res)
    _, hp, _ = gpu_run(hc0, hp0, bc, (1.0,) * len(res), 0.2, 1.0, 0.0, [(np.array(centre, np.float32), VALUE)], r2, centres, 1)
    m = disc_mask(split_centres(centres, res), centre, r2)
    assert m.any() and not m.all()
    assert np.all(hp[0][m] == VALUE) and np.array_equal(hp[0][~m], hc0[0][~m])


# ---- the notebook ---------------------------------------------------------------------------------------------------------------------
def load_example():
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    try:
        import importlib
        import waves as ex
        return importlib.reload(ex)
    finally:
        sys.path.remove(os.path.join(ROOT, 'examples'))


@pytest.mark.gpu
def test_notebook_against_float64():
    """The notebook's 300 frames of 16 substeps (examples/waves.py, fused): the library's distance from the float64 oracle (same
    discs and masks) is at most 2x the float32 oracle's own distance from it, plus 1e-6 where that is ~0.  The first two frames equal
    the fixture within 32 one-substep bounds."""
    ex = load_example()
    h, _ = ex.run(300)
    g = np.load(GOLD)
    centres = g['notebook/axis_centres']
    discs = [(c, VALUE) for c in g['notebook/centres']]
    bc, dx, dd = ((Z, Z), (Z, Z)), (0.1, 0.1), np.float32(ex.DT * ex.DT)
    zero = np.zeros((128, 128), np.float32)
    o32 = oracle_run(zero, zero, bc, dx, dd, 1.0, 0.0, discs, np.float32(1.0), centres)[0]
    o64 = oracle_run(zero, zero, bc, dx, dd, 1.0, 0.0, discs, np.float32(1.0), centres, dtype=np.float64)[0]
    assert np.abs(h[-1] - o64).max() <= 2 * np.abs(o32 - o64).max() + 1e-6
    for f in (1, 2):
        ref = g[f'notebook/f{f}/hn']
        assert np.abs(h[f] - ref).max() <= 32 * 4 * EPS * (np.abs(ref).max() + 1.0)


def check_mirror(flow, frames=2):
    """flow.wave_step against the notebook's cell on mirror ops (examples/waves.py), and the mirror's refusals."""
    ex = load_example()
    hf, tf = ex.run(frames)
    hc, tc = ex.run(frames, cell=True)
    assert tf == tc
    assert np.abs(hf - hc).max() <= 1e-6 * frames
    assert np.abs(hf[-1]).max() > 0.1
    h0 = ex.initial_state()
    n, c, t = flow.wave_step(h0, h0, 0, ex.DT, substeps=0)
    assert t == 0 and np.array_equal(n.numpy(), h0.numpy()) and n.boundary == h0.boundary
    with pytest.raises(NotImplementedError, match='c - c'):
        flow.wave_step(h0.with_extrapolation(flow.ONE), h0.with_extrapolation(flow.ONE), 0, ex.DT)
    with pytest.raises(NotImplementedError):
        flow.wave_step(h0, h0.with_extrapolation(flow.PERIODIC), 0, ex.DT)
    with pytest.raises(NotImplementedError):
        flow.wave_step(h0, h0, 0, ex.DT, source=lambda t: (flow.Box(x=(1, 2), y=(1, 2)), -0.5))


@pytest.mark.gpu
def test_mirror():
    import phiflow_b200.flow as flow
    check_mirror(flow, frames=5)


# ---- other checks --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_zero_substeps_same_array_refusals_and_inputs():
    import ctypes
    import torch
    from phiflow_b200 import _lib, _ops
    res = (64, 32)
    hc0, hp0 = rand_state((2,) + res, 5)
    dom = _ops.Domain(res, (1.0, 1.0), 2)
    hc, hp = dom.centered_from_numpy(hc0), dom.centered_from_numpy(hp0)
    cc, pc = hc.clone(), hp.clone()
    centres = unit_centres(res)
    discs, r2 = moving_discs(res, 3)
    n, c = _ops.wave(dom, ((P, P), (P, P)), hc, hp, 0.2, 1.0, 0.0, [], r2, centres, 0)
    assert torch.equal(n, hc) and torch.equal(c, hp)
    n, c = _ops.wave(dom, ((P, P), (P, P)), hc, hp, 0.2, 1.0, 0.0, discs, r2, centres, 3)
    assert torch.equal(hc, cc) and torch.equal(hp, pc) and not torch.equal(n, hc)           # inputs not modified
    same = _ops.wave(dom, ((P, P), (P, P)), hc, hc, 0.2, 1.0, 0.0, discs, r2, centres, 3)    # h_c is h_p, as the notebook starts
    ref = gpu_run(hc0, hc0, ((P, P), (P, P)), (1.0, 1.0), 0.2, 1.0, 0.0, discs, r2, centres, 3)
    assert np.array_equal(dom.centered_to_numpy(same[0], squeeze=False), ref[0])
    assert np.array_equal(dom.centered_to_numpy(same[1], squeeze=False), ref[1])
    # refusals through the C ABI with real device arrays leave them untouched
    lib = _lib.load()
    scratch = torch.empty(lib.phicuda_wave_scratch_bytes(ctypes.byref(dom.grid), 3) // 4 + 1, dtype=torch.float32, device='cuda')
    table = (_lib.PhiWaveDisc * 3)()
    for t in table:
        t.present, t.value = 1, -0.5
        t.center[0], t.center[1] = 30.0, 10.0
    cs = np.ascontiguousarray(centres)

    def call(spec=((P, P), (P, P)), substeps=3, dd=0.2):
        return lib.phicuda_wave_f32(ctypes.byref(dom.grid), ctypes.byref(_ops.make_bc(spec)), _ops._ptr(hc), _ops._ptr(hp), dd, 1.0, 0.0,
                                    table, 1.0, cs.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), substeps, _ops._ptr(scratch),
                                    scratch.numel() * 4, _ops._stream())
    assert call(((0.3, 0.3), (P, P))) == _lib.ERR_UNSUPPORTED
    assert call(substeps=-1) == _lib.ERR_INVALID
    assert call(dd=float('nan')) == _lib.ERR_INVALID
    table[1].value = float('inf')
    assert call() == _lib.ERR_INVALID
    torch.cuda.synchronize()
    assert torch.equal(hc, cc) and torch.equal(hp, pc)
