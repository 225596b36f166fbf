"""
The wave step without a GPU: the oracle against PhiML 1.7.2 (tests/golden/phiml_waves.npz), the host's disc centres and masks, the
boundary records, argument validation of phicuda_wave_f32, and the mirror, the notebook's own cell and examples/waves.py over the
oracle-backed engine.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import phiflow_b200.flow as flow
import test_gpu_waves as G
from oracle_waves import WaveOracleEngine, disc_mask, split_centres, wave
from phiflow_b200 import _lib

P, Z = 'periodic', 'zg'
CASES = ['zg', 'periodic', 'zero', 'const', 'const2', 'aniso', 'ragged', 'batch', 'mixed3', 'aniso3']


# ---- oracle and host construction vs PhiML ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_phiml(name):
    """One substep, every case: the float32 oracle is PhiML's result bit for bit (h_n and the stamped h_c)."""
    g = np.load(G.GOLD)
    hc0, hp0, bc, dx, dt, ks, kd, r, centre, centres = G.golden_case(g, name)
    m = disc_mask(split_centres(centres, hc0.shape[1:]), centre, np.float32(r * r)) if centre is not None else None
    for b in range(hc0.shape[0]):
        hn, hc = wave(hc0[b], hp0[b], bc, dx, np.float32(dt * dt), ks, kd, [m], G.VALUE)
        assert np.array_equal(hn, g[f'{name}/hn'][b]) and np.array_equal(hc, g[f'{name}/hc'][b])


@pytest.mark.parametrize('name', CASES)
def test_mirror_centres_and_mask_match_phiml(name, oracle_mirror):
    """CenteredGrid.axis_centres and Sphere.lies_inside of the mirror give the fixture's float32 cell centres and mask."""
    g = np.load(G.GOLD)
    hc0, _, _, _, _, _, _, r, centre, centres = G.golden_case(g, name)
    res = hc0.shape[1:]
    grid = flow.CenteredGrid(0, flow.ZERO, flow.Box(**{a: float(u) for a, u in zip('xyz', g[f'{name}/upper'])}), **dict(zip('xyz', res)))
    assert np.array_equal(np.concatenate(grid.axis_centres()), centres)
    if centre is not None:
        assert np.array_equal(flow.Sphere(center=centre, radius=r).lies_inside(np.stack(np.meshgrid(*grid.axis_centres(), indexing='ij'), -1)), g[f'{name}/mask'])


def test_notebook_centres_and_masks_match_phiml(oracle_mirror):
    """All 4800 disc centres of the notebook's run (Box.center + rotate_vector at the substep's Python-float time) and the first
    32 masks, through the example's own source function."""
    g = np.load(G.GOLD)
    ex = G.load_example()
    h0 = ex.initial_state()
    src = ex.source(h0.bounds)
    time, dt = 0, ex.DT
    centres = []
    for s in range(4800):
        sphere, value = src(time)
        centres.append(np.asarray(sphere.center, np.float32))
        if s < 32:
            assert np.array_equal(sphere.lies_inside(np.stack(np.meshgrid(*h0.axis_centres(), indexing='ij'), -1)), g['notebook/masks'][s])
            assert np.float32(value) == g['notebook/value']
        time = time + dt
    assert np.array_equal(np.stack(centres), g['notebook/centres'])


def test_boundary_records():
    """The reference's extrapolation of h_n: ZERO, ZERO_GRADIENT and PERIODIC are fixed points, a constant c becomes 0."""
    g = np.load(G.GOLD)
    assert str(g['ext/zg']) == 'zero-gradient' and str(g['ext/periodic']) == 'periodic' and str(g['ext/zero']) == '0'
    assert float(str(g['ext/c0.3'])) == 0.0 and float(str(g['ext/c-0.7'])) == 0.0


def test_disc_struct_matches_c():
    src = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "phicuda.h"
    int main(void) { printf("%zu %zu %zu\n", sizeof(PhiWaveDisc), offsetof(PhiWaveDisc, value), offsetof(PhiWaveDisc, present)); return 0; }'''
    with tempfile.TemporaryDirectory() as tmp:
        c, exe = os.path.join(tmp, 's.c'), os.path.join(tmp, 's')
        with open(c, 'w') as f:
            f.write(src)
        subprocess.check_call(['gcc', '-I', os.path.join(G.ROOT, 'include'), c, '-o', exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    assert sizes == [C.sizeof(_lib.PhiWaveDisc), _lib.PhiWaveDisc.value.offset, _lib.PhiWaveDisc.present.offset]


# ---- C ABI validation (no CUDA call is reached) -----------------------------------------------------------------------------------
def _grid(dim=2, n=(16, 8, 4), halo=0):
    g = _lib.PhiGrid()
    g.dim, g.batch, g.halo = dim, 2, halo
    for a in range(dim):
        g.n[a] = n[a]
        g.cext[a] = g.fext[a] = n[a] + (2 * halo if a == 2 else 0)
        g.dx[a] = 1.0
    return g


def _call(g=None, spec=((P, P), (P, P)), hc=16 << 20, hp=32 << 20, scratch=48 << 20, substeps=3, short=0, dd=0.2, kd=0.0,
          value=-0.5, centre=(3.0, 4.0, 1.0), centres=None, discs=True, null_bc=False):
    from phiflow_b200 import _ops
    lib = _lib.load()
    g = g or _grid()
    need = lib.phicuda_wave_scratch_bytes(C.byref(g), max(substeps, 0))
    table = (_lib.PhiWaveDisc * max(substeps, 1))()
    for t in table:
        t.present, t.value = 1, value
        for a in range(3):
            t.center[a] = centre[a]
    cs = np.ascontiguousarray(G.unit_centres(tuple(g.n[a] for a in range(g.dim))) if centres is None else centres, np.float32)
    bc = None if null_bc else C.byref(_ops.make_bc(spec))
    # addresses are never dereferenced: validation fails first (or substeps == 0 returns before any CUDA call)
    return lib.phicuda_wave_f32(C.byref(g), bc, C.c_void_p(hc), C.c_void_p(hp), dd, 1.0, kd, table if discs else None, 1.0,
                                cs.ctypes.data_as(C.POINTER(C.c_float)), substeps, C.c_void_p(scratch), C.c_size_t(need - short), None)


@pytest.mark.parametrize('kw,code,word', [
    ({'hc': 0}, _lib.ERR_INVALID, 'NULL'),
    ({'scratch': 0}, _lib.ERR_INVALID, 'NULL'),
    ({'null_bc': True}, _lib.ERR_INVALID, 'NULL'),
    ({'discs': False}, _lib.ERR_INVALID, 'NULL'),
    ({'short': 4}, _lib.ERR_INVALID, 'scratch'),
    ({'hp': 16 << 20}, _lib.ERR_INVALID, 'distinct'),
    ({'hp': (16 << 20) + 64}, _lib.ERR_INVALID, 'distinct'),
    ({'scratch': (32 << 20) - 64}, _lib.ERR_INVALID, 'overlaps'),
    ({'substeps': -1}, _lib.ERR_INVALID, 'substeps'),
    ({'dd': float('inf')}, _lib.ERR_INVALID, 'finite'),
    ({'kd': float('nan')}, _lib.ERR_INVALID, 'finite'),
    ({'value': float('nan')}, _lib.ERR_INVALID, 'disc 0'),
    ({'centre': (float('inf'), 1.0, 1.0)}, _lib.ERR_INVALID, 'disc 0'),
    ({'centres': np.full(24, np.nan, np.float32)}, _lib.ERR_INVALID, 'cell centre'),
    ({'spec': ((0.3, 0.0), (P, P))}, _lib.ERR_UNSUPPORTED, 'c - c = 0'),
    ({'spec': ((0.0, 0.0), (P, -1.0))}, _lib.ERR_INVALID, 'PERIODIC'),
    ({'g': _grid(3, halo=1), 'spec': ((P, P), (P, P), (P, P))}, _lib.ERR_UNSUPPORTED, 'z-slab'),
])
def test_argument_validation_without_gpu(kw, code, word):
    assert _call(**kw) == code
    assert word in _lib.last_error()


def test_zero_substeps_returns_before_any_cuda_call():
    assert _call(substeps=0) == 0


def test_no_ring_is_refused(monkeypatch):
    monkeypatch.setenv('PHICUDA_NO_RING', '1')
    assert _call() == _lib.ERR_UNSUPPORTED and 'PHICUDA_NO_RING' in _lib.last_error()


@pytest.mark.parametrize('dim,widest', [(2, 4096), (3, 3628)])
def test_ring_width_limit_is_named(dim, widest):
    assert _call(_grid(dim, (widest, 4, 4)), spec=((P, P),) * dim, substeps=0) == 0
    assert _call(_grid(dim, (widest + 4, 4, 4)), spec=((P, P),) * dim) == _lib.ERR_UNSUPPORTED
    assert f'at most {widest} cells' in _lib.last_error()


# ---- the mirror, the notebook's cell and the example over the oracle engine ------------------------------------------------------
@pytest.fixture()
def oracle_mirror():
    saved = flow.ops, flow._DEVICE
    flow.ops = WaveOracleEngine
    flow.set_device('cpu')
    try:
        yield
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])


def test_mirror(oracle_mirror):
    G.check_mirror(flow)


def test_example_matches_phiml(oracle_mirror):
    """examples/waves.py, fused and --cell, equals the fixture's first two frames bit for bit over the oracle engine."""
    g = np.load(G.GOLD)
    ex = G.load_example()
    for cell in (False, True):
        h, t = ex.run(2, cell=cell)
        assert np.array_equal(h[1], g['notebook/f1/hn']) and np.array_equal(h[2], g['notebook/f2/hn'])
    ex.main(1)
