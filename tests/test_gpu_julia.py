"""
Julia sets (the Julia_Set notebook) on the H100: phicuda_julia_f32 against PhiML 1.7.2's counts in tests/golden/phiml_julia.npz, bit
for bit on every case (the fixture, never a live NumPy run: NumPy's complex64 rounding depends on the CPU's SIMD dispatch), its launch
record, zero iterations, non-square and ragged grids against the oracle, refusals that leave the counts untouched, and
examples/julia_set.py.
"""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'phiml_julia.npz')
CASES = ['notebook', 'band_x', 'band_y', 'band_diag', 'iter0', 'iter1', 'iter50', 'big_c', 'nonfinite']


def golden_case(g, name):
    """(complex64 constants, per-axis centres, (n_x, n_y), iterations, int32 counts (batch, x, y)) of a fixture case."""
    c = np.ascontiguousarray(g[f'{name}/c']).view(np.complex64).reshape(-1)
    counts = g[f'{name}/counts'].astype(np.int32)
    return c, g[f'{name}/centres'], counts.shape[1:], int(g[f'{name}/iterations']), counts


def _run(res, centres, c, iterations, out=None):
    import torch
    from phiflow_b200 import _ops
    dom = _ops.Domain(res, (1.0, 1.0), len(c))
    counts = _ops.julia(dom, centres, c, iterations, out=out)
    torch.cuda.synchronize()
    return dom, counts


def _to_numpy(dom, t):
    return dom.centered_to_numpy(t, squeeze=False)


@pytest.mark.gpu
@pytest.mark.parametrize('name', CASES)
def test_counts_match_phiml(name):
    from phiflow_b200 import _lib, _ops
    c, centres, res, iterations, counts = golden_case(np.load(GOLD), name)
    dom, got = _run(res, centres, c, iterations)
    assert got.dtype.is_signed and got.element_size() == 4
    np.testing.assert_array_equal(_to_numpy(dom, got), counts)
    assert _ops.last_launch_info()['kernel'] == _lib.KERNEL_JULIA


@pytest.mark.gpu
def test_zero_iterations_write_zeros_and_only_owned_cells():
    import torch
    from oracle_julia import julia_counts
    res = (37, 23)                                       # cext[0] = 40: three padding columns per row
    centres = np.concatenate([np.linspace(-1.9, 1.7, res[0], dtype=np.float32), np.linspace(-1.1, 1.3, res[1], dtype=np.float32)])
    c = np.array([0.3 + 0.5j, -0.8 + 0.156j], np.complex64)
    from phiflow_b200 import _ops
    dom = _ops.Domain(res, (1.0, 1.0), len(c))
    out = torch.full(dom._shape(dom.cext), -7, dtype=torch.int32, device='cuda')
    _ops.julia(dom, centres, c, 0, out=out)
    torch.cuda.synchronize()
    assert (out[:, :, :res[0]] == 0).all() and (out[:, :, res[0]:] == -7).all()
    _ops.julia(dom, centres, c, 9, out=out)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(_to_numpy(dom, out), julia_counts(centres[:res[0]], centres[res[0]:], c, 9))
    assert (out[:, :, res[0]:] == -7).all()


@pytest.mark.gpu
@pytest.mark.parametrize('res,batch,iterations', [((5, 3), 1, 50), ((129, 7), 3, 20), ((300, 130), 2, 64), ((1, 1), 4, 30)])
def test_non_square_and_ragged_grids(res, batch, iterations):
    from oracle_julia import julia_counts
    rng = np.random.default_rng(sum(res) + batch)
    centres = np.concatenate([np.sort(rng.uniform(-2.2, 2.2, n)).astype(np.float32) for n in res])
    c = (rng.uniform(-1, 1, batch) + 1j * rng.uniform(-1, 1, batch)).astype(np.complex64)
    dom, got = _run(res, centres, c, iterations)
    np.testing.assert_array_equal(_to_numpy(dom, got), julia_counts(centres[:res[0]], centres[res[0]:], c, iterations))


@pytest.mark.gpu
def test_offsets_beyond_2_31():
    """4096^2 x 136 cells: counts at offsets past 2^31 land where the oracle puts them (seeded cells, most in the last entries)."""
    import torch
    from oracle_julia import abs32, square_plus
    n, batch, iterations = 4096, 136, 4
    axis = np.linspace(np.float32(0.5 / n), np.float32(1 - 0.5 / n), n, dtype=np.float32) * np.float32(4) + np.float32(-2)
    c = (0.7885 * np.exp(1j * np.linspace(0, 2 * np.pi, batch))).astype(np.complex64)
    dom, got = _run((n, n), np.concatenate([axis, axis]), c, iterations)
    rng = np.random.default_rng(3)
    b = np.concatenate([rng.integers(0, batch, 512), rng.integers(batch - 8, batch, 1536)])
    x, y = rng.integers(0, n, b.size), rng.integers(0, n, b.size)
    off = (b.astype(np.int64) * n + y) * n + x
    assert (off >= 2 ** 31).sum() >= 1024
    za, zb, want = axis[x].copy(), axis[y].copy(), np.zeros(b.size, np.int32)
    for _ in range(iterations):
        want += abs32(za, zb) < np.float32(2)
        za, zb = square_plus(za, zb, c.real[b], c.imag[b])
    np.testing.assert_array_equal(got.view(-1)[torch.from_numpy(off).cuda()].cpu().numpy(), want)


@pytest.mark.gpu
def test_refusals_leave_counts_untouched():
    import torch
    from phiflow_b200 import _lib, _ops
    res, c = (16, 8), np.array([0.2 + 0.1j, 0.3 - 0.4j], np.complex64)
    dom = _ops.Domain(res, (1.0, 1.0), 2)
    out = torch.full(dom._shape(dom.cext), 5, dtype=torch.int32, device='cuda')
    lib = _lib.load()
    need = lib.phicuda_julia_scratch_bytes(C.byref(dom.grid))
    scratch = torch.empty(need, dtype=torch.uint8, device='cuda')
    good = np.linspace(-2, 2, sum(res), dtype=np.float32)
    pairs = c.view(np.float32)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    calls = [
        (good, -1, need, 'iterations'),
        (np.where(np.arange(good.size) == 3, np.float32(np.nan), good).astype(np.float32), 5, need, 'cell centre'),
        (good, 5, need - 4, 'scratch'),
    ]
    for centres, iterations, nbytes, word in calls:
        e = lib.phicuda_julia_f32(C.byref(dom.grid), fp(centres), fp(pairs), iterations, C.c_void_p(out.data_ptr()),
                                  C.c_void_p(scratch.data_ptr()), C.c_size_t(nbytes), stream)
        assert e == _lib.ERR_INVALID and word in _lib.last_error()
    e = lib.phicuda_julia_f32(C.byref(dom.grid), fp(good), fp(pairs), 5, C.c_void_p(out.data_ptr()), C.c_void_p(out.data_ptr() + 64),
                              C.c_size_t(need), stream)
    assert e == _lib.ERR_INVALID and 'overlaps' in _lib.last_error()
    torch.cuda.synchronize()
    assert (out == 5).all()


@pytest.mark.gpu
def test_example_gives_the_fixture():
    """examples/julia_set.py at the notebook's size (100 constants, 256 x 256): the fixture's picked constants, count for count.  Its
    constants come from NumPy's complex64 exp on the host; they are compared with the fixture's where NumPy dispatches as recorded."""
    from numpy._core._multiarray_umath import __cpu_dispatch__, __cpu_features__
    g = np.load(GOLD)
    spec = importlib.util.spec_from_file_location('example_julia_set', os.path.join(ROOT, 'examples', 'julia_set.py'))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    c_fixture = np.ascontiguousarray(g['notebook/c_all']).view(np.complex64).reshape(-1)
    counts = ex.sample(c_fixture).numpy()
    assert counts.shape == (100, 256, 256) and counts.dtype == np.int32
    np.testing.assert_array_equal(counts[g['notebook/pick']], g['notebook/counts'].astype(np.int32))
    if ' '.join(f for f in __cpu_dispatch__ if __cpu_features__[f]) == str(g['numpy/simd_found']):
        assert np.array_equal(np.asarray(ex.constants()).view(np.float32).reshape(-1, 2), g['notebook/c_all'])
