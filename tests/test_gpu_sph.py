"""
SPH (DESIGN.md row N12) on the GPU: phicuda_sph_f32 against the NumPy restatement (tests/oracle_sph.py) bit for bit, on every fixture
case, the notebook's initial state and 2^20 particles; substeps fused and split, launch geometries, unsafe positions, refusals that
leave the outputs untouched, and examples/sph.py for the notebook's full 480 x 40 substeps.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_sph as O
from phiflow_b200 import _lib, _ops
from test_sph_host import GOLD, cases, golden_params, load_example

pytestmark = pytest.mark.gpu
F = np.float32


def c_params(prm):
    """PhiSphParams of an oracle parameter dict."""
    p = _lib.PhiSphParams()
    d = len(prm['lower'])
    for a in range(d):
        p.lower[a], p.upper[a], p.gravity[a] = prm['lower'][a], prm['upper'][a], prm['gravity'][a]
    p.support, p.smoothing_length, p.kernel_norm, p.mass = prm['s'], prm['h'], prm['norm'], prm['m']
    p.pressure_norm, p.viscous_norm, p.isotropic_exp, p.base_density = prm['P'], prm['V'], prm['iso'], prm['base']
    p.dt, p.damping = prm['dt'], prm['damping']
    return p


def gpu(x, v, prm, substeps):
    xo, vo, rho = _ops.sph(torch.from_numpy(x).cuda(), torch.from_numpy(v).cuda(), c_params(prm), substeps, rho=True)
    torch.cuda.synchronize()
    return xo.cpu().numpy(), vo.cpu().numpy(), rho.cpu().numpy()


def same(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize('name', cases())
def test_fixture_cases_match_oracle(name):
    g = np.load(GOLD)
    prm = golden_params(g, name)
    x0, v0 = g[f'{name}/x0'], g[f'{name}/v0']
    k = int(g[f'{name}/substeps'])
    want = O.sph(x0, v0, prm, k)
    got = gpu(x0, v0, prm, k)
    assert _ops.last_launch_info()['kernel'] == _lib.KERNEL_SPH
    for a, b in zip(got, want):
        assert same(a, b)


@pytest.mark.parametrize('substeps', [1, 40])
def test_notebook_initial_state(substeps):
    x0 = O.notebook_lattice()
    v0 = np.zeros_like(x0)
    prm = O.notebook_params(3)
    want = O.sph(x0, v0, prm, substeps)
    got = gpu(x0, v0, prm, substeps)
    for a, b in zip(got, want):
        assert same(a, b)


def test_fused_equals_one_launch_per_substep():
    g = np.load(GOLD)
    for name in ('special3_1', 'special2_1', 'lattice3_1'):
        prm = golden_params(g, name)
        x, v = g[f'{name}/x0'], g[f'{name}/v0']
        fused = gpu(x, v, prm, 7)
        for _ in range(7):
            x, v, rho = gpu(x, v, prm, 1)
        assert same(fused[0], x) and same(fused[1], v) and same(fused[2], rho)


def test_runs_and_launch_geometries_give_identical_bits(monkeypatch):
    rng = np.random.default_rng(3)
    n = 50000
    x = (rng.random((n, 3)) * 30).astype(F)          # ~ 1 particle per cell, several in many
    v = (rng.standard_normal((n, 3)) * 0.5).astype(F)
    prm = O.notebook_params(3, upper=(30.,) * 3)
    ref = gpu(x, v, prm, 6)
    ctas = _ops.last_launch_info()['grid_ctas']
    assert ctas > 3
    assert all(same(a, b) for a, b in zip(gpu(x, v, prm, 6), ref))
    monkeypatch.setenv('PHICUDA_SPH_CTAS', '3')
    assert all(same(a, b) for a, b in zip(gpu(x, v, prm, 6), ref))
    assert _ops.last_launch_info()['grid_ctas'] == 3
    want = O.sph(x, v, prm, 6)
    assert all(same(a, b) for a, b in zip(ref, want))


def test_two_to_the_twenty_particles_sampled():
    rng = np.random.default_rng(5)
    n = 1 << 20
    x = (rng.random((n, 3)) * 72).astype(F)
    v = (rng.standard_normal((n, 3)) * 0.1).astype(F)
    prm = O.notebook_params(3, upper=(72.,) * 3)
    got = gpu(x, v, prm, 1)
    rows = np.sort(rng.choice(n, 4000, replace=False))
    xo, vo, rho, _ = O.sph_substep(x, v, prm, rows)
    assert same(got[0][rows], xo) and same(got[1][rows], vo) and same(got[2][rows], rho)


def test_unsafe_positions():
    """NaN, +-inf, far outside and a crowd in one cell: no out-of-range access, and the oracle's values."""
    g = np.load(GOLD)
    prm = golden_params(g, 'special3_1')
    x = g['special3_1/x0'].copy()
    v = g['special3_1/v0'].copy()
    x[3] = (np.nan, 1.0, 1.0)
    x[4] = (np.inf, -np.inf, 2.0)
    x[5] = (-1e30, 1e30, 2.0)
    x[6] = (-3.0, 2.0, 9.0)
    crowd = np.full((300, 3), 3.9, F) + np.linspace(0, 0.05, 300, dtype=F)[:, None]
    x = np.concatenate([x, crowd]).astype(F)
    v = np.concatenate([v, np.zeros_like(crowd)]).astype(F)
    with np.errstate(all='ignore'):
        want = O.sph(x, v, prm, 3)
    got = gpu(x, v, prm, 3)
    for a, b in zip(got, want):
        assert same(a, b)


def test_refused_calls_leave_outputs_untouched():
    lib = _lib.load()
    prm = O.notebook_params(3, upper=(8.,) * 3)
    p = c_params(prm)
    n = 64
    x = torch.rand(n, 3, device='cuda') * 8
    v = torch.zeros(n, 3, device='cuda')
    xo, vo, ro = (torch.full((n, 3), 7.0, device='cuda'), torch.full((n, 3), 7.0, device='cuda'), torch.full((n,), 7.0, device='cuda'))
    need = lib.phicuda_sph_scratch_bytes(n, 3, C.byref(p))
    scratch = torch.empty(need, dtype=torch.uint8, device='cuda')
    ptr = lambda t: C.c_void_p(t.data_ptr())

    def call(substeps=2, nbytes=need, xo_=xo, prm_=p):
        return lib.phicuda_sph_f32(ptr(x), ptr(v), n, 3, C.byref(prm_), substeps, ptr(xo_), ptr(vo), ptr(ro), ptr(scratch), nbytes, None)

    bad = c_params(prm)
    bad.support = float('nan')
    for code in (call(substeps=0), call(nbytes=need - 1), call(xo_=x), call(prm_=bad)):
        assert code == _lib.ERR_INVALID, _lib.last_error()
    torch.cuda.synchronize()
    assert bool((xo == 7).all()) and bool((vo == 7).all()) and bool((ro == 7).all())
    assert call() == 0
    torch.cuda.synchronize()
    assert not bool((xo == 7).all())


def test_example_full_run():
    """examples/sph.py: the notebook's 480 frames x 40 substeps stay in the domain with finite values, and two runs give the same bits."""
    ex = load_example()
    a = ex.run()
    b = ex.run()
    x, v = a
    assert x.shape == (62500, 3)
    assert np.all((x >= 0) & (x <= 80)) and np.isfinite(x).all() and np.isfinite(v).all()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert np.abs(v).max() > 0
