"""
The fp64 path without a GPU: the float64 oracle, the C structs of the _f64 entry points, their argument checks (which run before any
CUDA call), the mirror in precision 64 and examples/taylor_green.py over the float64 oracle engine (tests/oracle_fp64.py), and the
refusal of every fp64 combination outside the path.  The kernels are tests/test_gpu_fp64.py's business.
"""
import ctypes as C
import importlib.util
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import oracle_np as O
from oracle_fp64 import Fp64OracleEngine, taylor_green_step
from phiflow_b200 import _lib, _ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the float64 oracle ---------------------------------------------------------------------------------------------------------

def test_oracle_honours_precision_64():
    """Every oracle function the fp64 path is compared with computes in float64 under precision(64)."""
    rng = np.random.default_rng(0)
    res, dx = (7, 5), (0.3, 2 * np.pi / 25)
    vbc = ((0.25, 'zg'), ('periodic', 'periodic'))
    lower, upper = (0.0, 0.0), tuple(n * h for n, h in zip(res, dx))
    v = [rng.standard_normal(s) for s in O.staggered_shapes(res, vbc)]
    s, p = rng.standard_normal(res), rng.standard_normal(res)
    with O.precision(64):
        outs = [O.laplace(s, dx, vbc), O.diffuse_explicit(s, vbc, dx, 0.1, 0.05), O.divergence_staggered(v, dx, O.component_bcs(vbc, 2)),
                O.semi_lagrangian_centered(s, vbc, v, vbc, lower, upper, 0.3)]
        outs += O.gradient_faces(p, dx, O.pressure_bc(vbc), vbc) + O.diffuse_explicit(v, vbc, dx, 0.1, 0.05)
        outs += O.semi_lagrangian_staggered(v, vbc, v, vbc, res, lower, upper, 0.3)
        A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
        info = O.cg(A, s.ravel(), np.zeros(s.size), 1e-12, 1e-12, 500)
        vn, pn, info2 = O.make_incompressible(v, vbc, res, dx, 1e-12, 1e-12, 500, use_matrix_offset=False)
    assert all(o.dtype == np.float64 for o in outs)
    assert A.dtype == np.float64 and info['x'].dtype == np.float64 and info['converged']
    assert pn.dtype == np.float64 and all(c.dtype == np.float64 for c in vn) and info2['converged']
    # and the float32 oracle is untouched outside the context
    assert O.laplace(s, dx, vbc).dtype == np.float32


GOLD = np.load(os.path.join(ROOT, 'tests', 'golden', 'phiml_fp64.npz'))
EPS = np.finfo(np.float64).eps


def spec_from_arr(arr):
    return tuple(tuple('periodic' if np.isnan(s) else ('zg' if np.isinf(s) else float(s)) for s in ax) for ax in arr)


def gold_names(prefix):
    return sorted({k.split('/')[1] for k in GOLD.files if k.startswith(prefix + '/')})


@pytest.mark.parametrize('name', gold_names('laplace'))
def test_fp64_oracle_stencils_match_phiml(name):
    """PhiML 1.7.2 under math.precision(64): laplace to a few float64 ulp, divergence and face gradient, grid_sample at back-traced
    points."""
    bc, dx = spec_from_arr(GOLD[f'laplace/{name}/bc']), GOLD[f'laplace/{name}/dx']
    a = GOLD[f'laplace/{name}/in']
    with O.precision(64):
        ref = GOLD[f'laplace/{name}/out']
        got = O.laplace(a, dx, bc)
        assert got.dtype == np.float64
        assert np.abs(got - ref).max() <= 8 * EPS * (np.abs(a).max() + 2) * 4 * np.sum(1 / dx ** 2)
        g = GOLD[f'sample/{name}/out']
        assert np.abs(O.grid_sample(a, GOLD[f'sample/{name}/coords'], bc) - g).max() <= 8 * EPS * (np.abs(a).max() + 2)
        if f'fluid/{name}/div' not in GOLD.files:
            return
        d = len(bc)
        v = [GOLD[f'fluid/{name}/v{c}'] for c in range(d)]
        div = O.divergence_staggered(v, dx, O.component_bcs(bc, d))
        assert np.abs(div - GOLD[f'fluid/{name}/div']).max() <= 4 * EPS * (max(np.abs(c).max() for c in v) + 2) * np.sum(1 / dx)
        grad = O.gradient_faces(GOLD[f'fluid/{name}/p'], dx, O.pressure_bc(bc), bc)
        for c in range(d):
            np.testing.assert_array_equal(grad[c], GOLD[f'fluid/{name}/grad{c}'])


@pytest.mark.parametrize('key', gold_names('cg'))
def test_fp64_oracle_cg_matches_phiml(key):
    """solve_linear(Solve('CG', 1e-12, 1e-12)) of PhiML in float64: the oracle's CG takes the same number of iterations."""
    vbc, dx, rhs = spec_from_arr(GOLD[f'cg/{key}/bc']), GOLD[f'cg/{key}/dx'], GOLD[f'cg/{key}/rhs']
    with O.precision(64):
        A = O.poisson_matrix(rhs.shape, dx, O.pressure_bc(vbc))
        info = O.cg(A, rhs, np.zeros(rhs.shape), 1e-12, 1e-12, 2000)
    assert info['converged'] and info['iterations'] == int(GOLD[f'cg/{key}/iterations'])
    x = GOLD[f'cg/{key}/x']
    assert np.abs(info['x'].reshape(x.shape) - x).max() <= 1e-9 * np.abs(x).max()


def test_fp64_oracle_taylor_green_step_matches_phiml():
    n, L, nu, dt = GOLD['tg/params']
    n = int(n)
    res, dx = (n, n), (L / n, L / n)
    v, p, info = taylor_green_step([GOLD['tg/u0'], GOLD['tg/v0']], GOLD['tg/p0'], dt, nu, O.uniform_bc(2, 'periodic'), res, dx,
                                   (0., 0.), (L, L))
    assert info['iterations'] == int(GOLD['tg/iterations'])
    for c, k in enumerate(('u1', 'v1')):
        assert np.abs(v[c] - GOLD[f'tg/{k}']).max() <= 1e-11
    assert np.abs((p - p.mean()) - (GOLD['tg/p1'] - GOLD['tg/p1'].mean())).max() <= 1e-11


# ---- C ABI without a GPU ---------------------------------------------------------------------------------------------------------

def test_fp64_struct_sizes_match_c():
    src = r'''
    #include <stdio.h>
    #include "phicuda.h"
    int main(void) { printf("%zu %zu %zu\n", sizeof(PhiValues64), sizeof(PhiCgParams64), sizeof(PhiCgResult64)); return 0; }'''
    with tempfile.TemporaryDirectory() as tmp:
        c, exe = os.path.join(tmp, 's.c'), os.path.join(tmp, 's')
        with open(c, 'w') as f:
            f.write(src)
        subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    assert sizes == [C.sizeof(_lib.PhiValues64), C.sizeof(_lib.PhiCgParams64), C.sizeof(_lib.PhiCgResult64)]
    assert _ops._RESULT_DTYPE64.itemsize == C.sizeof(_lib.PhiCgResult64)


def grid2(dx=(0.25, 2 * np.pi / 25), halo=0):
    dom = _ops.Domain((8, 8), dx, 1, device='cpu', dtype=torch.float64)
    g = dom.grid
    g.halo = halo
    return dom, g


def test_f64_entry_points_check_their_arguments_without_gpu():
    lib = _lib.load()
    spec = ((0.1, 'zg'), ('periodic', 'periodic'))
    dom, g = grid2()
    bc, vbc = _ops.make_bc(spec), _ops.make_vbc(spec, 2)
    fake = C.c_void_p(256)                                     # never dereferenced: every check runs before the first CUDA call
    ok = dom.values64(spec, 2)
    # the exact dx must round to PhiGrid.dx
    bad = dom.values64(spec, 2)
    bad.dx[1] = 2 * np.pi / 25 * (1 + 1e-6)
    assert lib.phicuda_laplace_f64(C.byref(g), C.byref(bc), C.byref(bad), fake, C.c_void_p(512), None) == _lib.ERR_INVALID
    assert 'dx[1]' in _lib.last_error()
    assert lib.phicuda_divergence_f64(C.byref(g), C.byref(vbc), C.byref(bad), _ops.F3(256, 512, 0), fake, None) == _lib.ERR_INVALID
    # ... and the exact constants to the PhiBC constants
    bad = dom.values64(spec, 2)
    bad.clo[1][0] = 0.1 + 1e-6
    assert lib.phicuda_grad_sub_f64(C.byref(g), C.byref(vbc), C.byref(bad), _ops.F3(256, 512, 0), fake, None) == _lib.ERR_INVALID
    assert 'clo/chi[1][0]' in _lib.last_error()
    assert lib.phicuda_laplace_f64(C.byref(g), C.byref(bc), None, fake, C.c_void_p(512), None) == _lib.ERR_INVALID
    # z-slabs are refused
    dom3 = _ops.Domain((8, 8, 8), (1.0, 1.0, 1.0), 1, device='cpu')
    g3 = dom3.grid
    g3.halo, g3.cext[2], g3.fext[2] = 1, 10, 10
    spec3 = O.uniform_bc(3, 'periodic')
    code = lib.phicuda_laplace_f64(C.byref(g3), C.byref(_ops.make_bc(spec3)), C.byref(dom3.values64(spec3)), fake, C.c_void_p(512), None)
    assert code == _lib.ERR_UNSUPPORTED and 'z-slab' in _lib.last_error()
    # the fp64 solve takes Shewchuk CG only
    prm = _ops.cg_params(spec, rtol=1e-12, atol=1e-12, method='CG-adaptive', dtype=torch.float64)
    args = (C.byref(g), C.byref(vbc), C.byref(ok), fake, C.c_void_p(512), C.byref(prm), C.c_void_p(1024), C.c_void_p(2048), C.c_size_t(1 << 30), None)
    assert lib.phicuda_cg_poisson_f64(*args) == _lib.ERR_UNSUPPORTED and 'CG-adaptive' in _lib.last_error()
    prm.method = 7
    assert lib.phicuda_cg_poisson_f64(*args) == _lib.ERR_INVALID and 'unknown solver method' in _lib.last_error()
    prm.method = 0
    small = args[:8] + (C.c_size_t(64), None)
    assert lib.phicuda_cg_poisson_f64(*small) == _lib.ERR_WORKSPACE
    assert lib.phicuda_cg_workspace_bytes_f64(C.byref(g)) >= 3 * 8 * 8 * 8
    code = lib.phicuda_make_incompressible_f64(C.byref(g), C.byref(vbc), C.byref(ok), _ops.F3(256, 512, 0), fake, C.c_void_p(4096),
                                               C.byref(prm), C.c_void_p(1024), C.c_void_p(2048), C.c_size_t(64), None)
    assert code == _lib.ERR_WORKSPACE
    # div and p must not alias a velocity component (the divergence reads v while it writes div, grad_sub writes v while it reads p)
    dom_v = _ops.Domain((8, 8), (0.25, 2 * np.pi / 25), 1, vbc=spec, device='cpu', dtype=torch.float64)
    ws = C.c_size_t(lib.phicuda_cg_workspace_bytes_f64(C.byref(dom_v.grid)))
    for v3, div, p in [(_ops.F3(256, 512, 0), C.c_void_p(512), C.c_void_p(4096)), (_ops.F3(256, 512, 0), C.c_void_p(8192), C.c_void_p(256)),
                       (_ops.F3(256, 256, 0), C.c_void_p(8192), C.c_void_p(4096))]:
        code = lib.phicuda_make_incompressible_f64(C.byref(dom_v.grid), C.byref(vbc), C.byref(ok), v3, p, div, C.byref(prm),
                                                   C.c_void_p(1024), C.c_void_p(2048), ws, None)
        assert code == _lib.ERR_INVALID and 'v[' in _lib.last_error()
    g.batch = 1025
    assert lib.phicuda_cg_poisson_f64(*args) == _lib.ERR_UNSUPPORTED and 'batch' in _lib.last_error()


def test_ops_arrays_take_the_domains_dtype(monkeypatch):
    """A domain's CG workspace and result records are sized and read for its dtype, so arrays of the other dtype are refused before
    any library call: float64 arrays on a float32 domain would get a too small workspace and 24-byte result records for 40-byte ones."""
    monkeypatch.setattr(_ops, 'require_cuda', lambda: None)
    spec = O.uniform_bc(2, 'periodic')
    d64 = _ops.Domain((64, 64), (1.0, 1.0), 2, vbc=spec, device='cpu', dtype=torch.float64)
    d32 = _ops.Domain((64, 64), (1.0, 1.0), 2, vbc=spec, device='cpu')
    x64, x32 = d64.alloc_centered(), d32.alloc_centered()
    for dom, x in [(d32, x64), (d64, x32)]:
        v = [t.to(x.dtype) for t in dom.alloc_faces()]
        with pytest.raises(AssertionError, match='domain'):
            _ops.cg_poisson(dom, spec, x, x.clone())
        with pytest.raises(AssertionError, match='domain'):
            _ops.laplace(dom, spec, x, out=x.clone())
        with pytest.raises(AssertionError, match='domain'):
            _ops.advect_centered(dom, spec, v, spec, x, 0.1, out=x.clone())
        with pytest.raises(AssertionError, match='domain'):
            _ops.divergence(dom, spec, v, out=x.clone())
        with pytest.raises(AssertionError, match='domain'):
            _ops.grad_sub(dom, spec, v, x)
        with pytest.raises(AssertionError, match='dtype'):
            _ops.make_incompressible(dom, spec, v, x.clone())
    # matching arrays get past the dispatch (without a GPU the call then fails at its stream or first CUDA call - not with Unsupported)
    if not torch.cuda.is_available():
        v = d64.alloc_faces()
        for call in (lambda: _ops.divergence(d64, spec, v), lambda: _ops.grad_sub(d64, spec, v, x64),
                     lambda: _ops.make_incompressible(d64, spec, v, x64.clone())):
            with pytest.raises(RuntimeError) as err:
                call()
            assert not isinstance(err.value, (_lib.Unsupported, AssertionError)), err.value
    with pytest.raises(_lib.Unsupported, match='float64'):           # no fp64 kernel: a float64 domain is refused with float32 arrays too
        _ops.reaction_diffusion(d64, spec, x32, x32, 0.1, 0.1, 0.01, 0.05, 1.0)
    with pytest.raises(_lib.Unsupported, match='float64'):
        _ops.diffuse_implicit(d64, spec, x32, 0.1)


def test_ops_refuse_mixed_and_float64_only_where_offered(monkeypatch):
    monkeypatch.setattr(_ops, 'require_cuda', lambda: None)
    spec = O.uniform_bc(2, 'periodic')
    d64 = _ops.Domain((8, 8), (1.0, 1.0), 1, vbc=spec, device='cpu', dtype=torch.float64)
    d32 = _ops.Domain((8, 8), (1.0, 1.0), 1, vbc=spec, device='cpu')
    x64, x32 = d64.alloc_centered(), d32.alloc_centered()
    assert x64.dtype == torch.float64 and d64.centered_from_numpy(np.ones((8, 8), np.float32)).dtype == torch.float64
    with pytest.raises(AssertionError, match='share a dtype'):
        _ops.laplace(d64, spec, x64, out=x32)
    with pytest.raises(_lib.Unsupported, match='float64'):
        _ops.reaction_diffusion(d64, spec, x64, x64, 0.1, 0.1, 0.01, 0.05, 1.0)
    with pytest.raises(_lib.Unsupported, match='float64'):
        _ops.mac_cormack_centered(d64, spec, d64.alloc_faces(), spec, x64, 0.5)
    with pytest.raises(_lib.Unsupported, match='float64'):
        _ops.diffuse_implicit(d64, spec, x64, 0.1)
    with pytest.raises(_lib.Unsupported, match='obstacles'):
        _ops.make_incompressible(d64, spec, d64.alloc_faces(), x64, accessible=d64.alloc_centered())


# ---- the mirror in precision 64 ---------------------------------------------------------------------------------------------------

@pytest.fixture()
def F():
    import phiflow_b200.flow as flow
    saved = flow.ops, flow._DEVICE
    flow.ops = Fp64OracleEngine
    flow.set_device('cpu')
    try:
        yield flow
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])
        flow.set_global_precision(32)


def test_mirror_precision(F):
    assert F.math.get_precision() == 32
    assert F.Solve('CG').rel_tol == 1e-5
    with F.math.precision(64):
        assert F.math.get_precision() == 64
        s = F.Solve('CG')
        assert s.rel_tol == 1e-12 and s.abs_tol == 1e-12
        c = F.CenteredGrid(np.arange(16.).reshape(4, 4) / 3, x=4, y=4)
        v = F.StaggeredGrid(0.5, F.PERIODIC, x=4, y=4)
    assert F.math.get_precision() == 32 and s.rel_tol == 1e-5          # _default_tolerance is read when the solve runs
    assert c.data.dtype == torch.float64 and c.numpy().dtype == np.float64
    assert c.numpy()[1, 1] == 5 / 3                                    # not rounded through float32
    for r in (c + 1, c - 1.5, c * 2.5, c ** 2, 1 - c, -c, c + c):
        assert r.data.dtype == torch.float64
    for r in (v + 1, v * 0.5, v - v):
        assert all(t.dtype == torch.float64 for t in r.data)
    c32 = F.CenteredGrid(1.0, x=4, y=4)
    assert c32.data.dtype == torch.float32
    with pytest.raises(NotImplementedError, match='mixing float32 and float64'):
        c + c32
    F.math.set_global_precision(64)
    assert F.CenteredGrid(0, x=4, y=4).data.dtype == torch.float64


def test_mirror_field_io_keeps_float64(F, tmp_path):
    with F.math.precision(64):
        c = F.CenteredGrid(np.arange(16.).reshape(4, 4) / 3, x=4, y=4)
    F.write(c, str(tmp_path / 'c.npz'))
    r = F.read(str(tmp_path / 'c.npz'))
    assert r.data.dtype == torch.float64
    np.testing.assert_array_equal(r.numpy(), c.numpy())


def load_example(name):
    spec = importlib.util.spec_from_file_location(f'example_{name}', os.path.join(ROOT, 'examples', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_taylor_green_example_over_the_oracle(F):
    tg = load_example('taylor_green')
    v, p, errs, iters = tg.run(4)
    vbc = O.uniform_bc(2, 'periodic')
    res, dx = (tg.N, tg.N), (2 * np.pi / tg.N,) * 2
    vo, po = tg.analytic_velocity(0.), tg.analytic_pressure(0.)
    for _ in range(4):
        vo, po, info = taylor_green_step(vo, po, tg.DT, tg.VISCOSITY, vbc, res, dx, (0., 0.), (2 * np.pi,) * 2)
    for c in range(2):
        assert v[c].dtype == np.float64
        np.testing.assert_allclose(v[c], vo[c], rtol=0, atol=1e-13)
    assert len(iters) == 4 and all(i > 0 for i in iters)
    assert errs.shape == (5, 2) and errs[0, 0] == 0 and 0 < errs[-1, 1] < 0.05


def test_fp64_refusals(F):
    """Every combination outside the fp64 path raises; nothing is computed in float32 instead."""
    with F.math.precision(64):
        v = F.StaggeredGrid(0.1, F.PERIODIC, x=8, y=8)
        s = F.CenteredGrid(0.2, F.PERIODIC, x=8, y=8)
        p = F.CenteredGrid(0, F.PERIODIC, x=8, y=8)
        cv = F.CenteredGrid(0, F.PERIODIC, x=8, y=8)
    v32 = F.StaggeredGrid(0.1, F.PERIODIC, x=8, y=8)
    p32 = F.CenteredGrid(0, F.PERIODIC, x=8, y=8)
    cases = [
        lambda: F.fluid.make_incompressible(v, (), F.Solve('auto')),
        lambda: F.fluid.make_incompressible(v, (), F.Solve('CG-adaptive')),
        lambda: F.fluid.make_incompressible(v),                                      # the default Solve() is 'auto'
        lambda: F.fluid.make_incompressible(v, F.Box(x=(2, 4), y=(2, 4)), F.Solve('CG')),
        lambda: F.fluid.make_incompressible(v, (), F.Solve('CG', x0=p32)),
        lambda: F.fluid.incompressible_step(v, s, p, 0.1),
        lambda: F.advect.mac_cormack(s, v, 0.1),
        lambda: F.advect.semi_lagrangian(s, v32, 0.1),
        lambda: F.diffuse.implicit(s, 0.1, 0.1),
        lambda: F.field.where(F.Sphere(x=4, y=4, radius=2), 1.0, s),
        lambda: F.resample(s * (0, 0.1), to=v),
        lambda: F.reaction_diffusion(s, s, 0.1, 0.1, 0.01, 0.05, 1.0),
        lambda: F.wave_step(s, s, 0.0, 0.1),
        lambda: F.fluid.make_incompressible(cv, (), F.Solve('CG')),
        lambda: F.CenteredGrid(F.Box(x=(2, 4), y=(2, 4)), x=8, y=8),           # geometry masks are sampled at float32 centres
        lambda: F.StaggeredGrid(F.Sphere(x=4, y=4, radius=2), x=8, y=8),
        lambda: F.resample(F.Sphere(x=4, y=4, radius=2), to=s),
    ]
    F.math.set_global_precision(64)                                            # grids the cases themselves create are float64
    for i, case in enumerate(cases):
        with pytest.raises(NotImplementedError):
            case()
