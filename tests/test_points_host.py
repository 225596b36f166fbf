"""
advect.points (DESIGN.md row N11) without a GPU: the kernel's restatement (tests/oracle_points.py) against PhiML's positions
(tests/golden/phiml_points.npz, tests/golden/make_points_golden.py), the host-built PhiPointMap against PhiML's component grids, the C
declaration, every argument check of phicuda_advect_points_f32 (all of them run before the first CUDA call) and every refusal of the
mirror.
"""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import phiflow_b200.flow as flow
from oracle_points import F, advect_points, to_int32
from phiflow_b200 import _lib, _ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'phiml_points.npz')


def _side(s):
    return s if isinstance(s, str) else float(s)


def golden_case(g, name):
    """(per-component specs for _ops, oracle velocity, points, (lower, upper), res) of one fixture case."""
    spec = [[tuple(_side(s) for s in ax) for ax in comp] for comp in json.loads(str(g[f'{name}/spec']))]
    d = len(spec)
    vel = []
    for c in range(d):
        st = g[f'{name}/stagger{c}']
        vel.append((g[f'{name}/v{c}'], spec[c], st[0], st[1], st[2]))
    bounds = g[f'{name}/bounds']
    res = tuple(int(g[f'{name}/stagger{(c + 1) % d}'][2][c]) for c in range(d))   # another component's count along c = n_c
    return [tuple(s) for s in spec], vel, g[f'{name}/points'], (tuple(bounds[0]), tuple(bounds[1])), res


def runs():
    return [tuple(r) for r in json.loads(str(np.load(GOLD)['meta']))['runs']]


def cases():
    return json.loads(str(np.load(GOLD)['meta']))['cases']


def same(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize('name', cases())
def test_oracle_matches_phiml(name):
    g = np.load(GOLD)
    _, vel, pts, _, _ = golden_case(g, name)
    for integ, steps, dt in runs():
        assert same(advect_points(vel, pts, dt, integ, steps), g[f'{name}/{integ}_{steps}_{dt}']), (integ, steps, dt)


def test_oracle_matches_phiml_notebook():
    g = np.load(GOLD)
    vel = [(g[f'notebook/v{c}'], [(0.0, 0.0), (0.0, 0.0)], *_notebook_map(c)) for c in range(2)]
    _, trj = advect_points(vel, g['notebook/points'], 0.1, 'rk4', 50, trajectory=True)
    assert same(trj, g['notebook/trajectory'])


def _notebook_map(c):
    m = _ops.point_map((0., 0.), (10., 10.), (256, 256), ((0.0, 0.0), (0.0, 0.0)))
    return np.array(m.lower[c][:2], F), np.array(m.size[c][:2], F), np.array(m.res[c][:2], F)


def test_int32_cast_as_recorded():
    """The kernel converts NaN, +-inf and |x| >= 2^31 to INT_MIN, as PhiML's to_int32 did where the fixture was recorded."""
    g = np.load(GOLD)
    assert np.array_equal(to_int32(np.floor(g['int32_cast/in'])), g['int32_cast/out'])


def test_rk4_constants():
    """1.f / 6.f in the kernel is f32(1 / 6.) (PhiML's Python constant), and f32(0.5) * dt = f32(0.5 * dt) for normal dt."""
    assert F(1) / F(6) == F(1 / 6.)
    for dt in (0.1, -0.3, 1e-3, 0.35, 7.0):
        assert F(0.5) * F(dt) == F(0.5 * dt)


@pytest.mark.parametrize('name', cases())
def test_point_map_matches_phiml_stagger(name):
    g = np.load(GOLD)
    spec, _, _, (lower, upper), res = golden_case(g, name)
    m = _ops.point_map(lower, upper, res, list(spec))
    d = len(res)
    for c in range(d):
        st = g[f'{name}/stagger{c}']
        assert np.array_equal(np.array(m.lower[c][:d], F), st[0]) and np.array_equal(np.array(m.size[c][:d], F), st[1])
        assert np.array_equal(np.array(m.res[c][:d], F), st[2])


def test_declaration_matches_c():
    src = r'''#include <stdio.h>
    #include "phicuda.h"
    typedef int (*fn_t)(const PhiGrid*, const PhiVBC*, const float* const[3], const PhiPointMap*, const float*, int64_t, int32_t, float,
                        int32_t, int32_t, float*, float*, void*);
    fn_t declared(void) { return phicuda_advect_points_f32; }     /* -Werror: the declaration has exactly this type */
    #ifndef CHECK_ONLY
    int main(void) { printf("%zu %d %d %d\n", sizeof(PhiPointMap), PHI_INTEGRATOR_EULER, PHI_INTEGRATOR_RK4, PHI_KERNEL_POINTS); return 0; }
    #endif'''
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, 'p.c'), os.path.join(d, 'p')
        open(c, 'w').write(src)
        subprocess.check_call(['gcc', '-Werror', '-DCHECK_ONLY', '-I', os.path.join(ROOT, 'include'), '-c', c, '-o', exe + '.o'])
        open(c, 'w').write(src.replace('fn_t declared(void) { return phicuda_advect_points_f32; }', ''))
        subprocess.check_call(['gcc', '-Werror', '-I', os.path.join(ROOT, 'include'), c, '-o', exe])
        vals = [int(v) for v in subprocess.check_output([exe]).split()]
    assert vals == [C.sizeof(_lib.PhiPointMap), _lib.INTEGRATOR_EULER, _lib.INTEGRATOR_RK4, _lib.KERNEL_POINTS]
    assert _lib.PROTOTYPES['phicuda_advect_points_f32'][1][5] is C.c_int64


# ---- C ABI validation (no CUDA call is reached; out and trajectory are host arrays that must stay untouched) ----------------------
Z = 0.0


def _grid(dim=2, n=(16, 8, 4), batch=2, halo=0):
    g = _lib.PhiGrid()
    g.dim, g.batch, g.halo = dim, batch, halo
    for a in range(dim):
        pad = 2 * halo if a == 2 else 0
        g.n[a] = n[a]
        g.cext[a] = g.fext[a] = ((n[a] + 3) // 4 * 4 if a == 0 else n[a]) + pad
        g.dx[a] = 1.0
    return g


def _call(g=None, spec=((Z, Z), (Z, Z)), npoints=5, points_batch=2, integrator=1, steps=3, tweak=None, null=None, alias=None,
          traj=True):
    lib = _lib.load()
    g = g or _grid()
    d = g.dim
    spec = spec if len(spec) == d else ((Z, Z),) * d
    m = _ops.point_map((0.,) * d, tuple(float(g.n[a]) for a in range(d)), tuple(g.n[a] for a in range(d)), spec)
    if tweak:
        tweak(m)
    B = max(g.batch, points_batch)
    n = max(npoints, 0)
    pts = np.zeros((points_batch, n, d), F)
    out = np.full((B, max(n, 1), d), 7.0, F)
    trj = np.full((max(steps, 0) + 1, B, max(n, 1), d), 7.0, F) if traj else None
    vel = _lib.F3()
    for c in range(3):
        vel[c] = (1 << 40) + (c << 32) if c < d else None       # device addresses, never dereferenced: validation fails first
    args = dict(points=pts.ctypes.data, out=out.ctypes.data, trajectory=trj.ctypes.data if trj is not None else None, map=C.byref(m))
    if alias == 'out=points':
        args['out'] = args['points']
    if alias == 'traj=out':
        args['trajectory'] = args['out']
    if alias == 'out=vel':
        args['out'] = vel[0]
    if null:
        args[null] = None
    code = lib.phicuda_advect_points_f32(C.byref(g), C.byref(_ops.make_vbc(spec, d)), vel, args['map'], C.c_void_p(args['points']),
                                         npoints, points_batch, C.c_float(0.1), integrator, steps, C.c_void_p(args['out']),
                                         C.c_void_p(args['trajectory']), None)
    untouched = np.all(out == 7.0) and (trj is None or np.all(trj == 7.0))
    return code, untouched


def _set(field, c, a, v):
    def f(m):
        getattr(m, field)[c][a] = v
    return f


@pytest.mark.parametrize('kw,code,word', [
    ({'null': 'points'}, _lib.ERR_INVALID, 'NULL'),
    ({'null': 'out'}, _lib.ERR_INVALID, 'NULL'),
    ({'null': 'map'}, _lib.ERR_INVALID, 'NULL'),
    ({'steps': 0}, _lib.ERR_INVALID, 'steps'),
    ({'steps': -2}, _lib.ERR_INVALID, 'steps'),
    ({'npoints': -1}, _lib.ERR_INVALID, 'npoints'),
    ({'integrator': 2}, _lib.ERR_INVALID, 'integrator'),
    ({'integrator': -1}, _lib.ERR_INVALID, 'integrator'),
    ({'points_batch': 3}, _lib.ERR_INVALID, 'broadcast'),
    ({'points_batch': 0}, _lib.ERR_INVALID, 'broadcast'),
    ({'tweak': _set('res', 0, 0, 16.0)}, _lib.ERR_INVALID, 'res'),       # ZERO: component x stores 15 faces along x
    ({'tweak': _set('res', 1, 0, 15.0)}, _lib.ERR_INVALID, 'res'),
    ({'tweak': _set('size', 0, 1, 0.0)}, _lib.ERR_INVALID, 'size'),
    ({'tweak': _set('size', 1, 0, -1.0)}, _lib.ERR_INVALID, 'size'),
    ({'tweak': _set('size', 1, 1, float('inf'))}, _lib.ERR_INVALID, 'size'),
    ({'tweak': _set('size', 0, 0, float('nan'))}, _lib.ERR_INVALID, 'size'),
    ({'tweak': _set('lower', 0, 0, float('nan'))}, _lib.ERR_INVALID, 'lower'),
    ({'g': _grid(3, halo=1)}, _lib.ERR_UNSUPPORTED, 'z-slab'),
    ({'g': _grid(batch=0)}, _lib.ERR_INVALID, 'batch'),
    ({'alias': 'out=points', 'points_batch': 1}, _lib.ERR_INVALID, 'broadcast'),
    ({'alias': 'traj=out'}, _lib.ERR_INVALID, 'trajectory overlaps'),
    ({'alias': 'out=vel'}, _lib.ERR_INVALID, 'velocity'),
])
def test_argument_validation_without_gpu(kw, code, word):
    got, untouched = _call(**kw)
    assert got == code, _lib.last_error()
    assert word in _lib.last_error()
    assert untouched


def test_no_points_returns_before_cuda():
    got, untouched = _call(npoints=0)
    assert got == 0 and untouched


def test_kernel_id():
    assert _lib.KERNEL_POINTS == 9


# ---- the mirror's refusals --------------------------------------------------------------------------------------------------------
class _NoKernels:
    def __getattr__(self, name):
        raise AssertionError(f"ops.{name} reached by a refused call")


@pytest.fixture()
def cpu_grids():
    saved = flow.ops, flow._DEVICE
    flow.set_device('cpu')
    try:
        box = flow.Box(x=4, y=4)
        v = flow.StaggeredGrid(0.1, 0, box, x=8, y=8)
        c = flow.CenteredGrid(0.1, 0, box, x=8, y=8)
        with flow.math.precision(64):
            v64 = flow.StaggeredGrid(0.1, 0, box, x=8, y=8)
        v3 = flow.StaggeredGrid(0.1, 0, flow.Box(x=4, y=4, z=4), x=4, y=4, z=4)
        flow.ops = _NoKernels()
        yield v, c, v64, v3
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])


def test_mirror_refusals(cpu_grids):
    v, c, v64, v3 = cpu_grids
    p2 = np.zeros((3, 2), np.float32)
    advect = flow.advect
    cases = [
        lambda: advect.points(flow.geom.Point(p2), v, 0.1, integrator=advect.finite_rk4),
        lambda: advect.points(p2, v, 0.1, integrator=lambda *a: None),
        lambda: advect.points(p2, v, 0.1, integrator='rk4'),
        lambda: advect.points(p2, c, 0.1),
        lambda: advect.points(p2, v64, 0.1, integrator=advect.rk4),
        lambda: advect.points(p2.astype(np.float64), v, 0.1),
        lambda: advect.points(torch.zeros(3, 2, dtype=torch.float64), v, 0.1),
        lambda: advect.points(torch.zeros(3, 2), v, 0.1),                       # a CPU tensor: points live on the GPU or in NumPy
        lambda: advect.points(p2, v3, 0.1),
        lambda: advect.points(np.zeros((3, 3), np.float32), v, 0.1),
        lambda: advect.points((1.0, 2.0, 3.0), v, 0.1),
        lambda: advect.advect(p2, v, 0.1, integrator=advect.finite_rk4),
        lambda: advect.advect(flow.geom.Point(p2), c, 0.1),
        lambda: advect.advect(flow.CenteredGrid(0.1, 0, flow.Box(x=4, y=4), x=8, y=8), v, 0.1, integrator=advect.rk4),
        lambda: advect.euler(p2, v, 0.1, v0=p2),
        lambda: advect.rk4(p2, c, 0.1),
        lambda: advect.finite_rk4(p2, v, 0.1),
        lambda: flow.streamlines(p2, v, 0.1, 0),
        lambda: flow.streamlines(p2, v, 0.1, 2.5),
        lambda: flow.streamlines(p2, v, 0.1, 5, integrator=advect.finite_rk4),
        lambda: flow.streamlines(p2, v64, 0.1, 5),
        lambda: flow.streamlines(p2, c, 0.1, 5),
    ]
    for i, case in enumerate(cases):
        with pytest.raises(NotImplementedError):
            case()


def test_ops_refuse_float64_and_unknown_integrators(monkeypatch):
    monkeypatch.setattr(_ops, 'require_cuda', lambda: None)
    spec = ((Z, Z), (Z, Z))
    dom = _ops.Domain((8, 8), (1.0, 1.0), 1, vbc=spec, device='cpu')
    v = dom.alloc_faces()
    pts = torch.zeros(1, 4, 2)
    with pytest.raises(_lib.Unsupported, match='float64'):
        _ops.advect_points(dom, spec, v, (0., 0.), (8., 8.), pts.double(), 0.1)
    with pytest.raises(_lib.Unsupported, match='float64'):
        _ops.advect_points(dom, spec, [t.double() for t in v], (0., 0.), (8., 8.), pts, 0.1)
    with pytest.raises(_lib.Unsupported, match='finite_rk4'):
        _ops.advect_points(dom, spec, v, (0., 0.), (8., 8.), pts, 0.1, integrator='finite_rk4')
