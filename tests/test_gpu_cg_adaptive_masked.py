"""
CG-adaptive with obstacles on the TMA ring (k_cg_ring<DIM, GENERIC, DIST=false, ADAPT=true, CgOp::Masked>) against the oracle:
oracle_np.cg_adaptive on oracle_np.masked_poisson_matrix_sparse, the solver make_incompressible(v, obstacle, Solve()) runs in the
reference.  Every case asserts the launch record (PHI_KERNEL_CG_RING, masked, adaptive, generic, two passes, the Poisson operator),
so a case cannot silently move to another kernel.  Helpers are those of test_gpu_cg_contract.py.

Widths (ring_config in ring_kernels.cu on an H100, 227 KiB of opt-in shared memory per block, batch 3): the masked stage holds
5 TY + 6 lines (pass A of CG-adaptive stages r, d and the mask with halos plus r element-wise = 4 TY + 6 of them), so at TY 1 a 2-D
line of 2628 cells is the widest the ring takes (2 stages) and 2632 is refused; in 3-D 1752 cells (3 stages) and 1756 is refused.
CG-adaptive has no register-marching kernel: a refused grid raises Unsupported and leaves x untouched.

Converged solves run on systems with an open side only: on closed and periodic systems with obstacles the iteration count of fp32
CG-adaptive depends on the summation order (PhiML 288 against the oracle's 249 on one closed 14 x 10 grid), which neither side pins.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle_np as O
import test_gpu_cg_contract as CC

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from phiflow_b200 import _ops as ops
    from phiflow_b200 import _lib

TRUNC_K = (1, 2, 3, 4, 7)
BCS = {
    'zero': ((0.0, 0.0), (0.0, 0.0)), 'open': (('zg', 'zg'), ('zg', 'zg')), 'periodic': (('periodic', 'periodic'), ('periodic', 'periodic')),
    'mixed': (('zg', 'zg'), (0.0, 'zg')), 'per_x_wall_y': (('periodic', 'periodic'), (0.0, 0.0)),
    'zero3': ((0.0, 0.0),) * 3, 'open3': (('zg', 'zg'),) * 3, 'periodic3': (('periodic', 'periodic'),) * 3,
    'mixed3': (('periodic', 'periodic'), (0.0, 'zg'), ('zg', 0.0)), 'wall_open3': (('periodic', 'periodic'), (0.0, 0.0), (0.0, 'zg')),
}
RAGGED = {2: [(37, 22), (150, 9)], 3: [(21, 14, 9), (133, 10, 6)]}


def launch(**kw):
    return {'kernel': 3, 'generic': 1, 'masked': 1, 'passes': 2, **kw}


def _cases():
    out = []
    for i, name in enumerate(sorted(BCS)):
        d = len(BCS[name])
        for res in RAGGED[d]:
            out.append(('ragged', name, res))
        if i % 2 == 0:
            res = (14, 11) if d == 2 else (10, 8, 7)
            out.append(('small', name, res))
    return out


def case_of(name, res, **kw):
    return CC.Case(f'acg-masked-{name}-{"x".join(map(str, res))}', res, BCS[name], launch(**kw), dx=tuple(50.0 / r for r in res),
                   acc=CC.obstacle_acc(res))


CASES = [case_of(n, r) for _, n, r in _cases()]
FLEX = [c for c in CASES if O.is_flexible(c.vbc)]


def run(case, dom, rhs, x0, prm):
    got, rec, info = CC.solve(case, dom, rhs, x0, prm, adaptive=True)
    assert ops.last_cg_operator() == 'poisson' and info['passes'] == 2, case.name
    return got, rec, info


def aparams(case, rtol, atol, max_iter):
    return CC.params(case, rtol, atol, max_iter, method='CG-adaptive')


@pytest.mark.parametrize('case', CASES, ids=str)
def test_truncated_iterates(case):
    """Exactly k iterations from a warm start that is non-zero inside the obstacles, batch 3 at scales 1 / 10 / 0.1: iterates, the
    result record and tol_sq = max(rtol^2 |y'|^2, atol^2) with |y' - A x0|^2 >= 100 |y'|^2."""
    A, rhs, y, x0 = CC.problem(case, 201)
    assert np.abs(x0[:, case.acc == 0]).min() > 0
    dom = CC.domain(case)
    for k in TRUNC_K:
        got, rec, _ = run(case, dom, rhs, x0, aparams(case, 1e-12, 0.0, k))
        for b in range(3):
            ref = CC.reference(case, A, y[b], x0[b], 1e-12, 0.0, k, adaptive=True, exact=True)
            CC.check_truncated(case, rec[b], ref, k)
            CC.check_record_start(case, rec[b], A, y[b], x0[b], 1e-12, 0.0, None, True)
            CC.check_iterate(case, got[b], ref)


@pytest.mark.parametrize('case', FLEX, ids=str)
@pytest.mark.parametrize('rtol', [1e-3, 1e-5])
def test_converged(case, rtol):
    """Converged solves from the warm start: both sides meet the rule, iteration counts within max(2, 10 %), solutions within
    20 rtol max|x|, tol_sq from |y'|^2."""
    A, rhs, y, x0 = CC.problem(case, 202, obstacle_x0=0.0)
    got, rec, _ = run(case, CC.domain(case), rhs, x0, aparams(case, rtol, 1e-5, 4000))
    for b in range(3):
        ref = CC.reference(case, A, y[b], x0[b], rtol, 1e-5, 4000, adaptive=True)
        CC.check_converged(case, rec[b], ref, got[b], A, y[b], rtol)
        CC.check_record_start(case, rec[b], A, y[b], x0[b], rtol, 1e-5, None, True)
        xr = CC.project(case, ref['x'].reshape(case.res).astype(np.float64))
        np.testing.assert_allclose(got[b], xr, rtol=0, atol=20 * rtol * np.abs(xr).max(), err_msg=case.name)


@pytest.mark.parametrize('name', ['mixed', 'open3'])
def test_entries_stop_apart_and_zero_entry(name):
    """Entry 1 starts close to its solution and stops early, entry 0 runs on, entry 2 is all zero (x0 = 0): converged at iteration 0,
    x untouched bit for bit."""
    d = len(BCS[name])
    case = case_of(name, RAGGED[d][0])
    A, rhs, y, x0 = CC.problem(case, 203, obstacle_x0=0.0)
    sol = CC.reference(case, A, y[1], np.zeros_like(x0[1]), 1e-6, 0.0, 4000, adaptive=True)['x'].reshape(case.res)
    x0[1] = sol + np.float32(1e-3) * np.float32(np.abs(sol).max()) * np.random.default_rng(3).standard_normal(case.res).astype(np.float32)
    rhs[2], x0[2] = 0.0, 0.0
    got, rec, _ = run(case, CC.domain(case), rhs, x0, aparams(case, 1e-5, 1e-5, 4000))
    its = [int(rec[b]['iterations']) for b in range(3)]
    assert its[2] == 0 and rec[2]['converged'] == 1 and its[1] < its[0], its
    np.testing.assert_array_equal(got[2], x0[2])
    for b in (0, 1):
        ref = CC.reference(case, A, y[b], x0[b], 1e-5, 1e-5, 4000, adaptive=True)
        CC.check_converged(case, rec[b], ref, got[b], A, y[b], 1e-5)


@pytest.mark.parametrize('name', ['mixed', 'zero3'])
def test_nan_entry_is_diverged_and_isolated(name):
    """One NaN in entry 1: entry 1 reports diverged at iteration 0; entries 0 and 2 are bit-identical to a run where entry 1 is zero."""
    d = len(BCS[name])
    case = case_of(name, RAGGED[d][1])
    _, rhs, _, x0 = CC.problem(case, 204)
    x0[1] = 0.0
    dom = CC.domain(case)
    prm = aparams(case, 1e-5, 1e-5, 40)
    clean = rhs.copy()
    clean[1] = 0.0
    bad = clean.copy()
    bad[1][(0,) * d] = np.nan
    got_c, rec_c, _ = run(case, dom, clean, x0, prm)
    got_n, rec_n, _ = run(case, dom, bad, x0, prm)
    assert (rec_n[1]['diverged'], rec_n[1]['converged'], rec_n[1]['iterations']) == (1, 0, 0), rec_n[1]
    for b in (0, 2):
        assert rec_n[b].tobytes() == rec_c[b].tobytes(), (rec_n[b], rec_c[b])
        np.testing.assert_array_equal(got_n[b], got_c[b])
    assert rec_c[0]['iterations'] > 0


WIDE = [((2628, 8), 'mixed', 2), ((1752, 6, 5), 'wall_open3', 3)]


@pytest.mark.parametrize('res,name,stages', WIDE, ids=['2d-2628', '3d-1752'])
def test_widest_line_runs_on_the_ring(res, name, stages):
    """The widest lines the masked adaptive ring takes (TY 1): truncated iterates against the oracle."""
    case = CC.Case(f'acg-masked-wide-{res[0]}', res, BCS[name], launch(TY=1, stages=stages), dx=(1.0,) * len(res), acc=CC.obstacle_acc(res))
    A, rhs, y, x0 = CC.problem(case, 205)
    dom = CC.domain(case)
    for k in (1, 3):
        got, rec, _ = run(case, dom, rhs, x0, aparams(case, 1e-12, 0.0, k))
        for b in range(3):
            ref = CC.reference(case, A, y[b], x0[b], 1e-12, 0.0, k, adaptive=True, exact=True)
            CC.check_truncated(case, rec[b], ref, k)
            CC.check_iterate(case, got[b], ref)


@pytest.mark.parametrize('res,name,limit', [((2632, 8), 'mixed', 2628), ((1756, 6, 5), 'wall_open3', 1752)], ids=['2d-2632', '3d-1756'])
def test_first_wider_line_is_refused(res, name, limit):
    """One group of four cells wider: Unsupported naming CG-adaptive and the limit, x untouched; plain CG still runs (marching kernel)."""
    case = CC.Case(f'acg-masked-refused-{res[0]}', res, BCS[name], CC.march(1), dx=(1.0,) * len(res), acc=CC.obstacle_acc(res))
    _, rhs, _, x0 = CC.problem(case, 206)
    dom = CC.domain(case)
    ws, rs = dom.workspace()
    x = dom.centered_from_numpy(x0)
    before = x.clone()
    acc = dom.centered_from_numpy(case.acc)
    prm = aparams(case, 1e-5, 1e-5, 100)
    with pytest.raises(_lib.Unsupported, match=f'CG-adaptive.*at most {limit} cells'):
        _lib.check(_lib.load().phicuda_cg_poisson_masked_f32(C.byref(dom.grid), C.byref(ops.make_vbc(case.vbc, dom.dim)),
                                                             ops._ptr(dom.centered_from_numpy(rhs)), ops._ptr(x), ops._ptr(acc), C.byref(prm),
                                                             ops._ptr(rs), ops._ptr(ws), C.c_size_t(ws.numel()), ops._stream()))
    torch.cuda.synchronize()
    assert torch.equal(x, before)
    CC.solve(case, dom, rhs, x0, CC.params(case, 1e-5, 1e-5, 3))


@pytest.mark.parametrize('name,res', [('mixed', (40, 28)), ('mixed3', (24, 14, 12))])
def test_make_incompressible_masked(name, res):
    """phicuda_make_incompressible_masked_f32 with CG-adaptive against the oracle's projection with CG-adaptive: velocity, pressure,
    and a divergence-free field on fluid cells."""
    from oracle_masked import make_incompressible_obstacles
    vbc = BCS[name]
    d = len(res)
    dx = tuple(50.0 / r for r in res)
    acc = CC.obstacle_acc(res)
    rng = np.random.default_rng(207)
    v = [rng.standard_normal((2,) + s).astype(np.float32) for s in O.staggered_shapes(res, vbc)]
    dom = ops.Domain(res, dx, 2, vbc=vbc)
    dv = dom.faces_from_numpy(v, vbc)
    p = dom.alloc_centered()
    dacc = dom.centered_from_numpy(np.stack([acc, acc]))
    prm = ops.cg_params(vbc, rtol=1e-5, atol=1e-5, max_iter=2000, method='CG-adaptive')
    ops.make_incompressible(dom, vbc, dv, p, prm, accessible=dacc)
    info = ops.last_launch_info()
    assert (info['kernel'], info['masked'], info['adaptive'], info['generic']) == (3, 1, 1, 1), info
    rec = ops.read_results(dom)
    got_v, got_p = dom.faces_to_numpy(dv, vbc, squeeze=False), dom.centered_to_numpy(p, squeeze=False)
    for b in range(2):
        vn, pn, ref = make_incompressible_obstacles([c[b] for c in v], vbc, res, dx, acc, None, 1e-5, 1e-5, 2000, method='CG-adaptive')
        assert rec[b]['converged'] == 1 and abs(int(rec[b]['iterations']) - ref['iterations']) <= max(2, ref['iterations'] // 10)
        scale = max(float(np.abs(pn).max()), 1e-3)
        np.testing.assert_allclose(got_p[b], pn, rtol=0, atol=2e-4 * scale)
        vmax = max(float(np.abs(c).max()) for c in vn)
        for c in range(d):
            np.testing.assert_allclose(got_v[c][b], vn[c], rtol=0, atol=2e-4 * vmax)
        div = O.divergence_staggered([c[b] for c in got_v], dx, O.component_bcs(vbc, d))
        assert float(np.abs(div[acc > 0]).max()) < 1e-3 * vmax / min(dx), float(np.abs(div[acc > 0]).max())


# ---- through the mirror --------------------------------------------------------------------------------------------------------

def _mirror_run(example_name, main_kwargs, engine):
    import phiflow_b200.flow as flow
    from test_cg_adaptive_masked_host import example
    saved = flow.ops, flow._DEVICE
    if engine is not None:
        flow.ops = engine
        flow.set_device('cpu')
    try:
        with flow.SolveTape() as tape:
            out = example(example_name).main(**main_kwargs)
        return out, [(int(r[1].iterations.max()), bool(r[1].converged.all())) for r in tape.records], flow
    finally:
        flow.ops = saved[0]
        flow.set_device(saved[1])


def test_mirror_default_solve_runs_the_new_kernel():
    """fluid.make_incompressible(v, obstacle, Solve(x0=p)) and Solve('CG-adaptive', 1e-5, x0=p) run on the masked adaptive ring;
    Solve('CG') on the masked plain ring; SolveTape counts match the oracle's CG-adaptive counts within the CG tolerance."""
    from phiflow_b200.flow import StaggeredGrid, Box, Solve, SolveTape, fluid
    from oracle_masked import make_incompressible_obstacles
    rng = np.random.default_rng(208)
    res, vbc = (48, 40), BCS['zero']
    v = StaggeredGrid([rng.standard_normal(s).astype(np.float32) for s in O.staggered_shapes(res, vbc)], 0, Box(x=48, y=40), x=48, y=40)
    obstacle = Box(x=(10, 20), y=(30, 40))
    v1, p = fluid.make_incompressible(v, obstacle, Solve('CG', 1e-5, 1e-5))
    assert (ops.last_launch_info()['adaptive'], ops.last_launch_info()['masked']) == (0, 1)
    import phiflow_b200.flow as flow
    accessible, factors = flow._obstacle_masks(v, obstacle)
    acc = v.dom.centered_to_numpy(accessible)
    vm = v.dom.faces_to_numpy([a * f for a, f in zip(v.data, factors)], v.vspec)
    for solve in (Solve(x0=p), Solve('CG-adaptive', 1e-5, x0=p)):
        w = v * 1.02
        with SolveTape() as tape:
            fluid.make_incompressible(w, obstacle, solve)
        info = ops.last_launch_info()
        assert (info['kernel'], info['masked'], info['adaptive'], info['generic']) == (3, 1, 1, 1), info
        assert info['passes'] == 2 and ops.last_cg_operator() == 'poisson'
        wm = [np.float32(1.02) * a for a in vm]
        _, _, ref = make_incompressible_obstacles(wm, vbc, res, (1.0, 1.0), acc, None, 1e-5, 1e-5, 1000, x0=p.numpy(), method='CG-adaptive')
        n = int(tape[0].iterations[0])
        assert abs(n - ref['iterations']) <= max(2, ref['iterations'] // 10), (n, ref['iterations'])


EXAMPLES = [('batched_smoke_obstacle', dict(res=64, steps=5)), ('wake_flow', dict(res=64, nz=8, steps=5))]


def _examples(example_name, kw):
    gpu_out, gpu_its, _ = _mirror_run(example_name, kw, None)
    info = ops.last_launch_info()
    assert (info['kernel'], info['masked'], info['adaptive']) == (3, 1, 1), info
    from oracle_masked import MaskedMethodEngine
    ref_out, ref_its, _ = _mirror_run(example_name, kw, MaskedMethodEngine)
    assert len(gpu_its) == len(ref_its) and all(c for _, c in gpu_its + ref_its), (gpu_its, ref_its)
    return gpu_out, gpu_its, ref_out, ref_its


@pytest.mark.parametrize('example_name,kw', EXAMPLES, ids=[e[0] for e in EXAMPLES])
def test_examples_match_the_oracle(example_name, kw):
    """The examples on the GPU against the same scripts over the oracle-backed engine (CG-adaptive with obstacles): every solve
    converges on both sides, final velocity and pressure within 1e-3 of their scale."""
    gpu_out, _, ref_out, _ = _examples(example_name, kw)
    for a, b in zip(gpu_out[0].numpy(), ref_out[0].numpy()):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-3 * max(float(np.abs(b).max()), 1.0))
    p_gpu, p_ref = gpu_out[-1].numpy(), ref_out[-1].numpy()
    np.testing.assert_allclose(p_gpu, p_ref, rtol=0, atol=1e-3 * max(float(np.abs(p_ref).max()), 1.0))


def test_batched_smoke_iteration_counts():
    """Batched_Smoke: every solve's iteration count within max(2, 10 %) of the oracle's, step for step.  (Wake_Flow has no such
    check: see test_wake_flow_projection_reaches_the_fp32_floor.)"""
    _, gpu_its, _, ref_its = _examples(*EXAMPLES[0])
    for (g, _), (r, _) in zip(gpu_its, ref_its):
        assert abs(g - r) <= max(2, r // 10), (gpu_its, ref_its)


def test_wake_flow_projection_reaches_the_fp32_floor():
    """The first Wake_Flow projection (64 x 32 x 8, Solve('CG-adaptive', 1e-5, 1e-5) from p = 0) on the masked adaptive ring.
    Iteration counts are no yardstick on this system: its fluid block has eigenvalues from 6.2e-5 to 11.1, the requested |r|^2 <=
    1.3e-7 lies below what fp32 can represent (the float64 solution rounded to fp32 and evaluated in fp32 leaves |r|^2 = 3.9e-4, with
    |p| ~ 1200 and stencil terms ~ 3000 per cell), and the iterates are rounding-chaotic - the oracle's fp32 and float64 runs of plain
    CG differ by 66 (of max|x| 231) after 10 iterations.  So every fp32 solver stops where its recurrence residual drifts below the
    tolerance (here 165 iterations; the oracle's fp32 run 531, float64 513).  What is checked: the pressure the kernel returns solves
    the oracle's operator to within 4x that fp32 floor, and lies within 1e-2 of max|p| of the float64 solution."""
    import phiflow_b200.flow as flow
    cyl = flow.geom.infinite_cylinder(x=20, y=50, radius=10, inf_dim='z')
    bnd = {'x-': flow.vec(x=2, y=0, z=0), 'x+': flow.ZERO_GRADIENT, 'y': flow.PERIODIC, 'z': flow.PERIODIC}
    v = flow.StaggeredGrid((8., 0, 0), bnd, x=64, y=32, z=8, bounds=flow.Box(x=200, y=100, z=5))
    acc, fac = flow._obstacle_masks(v, cyl)
    vd = [c.clone() for c in v.data]
    ops.mul_faces(v.dom, v.vspec, vd, fac)
    div = v.dom.centered_to_numpy(ops.divergence(v.dom, v.vspec, vd, accessible=acc))
    p = v.dom.alloc_centered()
    ops.make_incompressible(v.dom, v.vspec, vd, p, ops.cg_params(v.vspec, rtol=1e-5, atol=1e-5, max_iter=1000, method='CG-adaptive'),
                            accessible=acc)
    info = ops.last_launch_info()
    assert (info['kernel'], info['masked'], info['adaptive'], info['generic'], info['passes']) == (3, 1, 1, 1, 2), info
    rec = ops.read_results(v.dom)[0]
    assert rec['converged'] == 1 and rec['diverged'] == 0, rec
    a = v.dom.centered_to_numpy(acc)
    A = O.masked_poisson_matrix(v.res, v.dx, v.vspec[0], a)
    A64 = A.astype(np.float64)
    with O.precision(64):
        x64 = O.cg_adaptive(A64, div.astype(np.float64), np.zeros(v.res), 1e-10, 0.0, 4000)['x']
    floor = float(np.sum((div.ravel() - A.dot(x64.astype(np.float32)).astype(np.float32)).astype(np.float64) ** 2))
    got = v.dom.centered_to_numpy(p).ravel().astype(np.float64)
    true_sq = float(np.sum((div.ravel().astype(np.float64) - A64 @ got) ** 2))
    assert true_sq <= 4 * floor, (true_sq, floor, rec)
    np.testing.assert_allclose(got, x64, rtol=0, atol=1e-2 * np.abs(x64).max())
