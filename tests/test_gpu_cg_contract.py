"""
The pressure-CG contract on every kernel variant that can run it: the register-marching kernels (k_cg_poisson<2|3, MASK>,
k_laplace), the TMA ring in its generic, branch-free two-sweep, one-sweep (FUSED) and obstacle forms, at ragged shapes and at the
widths where the ring's configuration runs out, and CG-adaptive.  Every case asserts through phicuda_last_launch_info /
phicuda_last_cg_passes which variant ran, so a case that silently moves to another kernel fails.

What is checked on each variant, against the oracle (oracle/oracle_np.py, pinned against PhiML by tests/golden and
test_oracle_live_phiml.py) and against float64 recomputation:
  * warm starts: iterates after exactly k iterations from an x0 with a nonzero mean whose residual |y' - A x0|^2 is >= 100x |y'|^2
    (so a tolerance taken from the wrong base is off by orders of magnitude), and converged solves at rtol 1e-3 / 1e-5;
  * the rank-1 matrix offset with sum(x0) far from 0 (march, generic and branch-free two-sweep kernels; the one-sweep kernel does
    not take an offset);
  * the PhiCgResult record: iterations / converged / diverged, initial_residual_sq, tol_sq, residual_sq;
  * edges: max_iter = 0, an entry converged at iteration 0 next to running ones, an all-zero entry, an unbalanced singular system,
    obstacles with x0 nonzero inside them;
  * a NaN in one entry is reported as diverged and leaves the other entries bit for bit unchanged;
  * refusals: CG-adaptive and implicit diffusion have no marching kernel and raise Unsupported instead of returning numbers.

The fallback widths below are those of ring_config (ring_kernels.cu) on an H100 (227 KiB of opt-in shared memory per block) for
batch <= 4: 2-D lines of 4096 cells still fit (TY 1, 4 groups per thread, 2 stages), 4104 do not; 3-D CG lines fit up to 2408
cells (TY 1, 4 stages), 3-D CG with obstacles up to 1752 (3 stages), 3-D laplace up to 2396; the one-sweep CG takes lines up to
1024 cells (TY 1).  CG-adaptive at TY 1 needs a 7-line stage (DESIGN.md, TMA ring): 2-D 4096 still fits, 3-D 2408 does not.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from phiflow_b200 import _ops as ops
    from phiflow_b200 import _lib
    from test_gpu_cg_fused import env
    import test_gpu_kernels as K

F64 = np.float64
EPS = float(np.finfo(np.float32).eps)
SCALES = (1.0, 10.0, 0.1)            # batch entries at different scales
TRUNC_K = (1, 2, 3, 7)

BCS2 = {
    'zero': ((0.0, 0.0), (0.0, 0.0)),
    'open': (('zg', 'zg'), ('zg', 'zg')),
    'periodic': (('periodic', 'periodic'), ('periodic', 'periodic')),
    'mixed': (('zg', 'zg'), (0.0, 'zg')),
    'per_x_wall_y': (('periodic', 'periodic'), (0.0, 0.0)),
}
BCS3 = {
    'zero3': ((0.0, 0.0),) * 3,
    'open3': (('zg', 'zg'),) * 3,
    'periodic3': (('periodic', 'periodic'),) * 3,
    'mixed3': (('periodic', 'periodic'), (0.0, 'zg'), ('zg', 0.0)),
    'wall_open3': (('periodic', 'periodic'), (0.0, 0.0), (0.0, 'zg')),
}
ALL_V = {**BCS2, **BCS3}
RAGGED = {2: [(37, 22), (150, 9)], 3: [(21, 14, 9), (133, 10, 6)]}
NO_RING = {'PHICUDA_NO_RING': 1}


def dx_of(d):
    return (0.5, 0.25) if d == 2 else (0.5, 0.25, 2.0)


def march(masked=0):
    return {'kernel': 4, 'generic': 1, 'masked': masked, 'passes': 2}          # _lib.KERNEL_CG_MARCH


def ring(generic, passes=2, masked=0, **kw):
    return {'kernel': 3, 'generic': generic, 'masked': masked, 'passes': passes, **kw}   # _lib.KERNEL_CG_RING


class Case:
    """One kernel variant: grid, velocity boundary, environment, and the launch record it must produce.
    offset: the variant takes a matrix_offset; converge: converged solves are run (lines of thousands of cells with a singular
    or Neumann-only operator need thousands of iterations, those variants are checked on truncated runs only)."""

    def __init__(self, name, res, vbc, launch, envs=None, dx=None, acc=None, converge=True, adaptive=False, offset=True):
        self.name, self.res, self.vbc, self.launch = name, tuple(res), vbc, launch
        self.env = envs or {}
        self.dx = dx or dx_of(len(res))
        self.acc = acc
        self.converge, self.adaptive = converge, adaptive
        self.offset = offset and acc is None and not O.is_flexible(vbc)
        self.rank_def = not O.is_flexible(vbc)

    def __repr__(self):
        return self.name

    def matrix(self):
        if self.acc is not None:
            return O.masked_poisson_matrix_sparse(self.res, self.dx, self.vbc, self.acc)
        return O.poisson_matrix(self.res, self.dx, O.pressure_bc(self.vbc))


def obstacle_acc(res):
    """The obstacle layouts of test_gpu_kernels.test_make_incompressible_with_obstacle."""
    acc = np.ones(res, np.float32)
    if len(res) == 2:
        acc[res[0] // 3:res[0] // 2, 2:6] = 0
        acc[0:2, res[1] - 3:] = 0
    else:
        acc[res[0] // 3:res[0] // 2, 2:5, 1:4] = 0
    return acc


def _cases():
    out = []
    for i, name in enumerate(sorted(ALL_V)):
        d = len(ALL_V[name])
        res = RAGGED[d][i % 2]
        out.append(Case(f'march-{name}-{"x".join(map(str, res))}', res, ALL_V[name], march(), NO_RING))
        res = RAGGED[d][(i + 1) % 2]
        out.append(Case(f'ring-{name}-{"x".join(map(str, res))}', res, ALL_V[name], ring(1), adaptive=True))
    one = (1.0, 1.0)
    out += [
        # lines too long for the ring: the marching kernel without any environment switch
        Case('march-wide2-mixed', (4104, 10), BCS2['mixed'], march(), dx=one),
        Case('march-wide2-zero', (4104, 10), BCS2['zero'], march(), dx=one, converge=False),
        Case('march-wide3-wall_open3', (2560, 6, 5), BCS3['wall_open3'], march(), dx=(1.0,) * 3),
        Case('march-wide3-periodic3', (2560, 6, 5), BCS3['periodic3'], march(), dx=(1.0,) * 3, converge=False),
        # the ring at its limits, next to the first shape that falls back
        Case('ring2-4096-periodic', (4096, 8), BCS2['periodic'], ring(0, TY=1, groups=4, stages=2), dx=one, converge=False, adaptive=True),
        Case('ring2-4096-zero', (4096, 8), BCS2['zero'], ring(0, TY=1, groups=4, stages=2), dx=one, converge=False, adaptive=True),
        Case('ring2-4096-open', (4096, 8), BCS2['open'], ring(1, TY=1, groups=4, stages=2), dx=one, adaptive=True),
        Case('ring3-2408-open3', (2408, 6, 5), BCS3['open3'], ring(1, TY=1, stages=4), dx=(1.0,) * 3),
        Case('march3-2412-open3', (2412, 6, 5), BCS3['open3'], march(), dx=(1.0,) * 3),
        # branch-free two-sweep ring
        Case('ring-bf-zero3-256x16x12', (256, 16, 12), BCS3['zero3'], ring(0), adaptive=True),
        Case('ring-bf-periodic3-2pass', (256, 16, 12), BCS3['periodic3'], ring(0), {'PHICUDA_CG_PASSES': 2}, adaptive=True),
        Case('ring-bf-periodic3-2048', (2048, 4, 5), BCS3['periodic3'], ring(0, TY=1), dx=(1.0,) * 3, converge=False),
        # one-sweep ring (no offset: with one the launcher picks the two-sweep kernel)
        Case('fused-periodic3-256x16x12', (256, 16, 12), BCS3['periodic3'], ring(0, passes=1), offset=False),
        Case('fused-periodic3-1024', (1024, 4, 6), BCS3['periodic3'], ring(0, passes=1, TY=1), dx=(1.0,) * 3, converge=False, offset=False),
    ]
    for vname in ('zero', 'open', 'periodic', 'mixed', 'zero3', 'periodic3', 'wall_open3'):
        vbc = ALL_V[vname]
        d = len(vbc)
        for res in ([(14, 11), (128, 20)] if d == 2 else [(10, 8, 7), (128, 12, 8)]):
            tag = f'{vname}-{"x".join(map(str, res))}'
            out.append(Case(f'ring-masked-{tag}', res, vbc, ring(1, masked=1), dx=tuple(50.0 / r for r in res), acc=obstacle_acc(res)))
            out.append(Case(f'march-masked-{tag}', res, vbc, march(1), NO_RING, dx=tuple(50.0 / r for r in res), acc=obstacle_acc(res)))
    wide = (1792, 6, 5)
    out += [
        Case('march-masked-wide3-1792', wide, BCS3['wall_open3'], march(1), dx=(1.0,) * 3, acc=obstacle_acc(wide)),
        Case('ring-masked-1752', (1752, 6, 5), BCS3['wall_open3'], ring(1, masked=1, TY=1, stages=3), dx=(1.0,) * 3,
             acc=obstacle_acc((1752, 6, 5)), converge=False),
        Case('march-masked-1756', (1756, 6, 5), BCS3['wall_open3'], march(1), dx=(1.0,) * 3, acc=obstacle_acc((1756, 6, 5)), converge=False),
    ]
    return out


CASES = _cases()
BY_NAME = {c.name: c for c in CASES}


# ---- running a solve ---------------------------------------------------------------------------------------------------------

def params(case, rtol, atol, max_iter, offset=0.0, method='CG', balance=None, project=None):
    prm = ops.cg_params(case.vbc, rtol=rtol, atol=atol, max_iter=max_iter, matrix_offset=offset, method=method)
    if balance is not None:
        prm.balance_rhs = int(balance)
    if project is not None:
        prm.project_mean = int(project)
    return prm


def solve(case, dom, rhs, x0, prm, adaptive=False):
    """One CG launch with x0 (host arrays, batch first).  Returns (x, result record, launch info); asserts the variant."""
    x = dom.centered_from_numpy(x0)
    y = dom.centered_from_numpy(rhs)
    with env(**case.env):
        if case.acc is not None:
            ws, res = dom.workspace()
            acc = dom.centered_from_numpy(case.acc)
            _lib.check(_lib.load().phicuda_cg_poisson_masked_f32(C.byref(dom.grid), C.byref(ops.make_vbc(case.vbc, dom.dim)), ops._ptr(y),
                                                                 ops._ptr(x), ops._ptr(acc), C.byref(prm), ops._ptr(res), ops._ptr(ws),
                                                                 C.c_size_t(ws.numel()), ops._stream()))
        else:
            ops.cg_poisson(dom, case.vbc, y, x, prm)
        info = ops.last_launch_info()
    assert_launch(case, info, adaptive)
    return dom.centered_to_numpy(x, squeeze=False), ops.read_results(dom), info


def assert_launch(case, info, adaptive=False):
    want = dict(case.launch)
    if adaptive:
        want['adaptive'] = 1
        if want['passes'] == 1:                 # CG-adaptive runs the two-sweep body
            want['passes'] = 2
    for k, v in want.items():
        assert info[k] == v, (case.name, k, v, info)


# ---- host-side problem and references --------------------------------------------------------------------------------------

def problem(case, seed, batch=3, ratio=None, obstacle_x0=0.01):
    """Right-hand sides at SCALES, their balanced form y' (what the kernel solves), and warm starts x0 with a nonzero mean,
    scaled so that |y' - A x0|^2 >= ratio |y'|^2 (default 1000, with obstacles 100).  Inside obstacles x0 is scaled by obstacle_x0."""
    ratio = ratio or (1000.0 if case.acc is None else 100.0)
    rng = np.random.default_rng(seed)
    A = case.matrix()
    A64 = A.astype(F64)
    rhs = np.stack([rng.standard_normal(case.res).astype(np.float32) * np.float32(SCALES[b % 3]) for b in range(batch)])
    if case.acc is not None:
        rhs *= case.acc
    yb = np.stack([balanced(case, rhs[b]) for b in range(batch)])
    x0 = np.empty_like(rhs)
    for b in range(batch):
        n = rng.standard_normal(case.res) + 0.7
        if case.acc is not None:                # obstacle rows are identity rows: keep their share of r0 small
            n[case.acc == 0] *= obstacle_x0
        s = np.sqrt(1.2 * ratio * np.sum(yb[b].astype(F64) ** 2) / np.sum((A64 @ n.ravel()) ** 2))
        x0[b] = (s * n).astype(np.float32)
        r0 = yb[b].ravel().astype(F64) - A64 @ x0[b].ravel().astype(F64)
        assert np.sum(r0 ** 2) >= ratio * np.sum(yb[b].astype(F64) ** 2)
    return A, rhs, yb, x0


def balanced(case, y):
    """The rhs the kernel solves: mean removed on closed / periodic domains (with obstacles: y - acc mean(y)/mean(acc))."""
    if not case.rank_def:
        return y
    if case.acc is not None:
        return (y - case.acc * np.float32(float(np.sum(y, dtype=F64)) / float(np.sum(case.acc, dtype=F64)))).astype(np.float32)
    return (y - np.float32(np.mean(y, dtype=F64))).astype(np.float32)


def project(case, x, project_mean=None):
    """The kernel's final mean projection (acc-weighted with obstacles)."""
    if not (case.rank_def if project_mean is None else project_mean):
        return x
    if case.acc is not None:
        return x - case.acc * (np.sum(x * case.acc, dtype=F64) / np.sum(case.acc, dtype=F64))
    return x - x.mean(dtype=F64)


def reference(case, A, y, x0, rtol, atol, k, offset=None, adaptive=False, exact=False):
    """The oracle's fp32 run; exact: also its float64 run (ref['x64'], ref['residual_sq64'])."""
    fn = O.cg_adaptive if adaptive else O.cg
    ref = fn(A, y, x0, rtol, atol, k, offset)
    if exact:
        with O.precision(64):
            r64 = fn(A.astype(F64), y.astype(F64), x0.astype(F64), rtol, atol, k, offset)
        ref['x64'], ref['residual_sq64'] = r64['x'], r64['residual_sq']
    return ref


def check_iterate(case, got, ref, project_mean=None, rel=2e-5):
    """got within 2e-5 max|x| of the oracle; where the oracle's own fp32 run is further than that from its float64 run (a warm
    start far from the solution with an isolated large eigenvalue: obstacle identity rows, the offset c N), within 10x that gap."""
    xr = project(case, ref['x'].reshape(case.res).astype(F64), project_mean)
    tol = rel * max(1.0, np.abs(xr).max())
    if 'x64' in ref:
        tol = max(tol, 10 * np.abs(xr - project(case, ref['x64'].reshape(case.res), project_mean)).max())
    np.testing.assert_allclose(got, xr, rtol=0, atol=tol, err_msg=case.name)


def check_record_start(case, rec, A, y, x0, rtol, atol, offset, adaptive):
    """initial_residual_sq = |y' - (A + c 11^T) x0|^2, tol_sq = max(rtol^2 |y' - A x0|^2, atol^2) (CG-adaptive: rtol^2 |y'|^2),
    both against float64."""
    A64 = A.astype(F64)
    rt = y.ravel().astype(F64) - A64 @ x0.ravel().astype(F64)
    r = rt - (offset or 0.0) * np.sum(x0, dtype=F64)
    base = np.sum(y.astype(F64) ** 2) if adaptive else np.sum(rt ** 2)
    np.testing.assert_allclose(rec['initial_residual_sq'], np.sum(r ** 2), rtol=1e-4, err_msg=f'{case.name} initial_residual_sq')
    np.testing.assert_allclose(rec['tol_sq'], max(rtol ** 2 * base, atol ** 2), rtol=1e-4, err_msg=f'{case.name} tol_sq')


def check_truncated(case, rec, ref, k):
    assert (int(rec['iterations']), int(rec['converged']), int(rec['diverged'])) == (k, int(ref['converged']), int(ref['diverged'])) \
        == (ref['iterations'], 0, 0), (case.name, rec, ref['iterations'])
    # rtol 1e-3 against the exact recurrence, or 10x the oracle's own fp32 error where that is larger (see check_iterate)
    rtol = max(1e-3, 10 * abs(ref['residual_sq'] / ref['residual_sq64'] - 1))
    np.testing.assert_allclose(rec['residual_sq'], ref['residual_sq64'], rtol=rtol, err_msg=f'{case.name} residual_sq k={k}')


def check_converged(case, rec, ref, got, A, y, rtol, offset=None):
    n_ref = ref['iterations']
    assert ref['converged'] and rec['converged'] == 1 and rec['diverged'] == 0, (case.name, rec, n_ref)
    assert abs(int(rec['iterations']) - n_ref) <= max(2, n_ref // 10), (case.name, int(rec['iterations']), n_ref)
    assert rec['residual_sq'] <= rec['tol_sq'], (case.name, rec)
    r = y.ravel().astype(F64) - A.astype(F64) @ got.ravel().astype(F64)
    true_sq = float(np.sum(r * r))
    f = 4.0 if rtol > 1e-4 else 40.0
    # the fp32 recurrence residual drifts from the true one by O(eps cond); with an offset, |r|^2 also holds c^2 N sum(x)^2.  An
    # fp32 solve cannot get the true residual below ~eps |r0| (attainable accuracy): CG-adaptive at rtol 1e-5 from a warm start with
    # |r0| >> |y'| asks for less than that
    floor = (100 * EPS) ** 2 * float(rec['initial_residual_sq'])
    assert true_sq <= f * max(float(rec['residual_sq']), floor), (case.name, true_sq, floor, rec)
    if offset is None:
        assert true_sq >= float(rec['residual_sq']) / f, (case.name, true_sq, rec)


def domain(case, batch=3):
    return ops.Domain(case.res, case.dx, batch, vbc=case.vbc)


# ---- A + B1-B3: warm-start iterates, the offset, the record -----------------------------------------------------------------

@pytest.mark.parametrize('case', CASES, ids=str)
def test_warm_start_truncated(case):
    """Exactly k iterations from a warm start with a nonzero mean: iterates and the full result record against the oracle."""
    A, rhs, y, x0 = problem(case, 101)
    dom = domain(case)
    for k in TRUNC_K:
        got, rec, _ = solve(case, dom, rhs, x0, params(case, 1e-12, 0.0, k))
        for b in range(3):
            ref = reference(case, A, y[b], x0[b], 1e-12, 0.0, k, exact=True)
            check_truncated(case, rec[b], ref, k)
            check_record_start(case, rec[b], A, y[b], x0[b], 1e-12, 0.0, None, False)
            check_iterate(case, got[b], ref)


@pytest.mark.parametrize('case', [c for c in CASES if c.converge], ids=str)
@pytest.mark.parametrize('rtol', [1e-3, 1e-5])
def test_warm_start_converged(case, rtol):
    """Converged solves from the warm start (with obstacles: x0 = 0 inside them, where CG would otherwise spend its fp32 accuracy
    on the identity rows): iteration counts, the record, the true residual and the solution."""
    A, rhs, y, x0 = problem(case, 102, obstacle_x0=0.0)
    dom = domain(case)
    atol = 1e-5
    got, rec, _ = solve(case, dom, rhs, x0, params(case, rtol, atol, 4000))
    for b in range(3):
        ref = reference(case, A, y[b], x0[b], rtol, atol, 4000)
        check_converged(case, rec[b], ref, got[b], A, y[b], rtol)
        check_record_start(case, rec[b], A, y[b], x0[b], rtol, atol, None, False)
        xr = project(case, ref['x'].reshape(case.res).astype(F64))
        np.testing.assert_allclose(got[b], xr, rtol=0, atol=20 * rtol * np.abs(xr).max(), err_msg=case.name)


def offset_problem(case, seed):
    """x0 with sum(x0) so far from 0 that the offset term c sum(x0) carries at least as much of |r0|^2 as y' - A x0."""
    A, rhs, y, x0 = problem(case, seed)
    c = O.estimate_matrix_offset(A, int(np.prod(case.res)), np.random.default_rng(0))
    n = x0[0].size
    for b in range(3):
        rt = np.sqrt(np.sum((y[b].ravel().astype(F64) - A.astype(F64) @ x0[b].ravel().astype(F64)) ** 2))
        x0[b] += np.float32(rt / (c * n * np.sqrt(n)))         # constant: A x0 is unchanged, c sum(x0) sqrt(N) >= |rt|
        r = y[b].ravel().astype(F64) - A.astype(F64) @ x0[b].ravel().astype(F64) - c * np.sum(x0[b], dtype=F64)
        assert np.sum(r ** 2) >= 1.5 * rt ** 2        # |r0|^2 (with the offset) and the tolerance base (without) are far apart
    return A, rhs, y, x0, c


@pytest.mark.parametrize('case', [c for c in CASES if c.offset], ids=str)
def test_matrix_offset_warm_start(case):
    """(A + c 11^T) with sum(x0) far from 0: the offset part of r0 (c sum(x0)) is not multiplied by zero.  One and two iterations:
    from such a start the constant direction (eigenvalue c N) dominates r0, and beyond two iterations fp32 runs of the recurrence
    part ways (the oracle's own fp32 and float64 runs differ by up to 100 % at k = 7).  Converged offset solves from x0 = 0 are
    test_gpu_kernels.test_cg_matrix_offset_matches_reference_formulation."""
    A, rhs, y, x0, c = offset_problem(case, 103)
    dom = domain(case)
    for k in (1, 2):
        got, rec, _ = solve(case, dom, rhs, x0, params(case, 1e-12, 0.0, k, offset=c))
        for b in range(3):
            ref = reference(case, A, y[b], x0[b], 1e-12, 0.0, k, offset=c, exact=True)
            check_truncated(case, rec[b], ref, k)
            check_record_start(case, rec[b], A, y[b], x0[b], 1e-12, 0.0, c, False)
            check_iterate(case, got[b], ref)


@pytest.mark.parametrize('case', [c for c in CASES if c.adaptive], ids=str)
def test_cg_adaptive_warm_start(case):
    """CG-adaptive takes its tolerance from |y'|^2, not from |y' - A x0|^2; the two differ by >= 100x here."""
    A, rhs, y, x0 = problem(case, 104)
    dom = domain(case)
    for k in TRUNC_K:
        got, rec, _ = solve(case, dom, rhs, x0, params(case, 1e-12, 0.0, k, method='CG-adaptive'), adaptive=True)
        for b in range(3):
            ref = reference(case, A, y[b], x0[b], 1e-12, 0.0, k, adaptive=True, exact=True)
            check_truncated(case, rec[b], ref, k)
            check_record_start(case, rec[b], A, y[b], x0[b], 1e-12, 0.0, None, True)
            check_iterate(case, got[b], ref)
    if case.converge:
        for rtol in (1e-3, 1e-5):
            got, rec, _ = solve(case, dom, rhs, x0, params(case, rtol, 1e-5, 4000, method='CG-adaptive'), adaptive=True)
            for b in range(3):
                ref = reference(case, A, y[b], x0[b], rtol, 1e-5, 4000, adaptive=True)
                check_converged(case, rec[b], ref, got[b], A, y[b], rtol)
                check_record_start(case, rec[b], A, y[b], x0[b], rtol, 1e-5, None, True)


# ---- B4: edges ---------------------------------------------------------------------------------------------------------------

EDGE = ['march-mixed-37x22', 'march-mixed3-133x10x6', 'march-wide2-mixed', 'ring-mixed-150x9', 'ring-open3-21x14x9',
        'ring-bf-zero3-256x16x12', 'fused-periodic3-256x16x12', 'ring-masked-wall_open3-10x8x7', 'march-masked-wall_open3-10x8x7',
        'march-masked-zero-14x11', 'ring-masked-periodic-128x20']


@pytest.mark.parametrize('name', EDGE)
def test_max_iter_zero(name):
    """max_iter = 0: no iteration, the record holds r0 as the final residual and x is x0 bit for bit (no mean projection)."""
    case = BY_NAME[name]
    A, rhs, y, x0 = problem(case, 105)
    got, rec, _ = solve(case, domain(case), rhs, x0, params(case, 1e-5, 1e-5, 0, project=0))
    for b in range(3):
        assert rec[b]['iterations'] == 0 and rec[b]['converged'] == 0 and rec[b]['diverged'] == 0, rec[b]
        assert rec[b]['residual_sq'] == rec[b]['initial_residual_sq'], rec[b]
        check_record_start(case, rec[b], A, y[b], x0[b], 1e-5, 1e-5, None, False)
    np.testing.assert_array_equal(got, x0)


@pytest.mark.parametrize('name', EDGE)
def test_entries_converged_at_start(name):
    """Entry 1 starts at its own solution (|r0| below atol), entry 2 is all zero with x0 = 0 (tol 0 >= |r0|^2 = 0 with atol 0
    in a separate run); entry 0 runs.  The stopped entries never enter a CG pass: x stays x0 bit for bit."""
    case = BY_NAME[name]
    A, rhs, y, x0 = problem(case, 106)
    rng = np.random.default_rng(7)
    v = rng.standard_normal(case.res).astype(np.float32)
    if case.acc is not None:
        v *= case.acc
    Av = (A.astype(F64) @ v.ravel().astype(F64)).reshape(case.res)
    rhs[1], x0[1] = Av.astype(np.float32), v
    rhs[2], x0[2] = 0.0, 0.0
    A64 = A.astype(F64)
    r0 = [float(np.sum((balanced(case, rhs[b]).ravel().astype(F64) - A64 @ x0[b].ravel().astype(F64)) ** 2)) for b in range(2)]
    atol = 1e-3 * float(np.sqrt(np.sum(Av ** 2)))
    assert r0[1] < 1e-4 * atol ** 2 and r0[0] > 100 * atol ** 2
    for at in (atol, 0.0):
        got, rec, _ = solve(case, domain(case), rhs, x0, params(case, 1e-12 if at == 0.0 else 1e-3, at, 7, project=0))
        assert rec[0]['iterations'] == 7 and rec[0]['converged'] == 0, rec
        stopped = (1, 2) if at > 0 else (2,)
        for b in stopped:
            assert rec[b]['iterations'] == 0 and rec[b]['converged'] == 1 and rec[b]['diverged'] == 0, (b, rec[b])
            np.testing.assert_array_equal(got[b], x0[b])
        ref = reference(case, A, y[0], x0[0], 1e-12 if at == 0.0 else 1e-3, at, 7, exact=True)
        check_iterate(case, got[0], ref, project_mean=False)
        check_truncated(case, rec[0], ref, 7)


@pytest.mark.parametrize('name', ['march-zero-37x22', 'march-zero3-133x10x6', 'march-wide2-zero', 'ring-zero-150x9',
                                  'ring-periodic3-133x10x6', 'ring-bf-zero3-256x16x12', 'fused-periodic3-256x16x12',
                                  'ring-masked-zero3-10x8x7', 'march-masked-zero3-10x8x7'])
def test_unbalanced_singular_system(name):
    """balance_rhs = 0, project_mean = 0 on a closed / periodic domain: plain CG on the singular system, as the oracle runs it.
    The system is inconsistent, so the iterates drift along the null space, which dominates max|x|: three iterations are compared,
    to 4e-5 of max|x|."""
    case = BY_NAME[name]
    A, rhs, _, x0 = problem(case, 107)
    rhs += np.float32(0.3) * np.float32(np.abs(rhs).max())            # a large mean: inconsistent system
    if case.acc is not None:
        rhs *= case.acc
    dom = domain(case)
    for k in (1, 2, 3):
        got, rec, _ = solve(case, dom, rhs, x0, params(case, 1e-12, 0.0, k, balance=0, project=0))
        for b in range(3):
            ref = reference(case, A, rhs[b], x0[b], 1e-12, 0.0, k, exact=True)
            check_truncated(case, rec[b], ref, k)
            check_record_start(case, rec[b], A, rhs[b], x0[b], 1e-12, 0.0, None, False)
            check_iterate(case, got[b], ref, project_mean=False, rel=4e-5)


@pytest.mark.parametrize('name', [c.name for c in CASES if c.acc is not None and c.converge])
def test_masked_warm_start_inside_obstacles(name):
    """Obstacle cells are identity rows: a pressure that is nonzero inside obstacles is part of r0 and of the iterates."""
    case = BY_NAME[name]
    A, rhs, y, x0 = problem(case, 108)
    assert np.abs(x0[:, case.acc == 0]).min() > 0
    got, rec, _ = solve(case, domain(case), rhs, x0, params(case, 1e-12, 0.0, 3))
    for b in range(3):
        ref = reference(case, A, y[b], x0[b], 1e-12, 0.0, 3, exact=True)
        check_iterate(case, got[b], ref)
        assert np.abs(got[b][case.acc == 0] - x0[b][case.acc == 0]).max() > 0       # the obstacle cells move as well


# ---- B5: non-finite input and batch independence ------------------------------------------------------------------------------

NAN_CASES = ['march-periodic-150x9', 'march-mixed3-133x10x6', 'march-wide3-wall_open3', 'ring-open-150x9', 'ring-zero3-21x14x9',
             'ring2-4096-zero', 'ring-bf-zero3-256x16x12', 'fused-periodic3-256x16x12', 'ring-masked-wall_open3-10x8x7',
             'march-masked-zero-14x11']


@pytest.mark.parametrize('name', NAN_CASES)
def test_nan_entry_is_diverged_and_isolated(name):
    """One NaN in entry 1: entry 1 reports diverged at iteration 0; entries 0 and 2 are bit-identical to a run where entry 1 is
    all zeros (reductions are per entry and in a fixed order)."""
    case = BY_NAME[name]
    _, rhs, _, x0 = problem(case, 109)
    x0[1] = 0.0
    dom = domain(case)
    prm = params(case, 1e-5, 1e-5, 40)
    clean = rhs.copy()
    clean[1] = 0.0
    bad = clean.copy()
    bad[1][(0,) * len(case.res)] = np.nan
    got_c, rec_c, _ = solve(case, dom, clean, x0, prm)
    got_n, rec_n, _ = solve(case, dom, bad, x0, prm)
    assert (rec_n[1]['diverged'], rec_n[1]['converged'], rec_n[1]['iterations']) == (1, 0, 0), rec_n[1]
    for b in (0, 2):
        assert rec_n[b].tobytes() == rec_c[b].tobytes(), (rec_n[b], rec_c[b])
        np.testing.assert_array_equal(got_n[b], got_c[b])
    assert rec_c[0]['iterations'] > 0


# ---- B6: refusals on grids without a ring configuration ---------------------------------------------------------------------------

@pytest.mark.parametrize('name', ['march-open-37x22', 'march-zero3-133x10x6', 'march-wide2-mixed', 'march-wide3-periodic3'])
def test_refusals_without_ring(name):
    """CG-adaptive and implicit diffusion exist on the TMA ring only: on the marching path they raise Unsupported with a message
    and leave x untouched."""
    case = BY_NAME[name]
    _, rhs, _, x0 = problem(case, 110)
    dom = domain(case)
    spec = O.uniform_bc(len(case.res), 'zg')
    with env(**case.env):
        x = dom.centered_from_numpy(x0)
        before = x.clone()
        with pytest.raises(_lib.Unsupported, match='CG-adaptive'):
            ops.cg_poisson(dom, case.vbc, dom.centered_from_numpy(rhs), x, params(case, 1e-5, 1e-5, 100, method='CG-adaptive'))
        assert torch.equal(x, before)
        u = dom.centered_from_numpy(rhs)
        with pytest.raises(_lib.Unsupported, match='does not fit'):
            ops.diffuse_implicit(dom, spec, u, 0.5, x0=x)
        with pytest.raises(_lib.Unsupported, match='does not fit'):
            ops.diffuse_implicit_varying(dom, spec, u, torch.ones_like(u[:1]), 0.5, x0=x)
        assert torch.equal(x, before)


def test_flow_default_solve_without_ring():
    """The mirror's default Solve() maps to CG-adaptive, which has no marching kernel: without the ring it raises Unsupported
    (the reference-side façade falls through on it); Solve('CG') runs on the marching kernel."""
    from phiflow_b200.flow import StaggeredGrid, Solve, fluid, ZERO
    rng = np.random.default_rng(111)
    v = StaggeredGrid([rng.standard_normal((15, 20)).astype(np.float32), rng.standard_normal((16, 19)).astype(np.float32)], ZERO, x=16, y=20)
    with env(PHICUDA_NO_RING=1):
        with pytest.raises(_lib.Unsupported):
            fluid.make_incompressible(v)
        fluid.make_incompressible(v, solve=Solve('CG', 1e-5, 1e-5))
        assert ops.last_launch_info()['kernel'] == _lib.KERNEL_CG_MARCH


# ---- the marching laplace and the fused entry points --------------------------------------------------------------------------

@pytest.mark.parametrize('name', sorted(list(ALL_V) + ['one', 'const_mix']))
def test_march_laplace(name):
    """k_laplace (the fallback of phicuda_laplace_f32 / laplace_axpy_f32) on every boundary set, ragged shapes, batch 1 and 3."""
    with env(PHICUDA_NO_RING=1):
        K.test_laplace(name)
        info = ops.last_launch_info()
    assert info['kernel'] == _lib.KERNEL_LAPLACE_MARCH and info['generic'] == 1, info


@pytest.mark.parametrize('res,bname', [((4104, 10), 'mixed'), ((4104, 10), 'periodic'), ((2560, 6, 5), 'mixed3'), ((2560, 6, 5), 'open3'),
                                       ((4096, 10), 'periodic'), ((2396, 6, 5), 'mixed3')])
def test_laplace_wide(res, bname):
    """Lines longer than the laplace ring takes fall back to k_laplace without any switch; 4096 (2-D) and 2396 (3-D) still fit."""
    bc = O.pressure_bc(ALL_V[bname])
    d = len(res)
    rng = np.random.default_rng(112)
    dom = ops.Domain(res, K.dx_of(d), 3)
    a = rng.standard_normal((3,) + res).astype(np.float32)
    out = dom.centered_to_numpy(ops.laplace(dom, bc, dom.centered_from_numpy(a)), squeeze=False)
    fits = res[0] <= (4096 if d == 2 else 2396)
    info = ops.last_launch_info()
    assert info['kernel'] == (_lib.KERNEL_LAPLACE_RING if fits else _lib.KERNEL_LAPLACE_MARCH), info
    scale = np.abs(a).max() * sum(4.0 / h ** 2 for h in K.dx_of(d))
    for b in range(3):
        np.testing.assert_allclose(out[b], O.laplace(a[b], K.dx_of(d), bc), rtol=0, atol=4 * EPS * scale)
    out2 = dom.centered_to_numpy(ops.laplace_axpy(dom, bc, dom.centered_from_numpy(a), 0.01), squeeze=False)
    assert ops.last_launch_info()['kernel'] == info['kernel']
    for b in range(3):
        np.testing.assert_allclose(out2[b], a[b] + np.float32(0.01) * O.laplace(a[b], K.dx_of(d), bc), rtol=0, atol=4 * EPS * scale)


@pytest.mark.parametrize('vname', ['mixed', 'mixed3'])
def test_make_incompressible_march(vname):
    """make_incompressible through the fused C-ABI entry point on the marching CG, against the oracle."""
    with env(PHICUDA_NO_RING=1):
        K.test_make_incompressible(vname, False)
        info = ops.last_launch_info()
    assert info['kernel'] == _lib.KERNEL_CG_MARCH and info['passes'] == 2, info


def test_plume_step_march():
    """plume_step (warm-started pressure, 3 steps) on the marching CG, against the oracle."""
    with env(PHICUDA_NO_RING=1):
        K.test_plume_step('mixed3', True)
        info = ops.last_launch_info()
    assert info['kernel'] == _lib.KERNEL_CG_MARCH, info
