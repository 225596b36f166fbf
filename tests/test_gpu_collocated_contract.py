"""
The pressure-solve contract of the CenteredGrid (collocated, wide-stencil) projection, phicuda_make_incompressible_centered_host_f32
(csrc/collocated_kernels.cu): its own host loop, which polls the stopping flags every 8 iterations, and its own matrix-offset terms,
with the stopping rule, result record and right-hand-side balancing of the persistent CG kernels (csrc/cg_common.cuh).  Every
CenteredGrid projection runs through it (phi_cuda façade and _ops), so it is held to what
test_gpu_cg_contract.py holds the staggered solvers to, against the oracle (oracle/oracle_np.py, pinned against PhiML by
tests/golden/phiml_collocated.npz):
  * the stencils cell by cell, at bounds derived from the operations (not relative to max|ref|), with scalar, mixed and
    per-component constant boundaries, whose constants must reach the right-hand side and never the operator;
  * iterates after exactly k iterations from a warm start with a nonzero mean, k straddling the poll window, and converged solves;
  * every field of the PhiCgResult record against float64;
  * entries that stop inside a poll window next to running ones, max_iter = 0, the divergence rule, NaN isolation and run-to-run
    reproducibility, bit for bit;
  * refusals before any CUDA work.
Shapes include lines of 130 and 257 cells, which span two and three of the kernels' 128-thread x blocks, so every dot product is
summed over several blocks per line.

Iterates.  On this operator fp32 iterates drift from exact arithmetic by far more than a fixed tolerance (measured with the oracle:
up to 1e-2 max|x| after 16 iterations on a closed box from a warm start), so an iterate x is compared with the oracle run in float64,
x64, and must be at least nearly as accurate as the oracle's own fp32 run x32:
    max|x - x64| <= max(C max|x32 - x64|, 2e-5 max(1, max|x64|)),   C = DRIFT = 4.
The recurrence's |r|^2 at exit (residual_sq) is more sensitive still: on the small closed and periodic boxes the oracle's own fp32
run ends up to 10x away from its float64 run, and a NumPy replay of the kernel's arithmetic (dot products in double) up to 200x.  It
is compared within max(1e-3, 10x the oracle's own relative fp32 error) wherever that error is below 1/2, i.e. wherever fp32 still
resolves the recurrence at all.

Matrix offset.  The reference estimates one rank-1 offset c per batch entry (PhiML _optimize.py:705-714); the C ABI takes one c for
the whole batch.  The tests draw c once per case with O.estimate_matrix_offset and pass the same value to both sides.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from phiflow_b200 import _ops as ops
    from phiflow_b200 import _lib

F64 = np.float64
EPS = float(np.finfo(np.float32).eps)
SCALES = (1.0, 10.0, 0.1)            # batch entries at different scales
TRUNC_K = (1, 2, 3, 7, 8, 9, 17)     # the host reads the stopping flags after iterations 8, 16, ... and at max_iter
DRIFT = 4

BCS = {
    # the boundary sets of test_gpu_collocated.py
    'zero': ((0.0, 0.0), (0.0, 0.0)),
    'open': (('zg', 'zg'), ('zg', 'zg')),
    'periodic': (('periodic', 'periodic'), ('periodic', 'periodic')),
    'mixed': (('zg', 'zg'), (0.0, 'zg')),
    'zero3': ((0.0, 0.0),) * 3,
    'mixed3': (('periodic', 'periodic'), (0.0, 'zg'), ('zg', 0.0)),
    # constants: the same on every component, mixed with open sides, and per component (a list of one spec per component)
    'one': ((1.0, 1.0), (1.0, 1.0)),
    'const_mix': (('zg', 0.5), (-0.25, 'zg')),
    'lid': [((0.0, 0.0), (0.0, 1.0)), ((0.0, 0.0), (0.0, 0.0))],             # Lid_Driven_Cavity: {'y+': vec(x=1, y=0)}
    'inflow3': [((0.5, 'zg'), ('periodic', 'periodic'), (0.0, 0.0)),
                ((-0.25, 'zg'), ('periodic', 'periodic'), (0.0, 0.0)),
                ((0.125, 'zg'), ('periodic', 'periodic'), (0.0, 0.0))],        # inflow vec(0.5, -0.25, 0.125) at x-
}


class Case:
    def __init__(self, name, res, dx=None):
        self.name, self.res, self.vbc = name, tuple(res), BCS[name]
        self.d = len(res)
        self.dx = tuple(float(np.float32(v)) for v in (dx or ((0.5, 0.25) if self.d == 2 else (0.5, 0.25, 2.0))))
        self.kinds = O.kinds_of(self.vbc)
        self.vbc0 = O.remove_constant_offset(self.kinds)
        self.pbc = O.pressure_bc(self.vbc)
        self.rank_def = not O.is_flexible(self.vbc)

    def __repr__(self):
        return f'{self.name}-{"x".join(map(str, self.res))}'

    @property
    def n(self):
        return int(np.prod(self.res))


CASES = [Case('zero', (17, 12)), Case('open', (130, 5)), Case('periodic', (16, 9)), Case('mixed', (257, 3)),
         Case('one', (13, 10)), Case('const_mix', (130, 4)), Case('lid', (16, 12), dx=(100 / 16, 100 / 12)),
         Case('zero3', (11, 9, 7)), Case('mixed3', (130, 4, 3)), Case('inflow3', (257, 3, 2))]
BY_NAME = {repr(c): c for c in CASES}
# the flexible sets (no rank-1 offset) on which CG-adaptive converges from smooth inputs in a few hundred iterations at most; on
# 'mixed' at 257 x 3 it is flagged diverged after 20 iterations, in the oracle as well, and 'inflow3' at 257 x 3 x 2 needs 500-1200
# iterations, over which the fp32 recurrence residual leaves the true one behind by 10x (the oracle's fp32 run alike)
CONVERGE = ['open-130x5', 'const_mix-130x4', 'mixed3-130x4x3']


@functools.lru_cache(maxsize=None)
def matrices(key):
    """(A in float64, A in fp32, offset c or None), once per case: wide_poisson_matrix builds A column by column."""
    case = BY_NAME[key]
    with O.precision(64):
        A64 = O.wide_poisson_matrix(case.res, case.dx, case.kinds)
    A32 = A64.astype(np.float32)
    c = O.estimate_matrix_offset(A32, case.n, np.random.default_rng(0)) if case.rank_def else None
    return A64, A32, c


# ---- host-side references ------------------------------------------------------------------------------------------------------

def rhs(case, v, bits):
    """y' = the centred divergence of v (constants of the velocity boundary included), balanced on rank-deficient systems."""
    with O.precision(bits):
        t = F64 if bits == 64 else np.float32
        y = O.divergence_centered([a.astype(t) for a in v], case.dx, O.component_bcs(case.vbc, case.d))
        if case.rank_def:
            y = y - np.mean(y, dtype=t)
    return y


def oracle(case, v, x0, rtol, atol, max_iter, bits):
    A64, A32, c = matrices(repr(case))
    with O.precision(bits):
        t = F64 if bits == 64 else np.float32
        return O.cg_adaptive(A64 if bits == 64 else A32, rhs(case, v, bits), x0.astype(t), rtol, atol, max_iter, c)


def iterate_bound(x64, x32):
    return max(DRIFT * np.abs(x32 - x64).max(), 2e-5 * max(1.0, np.abs(x64).max()))


def check_iterate(case, got, case_v, x0, k, what=''):
    """got = the GPU iterate after k iterations from x0 (see the module docstring for the bound)."""
    r64 = oracle(case, case_v, x0, 0.0, 0.0, k, 64)
    r32 = oracle(case, case_v, x0, 0.0, 0.0, k, 32)
    x64, x32 = r64['x'].reshape(case.res), r32['x'].reshape(case.res).astype(F64)
    err, bound = np.abs(got - x64).max(), iterate_bound(x64, x32)
    assert err <= bound, (repr(case), what, k, err, bound)
    return r64, r32


def halfsum(a, dx, bc, c):
    """(|a[i+1]| + |a[i-1]|) / (2 dx_c) along axis c, ghosts from bc."""
    q = np.abs(O.pad_axis(a, c, 1, 1, bc[c]))
    n = a.shape[c]
    return (np.take(q, np.arange(2, n + 2), axis=c) + np.take(q, np.arange(0, n), axis=c)) / (2 * dx[c])


def check_correction(case, v, p, v_out):
    """v_out = v - gradient_centered(p) for the GPU's own p.  The kernel's gradient is phi_div(p[i+1] - p[i-1], 2 dx, 1 / (2 dx)): one
    rounding of the difference (eps/2 relative) and a quotient within 1 ulp of the IEEE one (1.5 eps), so it is within
    2 eps (|p[i+1]| + |p[i-1]|) / (2 dx) of the exact gradient; the subtraction adds one rounding, eps/2 |v_out| (bounded by eps)."""
    with O.precision(64):
        g = O.gradient_centered(p.astype(F64), case.dx, case.pbc)
    for c in range(case.d):
        want = v[c].astype(F64) - g[c]
        bound = 2 * EPS * halfsum(p.astype(F64), case.dx, case.pbc, c) + EPS * np.abs(want) + 1e-38
        err = np.abs(v_out[c] - want)
        assert (err <= bound).all(), (repr(case), c, float(err.max()), float((err / bound).max()))


# ---- running the entry point ----------------------------------------------------------------------------------------------------

def run(case, v, x0, rtol, atol, max_iter):
    """One projection of the batch v (list of components, batch first) from the warm start x0: (v_out, p, records)."""
    batch = x0.shape[0]
    dom = ops.Domain(case.res, case.dx, batch)
    dv = [dom.centered_from_numpy(a) for a in v]
    dp = dom.centered_from_numpy(x0)
    _, _, c = matrices(repr(case))
    ops.make_incompressible_centered(dom, case.vbc, dv, dp, rtol=rtol, atol=atol, max_iter=max_iter, matrix_offset=c)
    rec = ops.read_results(dom).copy()
    return [dom.centered_to_numpy(t, squeeze=False) for t in dv], dom.centered_to_numpy(dp, squeeze=False), rec


def entry(v, b):
    return [a[b] for a in v]


def white_problem(case, seed, ratio=100.0):
    """White-noise velocities at SCALES and warm starts with a nonzero mean, scaled so that |y' - (A + c 11^T) x0|^2 >= ratio |y'|^2."""
    rng = np.random.default_rng(seed)
    A64, _, c = matrices(repr(case))
    v = [np.stack([rng.standard_normal(case.res).astype(np.float32) * np.float32(s) for s in SCALES]) for _ in range(case.d)]
    x0 = np.empty((len(SCALES),) + case.res, np.float32)
    for b in range(len(SCALES)):
        nz = rng.standard_normal(case.res) + 2.0
        y = rhs(case, entry(v, b), 64).ravel()
        r = A64 @ nz.ravel() + (c or 0.0) * nz.sum()
        x0[b] = (nz * np.sqrt(1.5 * ratio * np.sum(y ** 2) / np.sum(r ** 2))).astype(np.float32)
        assert initial_residual_sq(case, y, x0[b]) >= ratio * np.sum(y ** 2)
    return v, x0


def smooth_problem(case, seed):
    """Gaussian blobs (as test_gpu_collocated: white noise leaves the range of the singular, non-symmetric operator) at SCALES, and a
    small smooth warm start."""
    rng = np.random.default_rng(seed)
    idx = np.indices(case.res).astype(F64)

    def blob(amp):
        centre = rng.uniform(0.3, 0.7, case.d) * np.array(case.res)
        sig = np.array(case.res) / 4.0
        return (amp * np.exp(-0.5 * sum(((idx[a] - centre[a]) / sig[a]) ** 2 for a in range(case.d)))).astype(np.float32)

    v = [np.stack([blob(0.1 * s) for s in SCALES]) for _ in range(case.d)]
    x0 = np.stack([blob(0.01 * s) for s in SCALES])
    return v, x0


def initial_residual_sq(case, y64, x0):
    A64, _, c = matrices(repr(case))
    x = x0.ravel().astype(F64)
    r = y64.ravel() - (A64 @ x + (c or 0.0) * x.sum())
    return float(np.sum(r ** 2))


def check_record_start(case, rec, v, x0, rtol, atol):
    """initial_residual_sq = |y' - (A + c 11^T) x0|^2 and tol_sq = max(rtol^2 |y'|^2, atol^2), against float64 (the former within
    1e-5, or eps^2 |y'|^2 when x0 solves the system up to rounding)."""
    y = rhs(case, v, 64)
    np.testing.assert_allclose(rec['initial_residual_sq'], initial_residual_sq(case, y, x0), rtol=1e-5, atol=EPS ** 2 * np.sum(y ** 2),
                               err_msg=f'{case!r} initial_residual_sq')
    np.testing.assert_allclose(rec['tol_sq'], max(rtol ** 2 * np.sum(y ** 2), atol ** 2), rtol=1e-5, err_msg=f'{case!r} tol_sq')


def check_residual_sq(case, rec, r64, r32):
    """residual_sq = the recurrence |r|^2 at exit (the initial residual when the solve stops at iteration 0)."""
    if r64['iterations'] == 0:
        assert rec['residual_sq'] == rec['initial_residual_sq'], (repr(case), rec)
        return
    own = abs(r32['residual_sq'] / r64['residual_sq'] - 1)
    if own < 0.5:
        np.testing.assert_allclose(rec['residual_sq'], r64['residual_sq'], rtol=max(1e-3, 10 * own), err_msg=f'{case!r} residual_sq')


# ---- the stencils -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('key', list(BY_NAME))
def test_wide_laplace_cellwise(key):
    """phicuda_wide_laplace_f32 against the float64 composition divergence_centered(gradient_centered(x)), cell by cell.  Per gradient
    component g_c = G_c (1 + d), |d| <= 2 eps (one rounding of the difference, a phi_div quotient within 1 ulp of the IEEE one); per
    divergence term the difference of two such g adds eps/2 and its quotient 1.5 eps, and summing the DIM terms eps Sum|term_c|, so
        |out - ref| <= 5 eps Sum_c (|G_c[i+1]| + |G_c[i-1]|) / (2 dx_c)
    to first order, with G the exact gradient and its ghosts from the velocity boundary with constants removed; 6 eps covers the
    second-order terms.  The constants must not reach the operator: the result equals bit for bit the one with every constant zeroed."""
    case = BY_NAME[key]
    rng = np.random.default_rng(61)
    x = (rng.standard_normal((2,) + case.res) + 1.5).astype(np.float32)
    dom = ops.Domain(case.res, case.dx, 2)
    out = ops.wide_laplace(dom, case.vbc, dom.centered_from_numpy(x))
    zeroed = ops.wide_laplace(dom, case.vbc0, dom.centered_from_numpy(x))
    assert torch.equal(out, zeroed), key
    got = dom.centered_to_numpy(out, squeeze=False)
    for b in range(2):
        with O.precision(64):
            G = O.gradient_centered(x[b].astype(F64), case.dx, case.pbc)
            ref = O.divergence_centered(G, case.dx, [case.vbc0] * case.d)
        S = sum(halfsum(G[c], case.dx, case.vbc0, c) for c in range(case.d))
        err = np.abs(got[b] - ref)
        assert (err <= 6 * EPS * S + 1e-38).all(), (key, float(err.max()), float((err / (EPS * S + 1e-38)).max()))


# ---- truncated iterates from a warm start, and the record -------------------------------------------------------------------------

@pytest.mark.parametrize('k', TRUNC_K)
@pytest.mark.parametrize('key', list(BY_NAME))
def test_warm_start_truncated(key, k):
    """Exactly k iterations from a warm start with a nonzero mean whose residual is >= 100x |y'|^2 (a tolerance or a step taken
    from the wrong base, or a dropped c sum(x0), is off by orders of magnitude): iterations, flags, every record field, the iterate
    and the final correction.  k = 1 also pins the right-hand side cell by cell (x1 - x0 = step r0)."""
    case = BY_NAME[key]
    v, x0 = white_problem(case, 71)
    rtol, atol = 1e-6, 1e-7
    v_out, p, rec = run(case, v, x0, rtol, atol, k)
    for b in range(len(SCALES)):
        vb = entry(v, b)
        r64, r32 = check_iterate(case, p[b], vb, x0[b], k, f'entry {b}')
        ref = oracle(case, vb, x0[b], rtol, atol, k, 32)
        assert (ref['iterations'], ref['converged'], ref['diverged']) == (k, False, False), (key, b, ref['iterations'])
        assert (int(rec['iterations'][b]), int(rec['converged'][b]), int(rec['diverged'][b])) == (k, 0, 0), (key, b, rec[b])
        check_record_start(case, rec[b], vb, x0[b], rtol, atol)
        check_residual_sq(case, rec[b], r64, r32)
        check_correction(case, vb, p[b], entry(v_out, b))


@pytest.mark.parametrize('rtol', [1e-3, 1e-5])
@pytest.mark.parametrize('key', CONVERGE)
def test_converged(key, rtol):
    """Converged solves on smooth inputs: iteration counts within max(2, it/10) of the oracle's fp32 run, the float64 true residual of
    the returned p at most 4 tol_sq, the record, and v_out = v - grad(p)."""
    case = BY_NAME[key]
    A64, _, _ = matrices(key)
    v, x0 = smooth_problem(case, 72)
    atol = 1e-7
    v_out, p, rec = run(case, v, x0, rtol, atol, 2000)
    for b in range(len(SCALES)):
        vb = entry(v, b)
        ref = oracle(case, vb, x0[b], rtol, atol, 2000, 32)
        assert ref['converged'] and rec['converged'][b] == 1 and rec['diverged'][b] == 0, (key, b, rec[b], ref['iterations'])
        n_ref = ref['iterations']
        assert abs(int(rec['iterations'][b]) - n_ref) <= max(2, n_ref // 10), (key, b, int(rec['iterations'][b]), n_ref)
        check_record_start(case, rec[b], vb, x0[b], rtol, atol)
        assert rec['residual_sq'][b] <= rec['tol_sq'][b], (key, b, rec[b])
        y = rhs(case, vb, 64).ravel()
        r = y - A64 @ p[b].ravel().astype(F64)
        assert np.sum(r ** 2) <= 4 * max(rtol ** 2 * np.sum(y ** 2), atol ** 2), (key, b, np.sum(r ** 2), rec[b])
        check_correction(case, vb, p[b], entry(v_out, b))


# ---- stops inside the poll window -------------------------------------------------------------------------------------------------

POLL_STOP = 5          # entry 1 stops here: not a multiple of 8, so inside the host's poll window


def poll_problem(case):
    """Entry 0 starts at its own solution (v = grad q, x0 = q), entry 1 (white noise) converges at iteration POLL_STOP under an atol
    chosen from the oracle's residual history, entry 2 (entry 1 x 1e4) keeps running."""
    rng = np.random.default_rng(73)
    q = (0.01 * rng.standard_normal(case.res)).astype(np.float32)
    v0 = O.gradient_centered(q, case.dx, case.pbc)
    v1 = [rng.standard_normal(case.res).astype(np.float32) for _ in range(case.d)]
    x1 = rng.standard_normal(case.res).astype(np.float32)
    v = [np.stack([v0[c], v1[c], v1[c] * np.float32(1e4)]) for c in range(case.d)]
    x0 = np.stack([q, x1, x1 * np.float32(1e4)])
    hist = [oracle(case, v1, x1, 0.0, 0.0, k, 32)['residual_sq'] for k in range(1, POLL_STOP + 1)]
    # converged at POLL_STOP with a margin of more than 2x on either side (fp32 paths that differ in summation order stay on the
    # same side of it)
    assert min(hist[:-1]) > 5 * hist[-1], hist
    atol = float(np.sqrt(np.sqrt(min(hist[:-1]) * hist[-1])))
    return v, x0, atol


@pytest.mark.parametrize('max_iter', [0, 1, 8, 9, 17])
@pytest.mark.parametrize('key', ['const_mix-130x4', 'mixed3-130x4x3'])
def test_poll_window_stops(key, max_iter):
    """An entry that stops at iteration 0, one that stops inside a poll window and one that runs to max_iter share a batch.  Each
    entry equals a batch-1 run of itself bit for bit (iterate, velocity, record) and the oracle at its own stop iteration; max_iter = 0
    returns p = x0 bit for bit with residual_sq = initial_residual_sq and v - grad(x0)."""
    case = BY_NAME[key]
    v, x0, atol = poll_problem(case)
    v_out, p, rec = run(case, v, x0, 0.0, atol, max_iter)
    want_it = [0, min(POLL_STOP, max_iter), max_iter]
    for b in range(3):
        vb = entry(v, b)
        ref = oracle(case, vb, x0[b], 0.0, atol, max_iter, 32)
        assert ref['iterations'] == want_it[b], (key, b, ref['iterations'])
        assert int(rec['iterations'][b]) == want_it[b], (key, b, rec[b])
        assert int(rec['converged'][b]) == int(ref['converged']) and int(rec['diverged'][b]) == 0, (key, b, rec[b])
        ov, op, orec = run(case, [a[b:b + 1] for a in v], x0[b:b + 1], 0.0, atol, max_iter)
        assert np.array_equal(op[0], p[b]) and all(np.array_equal(ov[c][0], v_out[c][b]) for c in range(case.d)), (key, b)
        assert orec.tobytes() == rec[b:b + 1].tobytes(), (key, b, orec, rec[b])
        if want_it[b] == 0:
            assert np.array_equal(p[b], x0[b]), (key, b)
            assert rec['residual_sq'][b] == rec['initial_residual_sq'][b], (key, b, rec[b])
        else:
            r64, r32 = check_iterate(case, p[b], vb, x0[b], want_it[b], f'entry {b}')
            check_residual_sq(case, rec[b], r64, r32)
        check_record_start(case, rec[b], vb, x0[b], 0.0, atol)
        check_correction(case, vb, p[b], entry(v_out, b))


# ---- the divergence rule ------------------------------------------------------------------------------------------------------------

def test_divergence_rule():
    """rsq / rsq0 > 1e5 after >= 8 iterations flags an entry as diverged, through the real entry point (y = the centred divergence of
    white-noise velocities on an open 17 x 12 box, warm start N(0, 1) + 2, rtol = atol = 1e-5): with the oracle, seeds 3, 5, 7
    diverge (at 253, 265, 229 iterations) and 4, 6, 8 converge (73, 70, 67), in fp32 and fp64 alike.  All six share one batch, so
    the diverged entries stop inside poll windows while the others run.  Same flags, iteration counts within 2."""
    case = Case('open', (17, 12))
    seeds = (3, 4, 5, 6, 7, 8)
    vs, xs = [], []
    for s in seeds:
        rng = np.random.default_rng(s)
        vs.append([rng.standard_normal(case.res).astype(np.float32) for _ in range(2)])
        xs.append((rng.standard_normal(case.res) + 2).astype(np.float32))
    v = [np.stack([vb[c] for vb in vs]) for c in range(2)]
    x0 = np.stack(xs)
    with O.precision(64):
        A64 = O.wide_poisson_matrix(case.res, case.dx, case.kinds)
    A32 = A64.astype(np.float32)
    dom = ops.Domain(case.res, case.dx, len(seeds))
    dv = [dom.centered_from_numpy(a) for a in v]
    ops.make_incompressible_centered(dom, case.vbc, dv, dom.centered_from_numpy(x0), rtol=1e-5, atol=1e-5, max_iter=1000)
    rec = ops.read_results(dom)
    flags = []
    for b, s in enumerate(seeds):
        y = O.divergence_centered(vs[b], case.dx, O.component_bcs(case.vbc, 2))
        ref = O.cg_adaptive(A32, y, xs[b], 1e-5, 1e-5, 1000)
        flags.append(ref['diverged'])
        assert (int(rec['converged'][b]), int(rec['diverged'][b])) == (int(ref['converged']), int(ref['diverged'])), (s, rec[b], ref['iterations'])
        assert abs(int(rec['iterations'][b]) - ref['iterations']) <= 2, (s, int(rec['iterations'][b]), ref['iterations'])
    assert flags == [True, False] * 3


# ---- NaN isolation and reproducibility ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('key', ['zero-17x12', 'mixed-257x3', 'zero3-11x9x7', 'inflow3-257x3x2'])
def test_nan_isolation_and_reproducibility(key):
    """A NaN in entry 1 is reported as diverged at iteration 0; entries 0 and 2 are bit for bit those of a run where entry 1 is zero
    (p, v and the record), and the same call twice gives the same bits: every dot product is summed in a fixed order."""
    case = BY_NAME[key]
    v, x0 = white_problem(case, 74)
    v_nan = [a.copy() for a in v]
    v_nan[0][1][tuple(r // 2 for r in case.res)] = np.nan
    v_zero = [a.copy() for a in v]
    for a in v_zero:
        a[1] = 0
    x0_zero = x0.copy()
    x0_zero[1] = 0
    a = run(case, v_nan, x0, 1e-5, 1e-5, 40)
    b = run(case, v_nan, x0, 1e-5, 1e-5, 40)
    z = run(case, v_zero, x0_zero, 1e-5, 1e-5, 40)
    assert (int(a[2]['iterations'][1]), int(a[2]['converged'][1]), int(a[2]['diverged'][1])) == (0, 0, 1), a[2][1]
    assert a[1].tobytes() == b[1].tobytes() and a[2].tobytes() == b[2].tobytes(), key
    assert all(a[0][c].tobytes() == b[0][c].tobytes() for c in range(case.d)), key
    for e in (0, 2):
        assert a[1][e].tobytes() == z[1][e].tobytes(), (key, e)
        assert all(a[0][c][e].tobytes() == z[0][c][e].tobytes() for c in range(case.d)), (key, e)
        assert a[2][e:e + 1].tobytes() == z[2][e:e + 1].tobytes(), (key, e, a[2][e], z[2][e])
        assert int(a[2]['iterations'][e]) > 0, (key, e, a[2][e])


# ---- refusals -----------------------------------------------------------------------------------------------------------------------

def _call(dom, vbc, dv, dp, prm, ws_bytes, ws):
    return _lib.load().phicuda_make_incompressible_centered_host_f32(
        C.byref(dom.grid), C.byref(ops.make_vbc(vbc, dom.dim)), ops._f3(dv, dom.coff), ops._ptr(dp, dom.coff), C.byref(prm),
        ops._ptr(dom.results()), ops._ptr(ws), C.c_size_t(ws_bytes), ops._stream())


def test_refusals():
    """Refused before any CUDA work, with a message, p and v unchanged: plain CG (the operator is not symmetric), z-slabs (halo > 0),
    a workspace one byte short; wide_laplace with x == y."""
    case = BY_NAME['zero3-11x9x7']
    rng = np.random.default_rng(75)
    dom = ops.Domain(case.res, case.dx, 2)
    dv = [dom.centered_from_numpy(rng.standard_normal((2,) + case.res)) for _ in range(3)]
    dp = dom.centered_from_numpy(rng.standard_normal((2,) + case.res))
    before = [t.clone() for t in dv + [dp]]
    ws = ops._collocated_workspace(dom)
    n = ws.numel()
    _, _, c = matrices(repr(case))

    def unchanged():
        torch.cuda.synchronize()
        return all(torch.equal(t, u) for t, u in zip(dv + [dp], before))

    prm = ops.cg_params(case.vbc, matrix_offset=c, method='CG')
    assert _call(dom, case.vbc, dv, dp, prm, n, ws) == _lib.ERR_UNSUPPORTED and 'CG_ADAPTIVE' in _lib.last_error()
    assert unchanged()
    prm = ops.cg_params(case.vbc, matrix_offset=c, method='CG-adaptive')
    assert _call(dom, case.vbc, dv, dp, prm, n - 1, ws) == _lib.ERR_WORKSPACE and 'workspace' in _lib.last_error()
    assert unchanged()
    assert _lib.load().phicuda_wide_laplace_f32(C.byref(dom.grid), C.byref(ops.make_vbc(case.vbc, 3)), ops._ptr(dp), ops._ptr(dp), ops._ptr(ws),
                                                C.c_size_t(n), ops._stream()) == _lib.ERR_INVALID and 'aliased' in _lib.last_error()
    assert unchanged()
    slab = ops.Domain(case.res, case.dx, 1, halo=1)
    sv = [slab.alloc_centered() + 1 for _ in range(3)]
    sp = slab.alloc_centered() + 2
    sbefore = [t.clone() for t in sv + [sp]]
    assert _call(slab, case.vbc, sv, sp, prm, n, ws) == _lib.ERR_UNSUPPORTED and 'z-slabs' in _lib.last_error()
    torch.cuda.synchronize()
    assert all(torch.equal(t, u) for t, u in zip(sv + [sp], sbefore))
