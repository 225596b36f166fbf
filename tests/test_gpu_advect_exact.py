"""
The advection kernels cell by cell against tests/oracle_advect.py, which restates their index-space lookup exactly and sums in
float64 (tests/test_advect_reference_host.py pins it to the oracle, and so to PhiML).  Every case runs on both kernel families:
the vectorised kernels (csrc/fused_kernels.cu) and the one-thread-per-sample kernels (csrc/advect_kernels.cu,
PHICUDA_SCALAR_KERNELS=1).  grid_sample has one kernel and runs once.

Bound, per cell, in units of u = eps / 2 times M = max |neighbour value| of that cell's lookup (constant ghosts included):
  * semi-Lagrangian: the lookup is exact, so the only error is the fp32 n-linear sum: c = 2d - 1 roundings in a weight, 1 in
    value * weight, 2^d - 1 in the accumulation, +1 for second-order terms -> c = 8 u (2-D), 14 u (3-D) = 4 / 7 eps.
  * MacCormack (M = max over the whole field and its constants; |strength / 2| <= 1): fwd is within c u M; the fp32 fwd the
    kernel stores is within (c + 1) u M of the reference's f32(fwd), so bwd is within (2c + 1) u M; s - bwd, the product with
    strength / 2 and the sum with fwd add 2 + 2 + 3 u M; the clamp limits are stored values, identical on both sides, and the
    clamp does not increase a difference.  Total (3c + 8) u M = 32 u (2-D), 50 u (3-D) = 16 / 25 eps.
  * epilogues (inflow, buoyancy): the sum's bound plus 2 u (|epilogue term| + |result|) for the fused multiply-add and the add.
No cell is exempt, and every output must be finite.

Shapes of section b and the chunks of k_advect_*_vec that take the straight-line path: a warp walks 32-cell chunks
[32 j, 32 j + 32) of its line; with periodic x every chunk whose y / z neighbour lines are stored lines does, otherwise chunk j
needs 32 j >= 1 + lo and 32 j + 32 <= n_x - 1 (stored x range [lo, n_x - 1] shared by the x and y components, lo = 1 for walls):
  n_x = 31, 33, 64: none (every chunk runs the boundary-aware per-sample code);  65: chunk 1;  128: 1, 2;  129: 1, 2, 3;
  200: 1 to 5.  The 128-cell warp segment boundary falls inside the 129- and 200-cell lines.  The staggered kernel also needs
  32 j + 32 <= n_x.  y extents 11, 13, 9, 17 leave the last CTA (8 lines) partly empty.
"""
import os
import time

import numpy as np
import pytest
import torch

import oracle_advect as R
from oracle import oracle_np as O
from test_advect_reference_host import EPILOGUE, FOREIGN, scalar_bc
from test_gpu_kernels import ALL_V, dx_of, rand_staggered

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from phiflow_b200 import _ops as ops
    from phiflow_b200 import flow

EPS = float(np.finfo(np.float32).eps)
U = EPS / 2
F32 = np.float32
FAMILIES = ['vectorised', 'scalar']
WORST = {f: 0.0 for f in FAMILIES}          # largest error / (eps M) seen per family, printed at the end of the module


@pytest.fixture(scope='module', autouse=True)
def _report():
    t0 = time.perf_counter()
    yield
    print(f"\ntest_gpu_advect_exact: largest error / (eps * max|neighbour|): "
          + ", ".join(f"{f} {w:.2f}" for f, w in WORST.items()) + f"; {time.perf_counter() - t0:.1f} s")


class family:
    """Selects the kernel family for the calls inside the block."""

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if self.name == 'scalar':
            os.environ['PHICUDA_SCALAR_KERNELS'] = '1'
        return self

    def __exit__(self, *exc):
        os.environ.pop('PHICUDA_SCALAR_KERNELS', None)


def check(fam, got, ref, scale, units, what, extra_scale=0.0):
    """|got - ref| <= units * u * scale + 2 u * extra_scale in every cell, every value finite.  extra_scale: |epilogue term| +
    |result| of an inflow / buoyancy epilogue (one fused multiply-add and one add)."""
    got = np.asarray(got, np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output at {np.argwhere(~np.isfinite(got))[:5].tolist()}"
    err = np.abs(got - ref)
    bad = np.argwhere(err > units * U * scale + 2 * U * extra_scale)
    denom = EPS * (scale + extra_scale)
    worst = float(np.max(np.where(denom > 0, err / np.where(denom > 0, denom, 1.0), 0.0)))
    WORST[fam] = max(WORST[fam], worst)
    assert bad.size == 0, (f"{what}: {len(bad)} cells beyond the bound ({units} u * max|neighbour|), first {bad[:5].tolist()}, "
                           f"largest error {worst:.1f} eps * max|neighbour|")


def scale_of(lo, hi):
    return np.maximum(np.abs(lo), np.abs(hi))


def mc_units(d):
    return 3 * R.rounding_units(d) + 8


def field_scale(a, bc):
    consts = [abs(s) for ax in O.kinds_of(bc) for s in ax if O.is_const(s)] if not isinstance(bc, list) else \
        [abs(s) for spec in bc for ax in spec for s in ax if O.is_const(s)]
    return max([float(np.abs(a).max())] + consts)


# ---- a. centred semi-Lagrangian and MacCormack: boundaries x strengths x dt signs x displacement regimes ----------------------
def velocity(rng, res, vbc, dt, regime):
    """Staggered velocity whose displacements -dt v / dx are in `regime` (cells)."""
    d = len(res)
    shapes = O.staggered_shapes(res, vbc)
    dx = dx_of(d)
    out = []
    for c, shp in enumerate(shapes):
        cell = dx[c] / abs(dt)                                       # velocity of one cell per step along axis c
        if regime == 'sub_cell':
            a = 0.4 * rng.standard_normal(shp)
        elif regime == 'cells_3_6':
            a = rng.choice([-1.0, 1.0], shp) * rng.uniform(3.0, 6.0, shp)
        elif regime == 'beyond_extent':                             # several periodic wraps, far past constant sides
            a = rng.choice([-1.0, 1.0], shp) * rng.uniform(2.0, 3.5, shp) * res[c]
        else:                                                        # 'integer': multiples of 4 cells -> integral averages
            a = 4.0 * rng.integers(-3, 4, shp)
        out.append((a * cell).astype(F32))
    return out


REGIMES = ['sub_cell', 'cells_3_6', 'beyond_extent', 'integer']


def _centered_cases():
    for vname in sorted(ALL_V):
        for sname in ['zero', 'open', 'one', 'const_mix', 'periodic']:
            if sname == 'periodic' and vname not in ('periodic', 'periodic3'):
                continue
            yield vname, sname


@pytest.mark.parametrize('fam', FAMILIES)
@pytest.mark.parametrize('vname,sname', list(_centered_cases()))
def test_centered(vname, sname, fam):
    vbc = ALL_V[vname]
    d = len(vbc)
    sbc = scalar_bc(sname, d)
    res = (37, 22) if d == 2 else (21, 14, 9)
    dx = dx_of(d)
    rng = np.random.default_rng(31)
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    s = rng.standard_normal(res).astype(F32)
    ds = dom.centered_from_numpy(s)
    M = field_scale(s, sbc)
    for regime in REGIMES:
        for dt in (0.5, -0.5):
            v = velocity(rng, res, vbc, dt, regime)
            if regime == 'integer':
                delta = (F32(-dt) * O._velocity_at_centers(v, res, vbc)).astype(F32) / np.asarray(dx, F32)
                assert np.all(delta == np.floor(delta)) and np.any(delta != 0)
            dv = dom.faces_from_numpy(v, vbc)
            what = f"{regime} dt={dt}"
            with family(fam):
                got = dom.centered_to_numpy(ops.advect_centered(dom, vbc, dv, sbc, ds, dt))
            ref, lo, hi = R.semi_lagrangian_centered(s, sbc, v, vbc, dx, dt)
            check(fam, got, ref, scale_of(lo, hi), R.rounding_units(d), 'semi-Lagrangian ' + what)
            for strength in (0.0, 0.5, 1.0, 2.0):
                with family(fam):
                    got = dom.centered_to_numpy(ops.mac_cormack_centered(dom, vbc, dv, sbc, ds, dt, correction_strength=strength))
                ref, lo, hi = R.mac_cormack_centered(s, sbc, v, vbc, dx, dt, strength)
                check(fam, got, ref, M, mc_units(d), f"MacCormack strength {strength} " + what)
                assert np.all(lo <= got) and np.all(got <= hi), "outside the clamp limits"


# ---- b. shapes across the chunk / segment / CTA decomposition, batch 3 -------------------------------------------------------
SHAPES = [((n, 11 if n % 2 else 13), vname) for n in (31, 33, 64, 65, 128, 129, 200) for vname in ('zero', 'open', 'per_x_wall_y')] \
    + [(res, vname) for res in ((65, 9, 5), (129, 17, 3)) for vname in ('zero3', 'open3', 'periodic3', 'wall_open3')]


@pytest.mark.parametrize('fam', FAMILIES)
@pytest.mark.parametrize('res,vname', SHAPES, ids=[f"{'x'.join(map(str, r))}-{v}" for r, v in SHAPES])
def test_shapes(res, vname, fam):
    vbc = ALL_V[vname]
    d = len(res)
    dx = dx_of(d)
    batch, dt = 3, 0.5
    sbc = scalar_bc('const_mix', d)
    rng = np.random.default_rng(32)
    dom = ops.Domain(res, dx, batch, vbc=vbc)
    # every entry its own velocity (about 3 cells per step) and field
    v = [a * F32(3.0 * dx[c] / dt) for c, a in enumerate(rand_staggered(rng, res, vbc, batch))]
    s = rng.standard_normal((batch,) + res).astype(F32)
    dv, ds = dom.faces_from_numpy(v, vbc), dom.centered_from_numpy(s)
    with family(fam):
        sl = dom.centered_to_numpy(ops.advect_centered(dom, vbc, dv, sbc, ds, dt), squeeze=False)
        mc = dom.centered_to_numpy(ops.mac_cormack_centered(dom, vbc, dv, sbc, ds, dt), squeeze=False)
        st = dom.faces_to_numpy(ops.advect_staggered(dom, vbc, dv, vbc, dv, dt), vbc, squeeze=False)
    for b in range(batch):
        vb = [c[b] for c in v]
        ref, lo, hi = R.semi_lagrangian_centered(s[b], sbc, vb, vbc, dx, dt)
        check(fam, sl[b], ref, scale_of(lo, hi), R.rounding_units(d), f"semi-Lagrangian entry {b}")
        ref, _, _ = R.mac_cormack_centered(s[b], sbc, vb, vbc, dx, dt)
        check(fam, mc[b], ref, field_scale(s[b], sbc), mc_units(d), f"MacCormack entry {b}")
        for c, (ref, lo, hi) in enumerate(R.semi_lagrangian_staggered(vb, vbc, vb, vbc, res, dx, dt)):
            check(fam, st[c][b], ref, scale_of(lo, hi), R.rounding_units(d), f"staggered component {c} entry {b}")


# ---- c. staggered advection of a foreign field ---------------------------------------------------------------------------------
@pytest.mark.parametrize('fam', FAMILIES)
@pytest.mark.parametrize('vname', sorted(FOREIGN))
def test_staggered_foreign_field(vname, fam):
    """The field keeps the velocity's kinds with its own per-component, per-side constants (the Variable_Boundaries form); x extents
    past 65 so that both the straight-line chunks and the boundary chunks of k_advect_staggered_vec run."""
    vbc, fbc = ALL_V[vname], FOREIGN[vname]
    d = len(vbc)
    res = (100, 13) if d == 2 else (70, 11, 6)
    dx = dx_of(d)
    rng = np.random.default_rng(33)
    dom = ops.Domain(res, dx, 2, vbc=vbc)
    for dt in (0.5, -0.5):
        v = [a * F32(2.5) for a in rand_staggered(rng, res, vbc, 2)]
        f = [a * F32(3.0) for a in rand_staggered(rng, res, vbc, 2)]
        dv, df = dom.faces_from_numpy(v, vbc), dom.faces_from_numpy(f, fbc)
        with family(fam):
            got = dom.faces_to_numpy(ops.advect_staggered(dom, vbc, dv, fbc, df, dt), fbc, squeeze=False)
        for b in range(2):
            refs = R.semi_lagrangian_staggered([a[b] for a in f], fbc, [a[b] for a in v], vbc, res, dx, dt)
            for c, (ref, lo, hi) in enumerate(refs):
                check(fam, got[c][b], ref, scale_of(lo, hi), R.rounding_units(d), f"dt={dt} entry {b} component {c}")


@pytest.mark.parametrize('fam', FAMILIES)
def test_flow_semi_lagrangian_of_staggered_field(fam):
    """flow.advect.semi_lagrangian sends a StaggeredGrid that is not the velocity to the staggered kernel."""
    res = (70, 13)
    rng = np.random.default_rng(34)
    vbc = ALL_V['zero']
    v = [a * F32(2.0) for a in rand_staggered(rng, res, vbc)]
    vel = flow.StaggeredGrid(v, flow.ZERO, x=res[0], y=res[1])
    boundary = {'x': 0, 'y-': flow.vec(x=0.5, y=-1.0), 'y+': flow.vec(x=1.0, y=2.0)}
    f = rand_staggered(rng, res, vbc)
    fld = flow.StaggeredGrid(f, boundary, x=res[0], y=res[1])
    assert isinstance(fld.vspec, list)
    with family(fam):
        got = flow.advect.semi_lagrangian(fld, vel, 0.7).numpy()
    for c, (ref, lo, hi) in enumerate(R.semi_lagrangian_staggered(f, fld.vspec, v, vbc, res, (1.0, 1.0), 0.7)):
        check(fam, got[c], ref, scale_of(lo, hi), R.rounding_units(2), f"component {c}")


# ---- d. the step's epilogues, observed exactly: plume_step with max_iter = 0 and p = 0 ---------------------------------------
def _no_iteration(vbc):
    """At max_iter = 0 the CG returns x0 = 0 bit for bit and the gradient of 0 subtracts exactly 0: the velocity after the step
    is the pre-projection v*."""
    prm = ops.cg_params(vbc, rtol=1e-5, atol=1e-5, max_iter=0)
    prm.project_mean = 0
    return prm




@pytest.mark.parametrize('fam', FAMILIES)
@pytest.mark.parametrize('mac', [False, True])
@pytest.mark.parametrize('name', sorted(EPILOGUE))
def test_plume_step_epilogues(name, mac, fam):
    """s' = adv(s) + rate * inflow and v* = adv(v) + dt * resample(s' * b, to=v), for both smoke advections."""
    vname, sbc, buoy, res = EPILOGUE[name]
    vbc = ALL_V[vname]
    d = len(res)
    dx = dx_of(d)
    dt, rate = 0.5, 0.2
    rng = np.random.default_rng(35)
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    v = [a * F32(2.0) for a in rand_staggered(rng, res, vbc)]
    s = rng.standard_normal(res).astype(F32)
    inflow = np.abs(rng.standard_normal(res)).astype(F32)
    dv, ds, dp, dinf = dom.faces_from_numpy(v, vbc), dom.centered_from_numpy(s), dom.alloc_centered(), dom.centered_from_numpy(inflow)
    with family(fam):
        ops.plume_step(dom, vbc, sbc, dv, ds, dp, dinf, dt, rate, buoy, _no_iteration(vbc), mac_cormack=mac)
    assert ops.read_results(dom)['iterations'][0] == 0
    assert not dp.any()
    got_s = dom.centered_to_numpy(ds)
    add = F32(rate) * inflow.astype(np.float64)
    if mac:
        ref, _, _ = R.mac_cormack_centered(s, sbc, v, vbc, dx, dt)
        scale, units = field_scale(s, sbc), mc_units(d)
    else:
        ref, lo, hi = R.semi_lagrangian_centered(s, sbc, v, vbc, dx, dt)
        scale, units = scale_of(lo, hi), R.rounding_units(d)
    ref = ref + add
    check(fam, got_s, ref, scale, units, "smoke + inflow", extra_scale=(np.abs(add) + np.abs(ref)))
    got_v = dom.faces_to_numpy(dv, vbc)
    bterm = R.buoyancy_faces(got_s, sbc, vbc, buoy, dt)
    for c, (ref, lo, hi) in enumerate(R.semi_lagrangian_staggered(v, vbc, v, vbc, res, dx, dt)):
        ref = ref + bterm[c]
        check(fam, got_v[c], ref, scale_of(lo, hi), R.rounding_units(d), f"velocity + buoyancy, component {c}",
              extra_scale=(np.abs(bterm[c]) + np.abs(ref)))


# ---- e. the forced step (static_scalar) ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fam', FAMILIES)
@pytest.mark.parametrize('vname,buoy', [('periodic', (1.0, 0.0)), ('zero', (0.3, -0.2)), ('mixed3', (0.2, -0.1, 0.3))])
def test_forced_step_epilogue(vname, buoy, fam):
    """v* = adv(v) + dt * resample(s * b, to=v) with s bit for bit unchanged (the scalar family runs the unfused sequence)."""
    vbc = ALL_V[vname]
    d = len(vbc)
    res = (96, 13) if d == 2 else (70, 11, 6)
    dx = dx_of(d)
    dt = 0.5
    sbc = (('periodic', 'periodic'),) * d if vname == 'periodic' else ((0.5, 'zg'),) + (('zg', 'zg'),) * (d - 1)
    rng = np.random.default_rng(36)
    dom = ops.Domain(res, dx, 1, vbc=vbc)
    v = [a * F32(2.0) for a in rand_staggered(rng, res, vbc)]
    s = rng.standard_normal(res).astype(F32)
    dv, ds, dp = dom.faces_from_numpy(v, vbc), dom.centered_from_numpy(s), dom.alloc_centered()
    s_before = ds.clone()
    with family(fam):
        ops.plume_step(dom, vbc, sbc, dv, ds, dp, None, dt, 0.0, buoy, _no_iteration(vbc), static_scalar=True)
    assert torch.equal(ds, s_before)
    got_v = dom.faces_to_numpy(dv, vbc)
    bterm = R.buoyancy_faces(s, sbc, vbc, buoy, dt)
    for c, (ref, lo, hi) in enumerate(R.semi_lagrangian_staggered(v, vbc, v, vbc, res, dx, dt)):
        ref = ref + bterm[c]
        check(fam, got_v[c], ref, scale_of(lo, hi), R.rounding_units(d), f"component {c}",
              extra_scale=(np.abs(bterm[c]) + np.abs(ref)))


@pytest.mark.parametrize('fam', FAMILIES)
def test_forced_step_c5_against_oracle(fam):
    """The c5 configuration (8 x 32^2, periodic, forcing sin 4y along x) for 3 full steps of plume_step(static_scalar=True) against
    the oracle, as test_gpu_kernels.test_config_c5_kolmogorov_batched_2d checks the unfused sequence."""
    n, batch = 32, 8
    res = (n, n)
    L = 2 * np.pi
    dx = (L / n, L / n)
    lower, upper = (0.0, 0.0), (L, L)
    vbc = O.uniform_bc(2, 'periodic')
    yc = (np.arange(n) + 0.5) * dx[1]
    forcing = np.broadcast_to(np.sin(4 * yc)[None, :], res).astype(F32)
    v0 = [np.stack([(0.01 * np.random.default_rng(100 + b).standard_normal(res)).astype(F32) for b in range(batch)]) for _ in range(2)]
    dom = ops.Domain(res, dx, batch, vbc=vbc)
    dv, dforce, dp = dom.faces_from_numpy(v0, vbc), dom.centered_from_numpy(forcing), dom.alloc_centered()
    prm = ops.cg_params(vbc, rtol=1e-4, atol=1e-6)
    dt = 0.05
    A = O.poisson_matrix(res, dx, O.pressure_bc(vbc))
    v = [[v0[0][b], v0[1][b]] for b in range(batch)]
    p = [np.zeros(res, F32) for _ in range(batch)]
    faces = O.centered_to_faces(forcing * F32(1.0), vbc, vbc)
    for _ in range(3):
        with family(fam):
            ops.plume_step(dom, vbc, vbc, dv, dforce, dp, None, dt, 0.0, (1.0, 0.0), prm, static_scalar=True)
        assert ops.read_results(dom)['converged'].all()
        for b in range(batch):
            vb = O.semi_lagrangian_staggered(v[b], vbc, v[b], vbc, res, lower, upper, dt)
            vb = [vb[0] + faces[0] * F32(dt), vb[1]]
            v[b], p[b], _ = O.make_incompressible(vb, vbc, res, dx, rtol=1e-4, atol=1e-6, x0=p[b], use_matrix_offset=False, matrix=A)
    got = dom.faces_to_numpy(dv, vbc, squeeze=False)
    for b in range(batch):
        for c in range(2):
            np.testing.assert_allclose(got[c][b], v[b][c], rtol=0, atol=5e-5)
    assert (dom.centered_to_numpy(dforce, squeeze=False) == forcing).all()


# ---- f. grid_sample --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bc', [O.uniform_bc(2, 'periodic'), scalar_bc('const_mix', 2), O.uniform_bc(2, 'zg'), O.uniform_bc(3, 1.0),
                                scalar_bc('const_mix', 3), (('periodic', 'periodic'), (0.0, 'zg'), ('zg', -1.0))],
                         ids=['periodic', 'const_mix', 'zg', 'one3', 'const_mix3', 'mixed3'])
def test_grid_sample(bc):
    """Integer and half-integer coordinates, points inside and up to three extents outside on every side."""
    d = len(bc)
    res = (23, 14) if d == 2 else (13, 9, 7)
    batch, npts = 2, 6000
    rng = np.random.default_rng(37)
    dom = ops.Domain(res, (1.0,) * d, batch)
    grid = rng.standard_normal((batch,) + res).astype(F32)
    coords = (rng.uniform(-3.0, 4.0, (batch, npts, d)) * np.array(res)).astype(F32)
    coords[:, :1000] = np.round(coords[:, :1000])
    coords[:, 1000:2000] = np.round(coords[:, 1000:2000]) + F32(0.5)
    out = ops.grid_sample(dom, bc, dom.centered_from_numpy(grid), torch.from_numpy(coords).cuda()).cpu().numpy()
    for b in range(batch):
        ref, lo, hi = R.grid_sample(grid[b], coords[b], bc)
        check('vectorised', out[b], ref, scale_of(lo, hi), R.rounding_units(d), f"entry {b}")
