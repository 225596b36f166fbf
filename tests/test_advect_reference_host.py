"""
tests/oracle_advect.py (the advection kernels' index-space formulation, float64 sum) against the oracle's world-space
advection (oracle_np, pinned to PhiML), cell by cell at the tolerance of tests/test_gpu_kernels.py and with no exempt cell, so that
the GPU comparisons against oracle_advect (tests/test_gpu_advect_exact.py) inherit the PhiML pin.

The two formulations differ only in the oracle's world-space coordinate rounding, which the tolerance covers.  Where that rounding
puts a world-space lookup on the other side of a cell boundary than the index-space lookup, the floors differ and so may the
MacCormack clamp limits; `test_index_space_floor_matches_world_space` shows that no input here has such a cell.
"""
import numpy as np
import pytest

import oracle_advect as R
from oracle import oracle_np as O
from test_gpu_kernels import ALL_V, SCALAR_EXTRA, _advect_tol, dx_of, rand_staggered

F32 = np.float32
SCALAR_BCS = {'zero': 0.0, 'open': 'zg', 'one': 1.0, 'periodic': 'periodic'}


def scalar_bc(sname, d):
    """Scalar boundary by name; 'const_mix' has a different constant or kind on every side."""
    return SCALAR_EXTRA['const_mix'][:d] + ((0.75, 'zg'),) * (d - 2) if sname == 'const_mix' else O.uniform_bc(d, SCALAR_BCS[sname])


def _cases():
    for vname, vbc in sorted(ALL_V.items()):
        for sname in ['zero', 'open', 'one', 'const_mix', 'periodic']:
            if sname == 'periodic' and vname not in ('periodic', 'periodic3'):
                continue
            yield vname, sname


def _setup(vname, sname, seed=3):
    vbc = ALL_V[vname]
    d = len(vbc)
    res = (37, 22) if d == 2 else (21, 14, 9)
    rng = np.random.default_rng(seed)
    v = [c * F32(1.7) for c in rand_staggered(rng, res, vbc)]
    s = rng.standard_normal(res).astype(F32)
    lower = (0.0,) * d
    upper = tuple(r * h for r, h in zip(res, dx_of(d)))
    return vbc, scalar_bc(sname, d), d, res, lower, upper, v, s


def _world_and_index_floors(s, v, vbc, lower, upper, dx, dt):
    v0 = O._velocity_at_centers(v, s.shape, vbc)
    world = O.to_index_space((O.points_of(lower, upper, s.shape) + v0 * F32(-dt)).astype(F32), lower, upper, s.shape)
    delta = ((F32(-dt) * v0).astype(F32) / np.asarray(dx, F32)).astype(F32)
    return np.floor(world), R.indices(s.shape) + np.floor(delta)


@pytest.mark.parametrize('vname,sname', list(_cases()))
def test_index_space_floor_matches_world_space(vname, sname):
    """The base index of every lookup (-dt for the semi-Lagrangian pass, +dt for MacCormack's backward pass) is the same in both
    formulations; a cell where it is not would be listed here by index."""
    vbc, sbc, d, res, lower, upper, v, s = _setup(vname, sname)
    for dt in (0.8, -0.8):
        world, index = _world_and_index_floors(s, v, vbc, lower, upper, dx_of(d), dt)
        differ = np.argwhere((world != index).any(-1))
        assert differ.size == 0, f"dt={dt}: floors differ at cells {differ.tolist()}"


@pytest.mark.parametrize('vname,sname', list(_cases()))
@pytest.mark.parametrize('dt', [0.8, -0.8])
def test_centered_matches_oracle(vname, sname, dt):
    vbc, sbc, d, res, lower, upper, v, s = _setup(vname, sname)
    tol = _advect_tol(res, [s])
    got, _, _ = R.semi_lagrangian_centered(s, sbc, v, vbc, dx_of(d), dt)
    ref = O.semi_lagrangian_centered(s, sbc, v, vbc, lower, upper, dt)
    np.testing.assert_allclose(got, ref, rtol=0, atol=tol)
    for strength in (0.0, 0.5, 1.0, 2.0):
        got, lo, hi = R.mac_cormack_centered(s, sbc, v, vbc, dx_of(d), dt, strength)
        ref = O.mac_cormack_centered(s, sbc, v, vbc, lower, upper, dt, correction_strength=strength)
        bad = np.argwhere(np.abs(got - ref) > tol)
        assert bad.size == 0, f"strength {strength}: cells {bad.tolist()} differ by more than {tol:.3g}"
        # the oracle's clamp limits (from its world-space lookup) are the index-space ones
        assert np.all(lo <= ref) and np.all(ref <= hi)


FOREIGN = {     # vbc kinds, the field's per-component boundary (same kinds, other constants per component and side)
    'zero': [((0.0, 0.0), (0.5, -1.5)), ((0.25, 0.0), (0.0, 2.0))],
    'mixed': [(('zg', 'zg'), (1.5, 'zg')), (('zg', 'zg'), (-0.75, 'zg'))],
    'per_x_wall_y': [(('periodic', 'periodic'), (0.0, 1.0)), (('periodic', 'periodic'), (-2.0, 0.5))],
    'mixed3': [(('periodic', 'periodic'), (1.5, 'zg'), ('zg', -0.5)), (('periodic', 'periodic'), (0.0, 'zg'), ('zg', 2.0)),
               (('periodic', 'periodic'), (-1.0, 'zg'), ('zg', 0.25))],
    'zero3': [((0.5, -0.5), (0.0, 1.0), (2.0, 0.0)), ((0.0, 0.0), (1.5, 0.0), (0.0, -1.0)), ((0.25, 0.0), (0.0, 0.0), (-2.0, 3.0))],
}


@pytest.mark.parametrize('vname,foreign', [(v, False) for v in sorted(ALL_V)] + [(v, True) for v in sorted(FOREIGN)])
@pytest.mark.parametrize('dt', [0.6, -0.6])
def test_staggered_matches_oracle(vname, foreign, dt):
    """Self-advection, and a foreign field with the velocity's kinds but its own per-component, per-side constants."""
    vbc = ALL_V[vname]
    d = len(vbc)
    res = (37, 22) if d == 2 else (21, 14, 9)
    lower = (0.0,) * d
    upper = tuple(r * h for r, h in zip(res, dx_of(d)))
    rng = np.random.default_rng(4)
    v = [c * F32(1.3) for c in rand_staggered(rng, res, vbc)]
    fbc = FOREIGN[vname] if foreign else vbc
    f = rand_staggered(rng, res, vbc) if foreign else v
    got = R.semi_lagrangian_staggered(f, fbc, v, vbc, res, dx_of(d), dt)
    ref = O.semi_lagrangian_staggered(f, fbc, v, vbc, res, lower, upper, dt)
    tol = _advect_tol(res, f)
    for c in range(d):
        np.testing.assert_allclose(got[c][0], ref[c], rtol=0, atol=tol)


def test_grid_sample_matches_oracle():
    rng = np.random.default_rng(12)
    for bc in (O.uniform_bc(2, 'periodic'), SCALAR_EXTRA['const_mix'], O.uniform_bc(3, 'zg'), ((0.0, 'zg'), ('periodic', 'periodic'), (1.0, -1.0))):
        d = len(bc)
        res = (23, 14) if d == 2 else (13, 9, 7)
        grid = rng.standard_normal(res).astype(F32)
        coords = (rng.uniform(-3, 4, (3000, d)) * np.array(res)).astype(F32)
        coords[:500] = np.round(coords[:500] * 2) / 2
        got, _, _ = R.grid_sample(grid, coords, bc)
        # the oracle's fp32 sum is within the kernels' rounding bound of the float64 one
        tol = R.rounding_units(d) * 0.5 * np.finfo(F32).eps * max(np.abs(grid).max(), 2.0)
        np.testing.assert_allclose(got, O.grid_sample(grid, coords, bc), rtol=0, atol=tol)


EPILOGUE = {    # vbc, sbc, buoyancy, shape of the step-epilogue cases
    # constant x sides of s under zero-gradient x faces (both x boundary faces stored), b_x = 0: those faces get c/2 * dt
    'open-by': ('open', ((-1.0, 0.25), ('zg', 'zg')), (0.0, 0.2), (70, 9)),
    # wall x velocity: the constant lower x side of s is never read by a stored face
    'zero-bx': ('zero', ((0.5, 'zg'), ('zg', 'zg')), (0.3, 0.0), (100, 13)),
    'zero-bxy': ('zero', ((0.5, 'zg'), ('zg', 'zg')), (0.3, -0.2), (100, 13)),
    # periodic x velocity with a constant lower x side of s: face x = 0 reads the ghost, the `xb >= 1` rule of the fast chunks
    'per_x_wall_y-bx': ('per_x_wall_y', ((0.5, 'zg'), (-1.0, 'zg')), (0.3, 0.0), (96, 11)),
    'wall_open3-bxz': ('wall_open3', ((0.5, 'zg'), ('zg', 'zg'), ('zg', 'zg')), (0.15, 0.0, 0.2), (96, 9, 5)),
    'periodic-bxy': ('periodic', (('periodic', 'periodic'), ('zg', 1.5)), (-0.25, 0.1), (96, 11)),
    # constant lower z side of s under a zero-gradient lower z face
    'mixed3-bxyz': ('mixed3', (('periodic', 'periodic'), ('zg', 'zg'), (0.5, 'zg')), (0.2, -0.1, 0.3), (70, 11, 6)),
}


@pytest.mark.parametrize('name', sorted(EPILOGUE))
@pytest.mark.parametrize('mac', [False, True])
def test_step_epilogues_match_oracle_plume_step(name, mac):
    """oracle_np.plume_step with max_iter = 0 and p = 0 returns the pre-projection state: s' = adv(s) + rate * inflow and
    v* = adv(v) + dt * resample(s' * b, to=v).  The same from oracle_advect and buoyancy_faces (which the GPU epilogue tests use)."""
    vname, sbc, buoy, res = EPILOGUE[name]
    vbc = ALL_V[vname]
    d = len(res)
    dx = dx_of(d)
    lower = (0.0,) * d
    upper = tuple(r * h for r, h in zip(res, dx))
    dt, rate = 0.5, 0.2
    rng = np.random.default_rng(35)
    v = [a * F32(2.0) for a in rand_staggered(rng, res, vbc)]
    s = rng.standard_normal(res).astype(F32)
    inflow = np.abs(rng.standard_normal(res)).astype(F32)
    v_ref, s_ref, p_ref, info = O.plume_step(v, s, np.zeros(res, F32), dt, vbc, sbc, lower, upper, res, inflow, rate, buoy,
                                             max_iter=0, smoke_advection='mac_cormack' if mac else 'semi_lagrangian',
                                             use_matrix_offset=False)
    assert info['iterations'] == 0 and not p_ref.any()
    adv = R.mac_cormack_centered if mac else R.semi_lagrangian_centered
    np.testing.assert_allclose(adv(s, sbc, v, vbc, dx, dt)[0] + F32(rate) * inflow, s_ref, rtol=0, atol=_advect_tol(res, [s]))
    bterm = R.buoyancy_faces(s_ref, sbc, vbc, buoy, dt)
    for c, (a, _, _) in enumerate(R.semi_lagrangian_staggered(v, vbc, v, vbc, res, dx, dt)):
        np.testing.assert_allclose(a + bterm[c], v_ref[c], rtol=0, atol=_advect_tol(res, v))
