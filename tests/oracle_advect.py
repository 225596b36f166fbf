"""
The advection kernels' formulation (csrc/advect_kernels.cu, csrc/fused_kernels.cu) restated in index space with a float64
interpolation sum - test infrastructure only, like tests/oracle_diffuse.py.

The oracle (oracle_np.semi_lagrangian_centered / semi_lagrangian_staggered / mac_cormack_centered, pinned to PhiML) traces back
in world space: point - dt v, then Box.global_to_local * resolution - 0.5.  The kernels keep (sample index, displacement in
cells) instead, and so does this file:
    v      the velocity at the sample point: the oracle's own fp32 shift resampling (_velocity_at_centers / _velocity_at_faces,
           the same fp32 operations in the same order as phi_velocity_at / fk_avg4)
    delta  f32(f32(-dt) * v) / f32(dx), correctly rounded in fp32 like phi_div
    base   i + floor(delta), frac = delta - floor(delta)               (fp32, exact)
    values oracle_np.closest_grid_values(field, base, bc): wrap, clamp, constants and corner order exactly as in the oracle
    result the weighted sum over the 2^d neighbours, weights prod(frac or 1 - frac), in float64
The lookup is the kernels' lookup bit for bit; what is left between a kernel and this file is the kernel's fp32 weights and sum.
tests/test_advect_reference_host.py pins this file to the oracle cell by cell.

Every sampler returns (value, lo, hi): the float64 result and the min / max of the 2^d neighbour values per sample point
(MacCormack's clamp limits; max(|lo|, |hi|) is the scale of the fp32 rounding bound).
"""
import itertools

import numpy as np

from oracle import oracle_np as O

F32 = np.float32


def indices(shape):
    """Index of every sample point, shape + (d,), fp32 (integers below 2^24 are exact)."""
    return np.stack(np.meshgrid(*[np.arange(n) for n in shape], indexing='ij'), -1).astype(F32)


def interpolate(field, bc, base, frac):
    """n-linear interpolation of `field` (boundary spec `bc`) at index base + frac, base integral, 0 <= frac < 1."""
    d = base.shape[-1]
    nb = O.closest_grid_values(np.asarray(field, F32), base.astype(F32), bc).astype(np.float64)
    t = np.asarray(frac, F32).astype(np.float64)
    out = np.zeros(base.shape[:-1])
    for corner in itertools.product((0, 1), repeat=d):
        w = np.ones(base.shape[:-1])
        for a in range(d):
            w = w * (t[..., a] if corner[a] else 1.0 - t[..., a])
        out += w * nb[(Ellipsis,) + corner]
    flat = nb.reshape(nb.shape[:-d] + (-1,))
    return out, flat.min(-1), flat.max(-1)


def sample_at(field, bc, v, dt, dx):
    """`field` at its own sample points displaced by -dt v; v: the velocity at those points, field.shape + (d,), fp32."""
    delta = ((F32(-dt) * np.asarray(v, F32)).astype(F32) / np.asarray(dx, F32)).astype(F32)
    fl = np.floor(delta)
    return interpolate(field, bc, indices(np.shape(field)) + fl, (delta - fl).astype(F32))


def semi_lagrangian_centered(s, sbc, v, vbc, dx, dt):
    return sample_at(s, sbc, O._velocity_at_centers(v, np.shape(s), vbc), dt, dx)


def mac_cormack_centered(s, sbc, v, vbc, dx, dt, correction_strength=1.0):
    """fwd = semi-Lagrangian; bwd = fwd rounded to fp32 (as the kernel stores it) sampled at +dt;
    new = fwd + strength * 0.5 * (s - bwd), clamped to the min / max of the 2^d neighbours of the -dt lookup."""
    v0 = O._velocity_at_centers(v, np.shape(s), vbc)
    fwd, lo, hi = sample_at(s, sbc, v0, dt, dx)
    bwd, _, _ = sample_at(fwd.astype(F32), sbc, v0, -dt, dx)
    half = float(F32(correction_strength) * F32(0.5))
    return np.clip(fwd + half * (np.asarray(s, np.float64) - bwd), lo, hi), lo, hi


def semi_lagrangian_staggered(f, fbc, v, vbc, res, dx, dt):
    """Per component c of `f`: its stored faces (in the oracle's compact component index) displaced by -dt v(face), interpolated
    with the component's own boundary (fbc: one spec, or a list of per-component specs with vector-valued constants)."""
    d = len(res)
    fbcs = O.component_bcs(fbc, d)
    return [sample_at(f[c], fbcs[c], O._velocity_at_faces(v, res, vbc, c, fbc), dt, dx) for c in range(d)]


def buoyancy_faces(s, sbc, vbc, b, dt):
    """dt * resample(s * b, to=faces) as oracle_np.plume_step computes it, in the kernels' fp32 operations:
    ((s b_c)[upper] * 0.5 + (s b_c)[lower] * 0.5) * dt.  The product keeps the boundary of s (phi/field/_field.py:809), so a
    constant side c of s enters unscaled, also for b_c = 0."""
    faces = [O.centered_to_faces(np.asarray(s, F32) * F32(bc), sbc, vbc)[c] for c, bc in enumerate(b)]
    return [(a * F32(dt)).astype(F32) for a in faces]


def grid_sample(grid, coords, bc):
    """math.grid_sample at fp32 index-space coordinates, frac = c - floor(c) as k_grid_sample computes it."""
    c = np.asarray(coords, F32)
    fl = np.floor(c)
    return interpolate(grid, bc, fl, (c - fl).astype(F32))


def rounding_units(d):
    """Bound on the error of the kernels' fp32 n-linear sum, in units of u = eps / 2 times max |neighbour value|: 2d - 1 roundings
    in a weight (1 - t per axis, d - 1 products), 1 in value * weight, 2^d - 1 in the accumulation, plus 1 for the second-order
    terms.  7 + 1 in 2-D, 13 + 1 in 3-D."""
    return 2 * d + 2 ** d
