"""
NumPy restatement of k_advect_points (phiflow_b200/csrc/points_kernels.cu, DESIGN.md row N11): advect.points through a StaggeredGrid
velocity with Euler or RK4, operation for operation in float32 (every NumPy float32 operation below is one correctly rounded
operation, as each of the kernel's intrinsics is).  The index rule is the kernel's, not PhiML's: non-periodic indices are clamped to
[-2, N] before they are resolved, periodic ones reduced mod n, NaN / inf / |x| >= 2^31 converted to INT_MIN.  Reproducing PhiML's
positions (tests/golden/phiml_points.npz) with it checks the argument in the kernel's comment.

A velocity is a list over components c of (values (B, *stored shape) in (x, y[, z]) order, spec_c = ((lo, hi) per axis) with sides
'periodic', 'zg' or a float, lower_c, size_c, res_c (per axis, float32)).
"""
import numpy as np

F = np.float32
INT_MIN = np.int64(-2 ** 31)


def to_int32(x: np.ndarray) -> np.ndarray:
    """NumPy's float32 -> int32 cast on x86 for integral x: the value for |x| < 2^31, INT_MIN otherwise (NaN and +-inf included)."""
    ok = (x >= F(-2.0 ** 31)) & (x < F(2.0 ** 31))
    return np.where(ok, np.where(ok, x, 0).astype(np.int64), INT_MIN)


def _axis_resolve(i, lo, hi, side_lo, side_hi):
    """phi_resolve on one axis: (index into the stored array, is constant, constant); i int64 within [lo - 3, hi + 2]."""
    n = hi - lo + 1
    idx = i.copy()
    const = np.zeros(i.shape, F)
    is_const = np.zeros(i.shape, bool)
    below, above = i < lo, i > hi
    if side_lo == 'periodic':
        idx = np.where(below | above, lo + np.mod(i - lo, n), idx)
        return idx, is_const, const
    if side_lo == 'zg':
        idx = np.where(below, lo, idx)
    else:
        is_const |= below
        const = np.where(below, F(side_lo), const)
    if side_hi == 'zg':
        idx = np.where(above, hi, idx)
    else:
        is_const |= above
        const = np.where(above, F(side_hi), const)
    return idx, is_const, const


def _fetch(values, b, idx_res, d):
    """phi_fetch: the last axis is resolved first, so the constant of the LAST out-of-range axis in the order z, y, x wins."""
    out = None
    done = np.zeros(b.shape, bool)
    for a in reversed(range(d)):
        _, is_c, c = idx_res[a]
        take = is_c & ~done
        out = np.where(take, c, out if out is not None else F(0))
        done |= is_c
    safe = tuple(np.where(done, 0, idx_res[a][0]) for a in range(d))
    stored = values[(b,) + safe]
    return np.where(done, out, stored).astype(F)


def sample(vel, b, p):
    """Velocity at p (M, d) of batch entries b (M,): (M, d) float32."""
    d = p.shape[-1]
    v = np.empty(p.shape, F)
    for c, (values, spec, lower, size, res) in enumerate(vel):
        shape = values.shape[1:]
        i0, t = [], []
        for a in range(d):
            idx = (((p[:, a] - F(lower[a])) / F(size[a])) * F(res[a]) - F(0.5)).astype(F)
            with np.errstate(invalid='ignore'):
                t.append((idx - np.floor(idx)).astype(F))
            side_lo, side_hi = spec[a]
            n = shape[a]
            if side_lo == 'periodic':
                i0.append(np.mod(to_int32(np.floor(idx)), n))
            else:
                s = 0 if isinstance(side_lo, str) else 1
                N = n + s + (0 if isinstance(side_hi, str) else 1)
                k = np.clip(to_int32(np.floor((idx + F(s)).astype(F))), -2, N)
                i0.append(k - s)
        vals = []
        for corner in np.ndindex(*(2,) * d):
            res_ax = [_axis_resolve(i0[a] + corner[a], 0, shape[a] - 1, *spec[a]) for a in range(d)]
            vals.append(_fetch(values, b, res_ax, d))
        u = [(F(1) - ta).astype(F) for ta in t]
        r = []
        for k, corner in enumerate(np.ndindex(*(2,) * d)):
            w = t[0] if corner[0] else u[0]
            for a in range(1, d):
                w = (w * (t[a] if corner[a] else u[a])).astype(F)
            r.append((vals[k] * w).astype(F))
        if d == 2:
            v[:, c] = (((r[0] + r[1]).astype(F) + r[2]).astype(F) + r[3]).astype(F)
        else:
            v[:, c] = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    return v


def step(vel, b, p, dt, integrator):
    dt = F(dt)
    with np.errstate(invalid='ignore', over='ignore'):
        v0 = sample(vel, b, p)
        if integrator == 'euler':
            return (p + v0 * dt).astype(F)
        h = F(0.5) * dt
        vh = sample(vel, b, (p + h * v0).astype(F))
        vh2 = sample(vel, b, (p + h * vh).astype(F))
        v1 = sample(vel, b, (p + dt * vh2).astype(F))
        acc = (v0 + F(2) * (vh + vh2)).astype(F)
        return (p + dt * (F(1 / 6.) * (acc + v1))).astype(F)


def advect_points(vel, points, dt, integrator, steps, trajectory=False):
    """points (Bp, N, d); the velocity's batch Bv; returns (B, N, d) (and the (steps + 1, B, N, d) trajectory)."""
    Bv = vel[0][0].shape[0]
    Bp, N, d = points.shape
    B = max(Bv, Bp)
    p = np.broadcast_to(points, (B, N, d)).reshape(-1, d).astype(F)
    b = np.repeat(np.arange(B) if Bv > 1 else np.zeros(B, int), N)
    trj = [p.reshape(B, N, d)]
    for _ in range(steps):
        p = step(vel, b, p, dt, integrator)
        trj.append(p.reshape(B, N, d))
    out = p.reshape(B, N, d)
    return (out, np.stack(trj)) if trajectory else out
