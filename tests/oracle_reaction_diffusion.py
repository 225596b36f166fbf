"""
The Reaction_Diffusion notebook's Gray-Scott step restated on the oracle's laplace (oracle/oracle_np.py) - test infrastructure only.

    uvv = u * v**2;  su = du * laplace(u) - uvv + f * (1 - u);  sv = dv * laplace(v) + uvv - (f + k) * v;  u + dt su, v + dt sv

Pinned against PhiML 1.7.2 by tests/golden/phiml_reaction_diffusion.npz (tests/golden/make_reaction_diffusion_golden.py).  The
float32 mode rounds every operation as the reference's float32 field arithmetic does; the float64 mode is the accuracy yardstick.
As with the other restated pieces of phi glue (DESIGN.md section 5), the glue is restated on both sides: here field.laplace =
math.laplace(values, dx, padding=extrapolation) and the step's arithmetic on plain arrays.

ReactionDiffusionOracleEngine is tests/oracle_engine.OracleEngine plus the engine's reaction_diffusion, for the host tests of the mirror.
"""
import numpy as np

from oracle import oracle_np as O
from oracle_engine import OracleEngine


def laplace(x, dx, bc, dtype=np.float32):
    """oracle_np.laplace in float32; the same sum in float64 for dtype=np.float64."""
    if dtype == np.float32:
        return O.laplace(x, dx, bc)
    x = x.astype(np.float64)
    result = None
    for axis in range(x.ndim):
        p = O.pad_axis(x, axis, 1, 1, bc[axis])
        n = x.shape[axis]
        term = (np.take(p, np.arange(0, n), axis=axis) + np.take(p, np.arange(2, n + 2), axis=axis) - 2.0 * x) / (float(dx[axis]) ** 2)
        result = term if result is None else result + term
    return result


def reaction_diffusion(u, v, bc, dx, du, dv, f, k, dt, substeps=1, dtype=np.float32):
    """`substeps` steps of one entry (arrays in (x, y[, z]) order).  The parameters enter as float32 numbers in float32 mode, and
    f + k is formed in float32 (as the library forms it)."""
    c = dtype
    du, dv, f, k, dt = (c(p) for p in (du, dv, f, k, dt))
    fk = c(f + k)
    u, v = u.astype(c), v.astype(c)
    for _ in range(substeps):
        uvv = u * (v * v)
        su = du * laplace(u, dx, bc, c) - uvv + f * (c(1) - u)
        sv = dv * laplace(v, dx, bc, c) + uvv - fk * v
        u, v = u + dt * su, v + dt * sv
    return u, v


class ReactionDiffusionOracleEngine(OracleEngine):
    @staticmethod
    def reaction_diffusion(dom, spec, u, v, du, dv, f, k, dt, substeps=1):
        specs = spec if isinstance(spec, list) else [spec, spec]
        assert specs[0] == specs[1] or all(not isinstance(s, str) for ax in specs[0] for s in ax), "one boundary for u and v"
        un, vn = dom.centered_to_numpy(u, squeeze=False), dom.centered_to_numpy(v, squeeze=False)
        outs = [reaction_diffusion(un[b], vn[b], specs[0], dom.dx, du, dv, f, k, dt, substeps) for b in range(dom.batch)]
        return dom.centered_from_numpy(np.stack([o[0] for o in outs])), dom.centered_from_numpy(np.stack([o[1] for o in outs]))
