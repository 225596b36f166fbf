"""
The Waves notebook's step restated on the oracle's laplace (oracle/oracle_np.py) - test infrastructure only.

    h_c, h_p = where(disc, value, h_c), where(disc, value, h_p)
    h_n = 2 h_c - h_p + dd (k_speed laplace(h_c) - k_damp (h_c - h_p));  returns (h_n, h_c)

Pinned against PhiML 1.7.2 by tests/golden/phiml_waves.npz (tests/golden/make_waves_golden.py).  The float32 mode rounds every
operation as the reference's float32 field arithmetic does; the float64 mode is the accuracy yardstick (same masks).  As with the
other restated pieces of phi glue (DESIGN.md section 5), the glue is restated on both sides: the cell centres, Sphere.lies_inside,
field.where and field.laplace = math.laplace(values, dx, padding=extrapolation).

WaveOracleEngine is tests/oracle_engine.OracleEngine plus the engine's `wave`, for the host tests of the mirror.
"""
import numpy as np

from oracle_engine import OracleEngine
from oracle_reaction_diffusion import laplace


def disc_mask(axis_centres, centre, radius_sq):
    """Sphere.lies_inside at the cell centres in float32: (p_x - c_x)^2 + (p_y - c_y)^2 [+ (p_z - c_z)^2] <= r^2, summed in axis order.
    axis_centres: one float32 array per axis."""
    grids = np.meshgrid(*axis_centres, indexing='ij')
    s = None
    for g, c in zip(grids, np.asarray(centre, np.float32)):
        t = (g - c) * (g - c)
        s = t if s is None else s + t
    return s <= np.float32(radius_sq)


def split_centres(centres, res):
    """The concatenated per-axis cell centres (x, then y[, z]) as one array per axis."""
    return np.split(np.asarray(centres, np.float32), np.cumsum(res)[:-1])


def wave(h_c, h_p, bc, dx, dd, k_speed, k_damp, masks=None, value=0.0, substeps=1, dtype=np.float32):
    """`substeps` steps of one entry (arrays in (x, y[, z]) order).  masks: None or one boolean mask (or None) per substep; value: the
    stamped value (float32).  dd, k_speed and k_damp enter as float32 numbers in float32 mode.  Returns (h_n, h_c') of the last step."""
    c = dtype
    dd, ks, kd, v = (c(np.float32(p)) for p in (dd, k_speed, k_damp, value))
    h_c, h_p = h_c.astype(c), h_p.astype(c)
    for s in range(substeps):
        m = masks[s] if masks is not None else None
        if m is not None:
            h_c, h_p = np.where(m, v, h_c).astype(c), np.where(m, v, h_p).astype(c)
        h_n = (c(2) * h_c - h_p) + dd * (ks * laplace(h_c, dx, bc, c) - kd * (h_c - h_p))
        h_c, h_p = h_n, h_c
    return h_c, h_p


class WaveOracleEngine(OracleEngine):
    @staticmethod
    def wave(dom, spec, h_c, h_p, dd, k_speed, k_damp, discs, radius_sq, centers, substeps=1):
        axes = split_centres(centers, dom.res)
        hc, hp = dom.centered_to_numpy(h_c, squeeze=False), dom.centered_to_numpy(h_p, squeeze=False)
        outs = []
        for b in range(dom.batch):
            x, y = hc[b], hp[b]
            for d in discs:                  # one substep at a time: each disc has its own value
                m = disc_mask(axes, d[0], radius_sq) if d is not None else None
                x, y = wave(x, y, spec, dom.dx, dd, k_speed, k_damp, [m], d[1] if d is not None else 0.0)
            outs.append((x, y))
        return dom.centered_from_numpy(np.stack([o[0] for o in outs])), dom.centered_from_numpy(np.stack([o[1] for o in outs]))
