"""
The notebook step with static obstacles on the oracle (test infrastructure; the product never imports this file): oracle_np.plume_step
for the smoke and the pre-projection velocity v* (run with max_iter = 0 from p = 0, where its projection returns v* unchanged), v* times
the obstacle face factors (apply_boundary_conditions, phi/physics/fluid.py:212-240), then the obstacle projection of
tests/oracle_masked.py with the solver the step asks for.  ObstacleStepEngine is the oracle-backed engine of tests/oracle_engine.py
whose plume_step takes the masks, as phiflow_b200._ops.plume_step does.
"""
import numpy as np

from oracle import oracle_np as O
from oracle_masked import MaskedMethodEngine, make_incompressible_obstacles

F32 = np.float32


def pre_projection(v, s, dt, vbc, sbc, lower, upper, res, inflow, inflow_rate, buoyancy, smoke_advection='semi_lagrangian'):
    """(v* before the face factors, s') of one step, both as oracle_np.plume_step computes them."""
    zero = np.zeros(res, F32)
    v_b, s_new, p0, info = O.plume_step(v, s, zero, dt, vbc, sbc, lower, upper, res, inflow, inflow_rate, buoyancy, max_iter=0,
                                        use_matrix_offset=False, smoke_advection=smoke_advection)
    assert info['iterations'] == 0 and not p0.any()
    return v_b, s_new


def step(v, s, p, dt, vbc, sbc, lower, upper, res, inflow, inflow_rate, buoyancy, accessible, factors, rtol, atol, max_iter,
         method='CG', smoke_advection='semi_lagrangian'):
    """One step with obstacles.  Returns (v*, v', s', p', info); v* = the velocity the projection starts from."""
    v_b, s_new = pre_projection(v, s, dt, vbc, sbc, lower, upper, res, inflow, inflow_rate, buoyancy, smoke_advection)
    v_star = [(a * f).astype(F32) for a, f in zip(v_b, factors)]
    dx = [(F32(upper[a]) - F32(lower[a])) / F32(res[a]) for a in range(len(res))]
    v_new, p_new, info = make_incompressible_obstacles(v_star, vbc, res, dx, accessible, None, rtol, atol, max_iter, x0=p, method=method)
    return v_star, v_new, s_new, p_new, info


class ObstacleStepEngine(MaskedMethodEngine):
    @classmethod
    def plume_step(cls, dom, vspec, sbc, v, s, p, inflow, dt, inflow_rate, buoyancy, prm, mac_cormack=False, cg_events=None,
                   static_scalar=False, accessible=None, factors=None):
        if accessible is None:
            return super().plume_step(dom, vspec, sbc, v, s, p, inflow, dt, inflow_rate, buoyancy, prm, mac_cormack, cg_events, static_scalar)
        assert not static_scalar, "forced step: not in the stand-in"
        lower, upper = cls._geom(dom)
        comps = dom.faces_to_numpy(v, vspec, squeeze=False)
        ss, pp = dom.centered_to_numpy(s, squeeze=False), dom.centered_to_numpy(p, squeeze=False)
        infl = dom.centered_to_numpy(inflow, squeeze=False) if inflow is not None else np.zeros_like(ss)
        acc, fac = dom.centered_to_numpy(accessible, squeeze=False), dom.faces_to_numpy(factors, vspec, squeeze=False)
        method = 'CG-adaptive' if prm.method == 1 else 'CG'
        outs, s_new, p_new, infos = [], [], [], []
        for b in range(dom.batch):
            _, vb, sb, pb, info = step([c[b] for c in comps], ss[b], pp[b], dt, vspec, sbc, lower, upper, dom.res, infl[b], inflow_rate,
                                       tuple(buoyancy), acc[b], [f[b] for f in fac], prm.rtol, prm.atol, prm.max_iter, method,
                                       'mac_cormack' if mac_cormack else 'semi_lagrangian')
            outs.append(vb); s_new.append(sb); p_new.append(pb); infos.append(info)
        for c, t in enumerate(dom.faces_from_numpy([np.stack([o[c] for o in outs]) for c in range(dom.dim)], vspec)):
            v[c].copy_(t)
        s.copy_(dom.centered_from_numpy(np.stack(s_new)))
        p.copy_(dom.centered_from_numpy(np.stack(p_new)))
        cls._record(dom, infos)
        return v, s, p
