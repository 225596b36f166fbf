"""
The obstacle projection with a choice of solver, for the tests of CG-adaptive with obstacles (test infrastructure; the product never
imports this file).  oracle_np.make_incompressible_obstacles runs plain CG; make_incompressible_obstacles(method='CG-adaptive') below
runs the same sequence (phi/physics/fluid.py:121-162) with oracle_np.cg_adaptive, as make_incompressible(v, obstacle, Solve()) does
in the reference ('auto' = CG-adaptive, PhiML backend/_backend.py:1446-1447).  MaskedMethodEngine is the oracle-backed engine of
tests/oracle_engine.py whose obstacle projection honours prm.method, as its projection without obstacles already does.
"""
import numpy as np

from oracle import oracle_np as O
from oracle_engine import OracleEngine

F32 = np.float32


def make_incompressible_obstacles(v, vbc, res, dx, accessible, vmask=None, rtol=1e-5, atol=1e-5, max_iter=1000, x0=None, matrix=None,
                                  method='CG'):
    """oracle_np.make_incompressible_obstacles with method 'CG' (the same call) or 'CG-adaptive'.  Returns (v_new, p, info)."""
    if method == 'CG':
        return O.make_incompressible_obstacles(v, vbc, res, dx, accessible, vmask, rtol, atol, max_iter, x0, matrix)
    assert method == 'CG-adaptive', method
    d = len(res)
    kinds = vbc[0] if isinstance(vbc, list) else vbc          # per-component constants (vec boundaries) share the side kinds
    accessible = accessible.astype(F32)
    if vmask is not None:
        v = [a * m for a, m in zip(v, vmask)]
    div = O.divergence_staggered(v, dx, O.component_bcs(vbc, d)) * accessible
    if not O.is_flexible(kinds):
        div = div - accessible * (np.mean(div, dtype=F32) / np.mean(accessible, dtype=F32))
    A = matrix if matrix is not None else O.masked_poisson_matrix(res, dx, kinds, accessible)
    x0 = np.zeros(res, F32) if x0 is None else x0
    info = O.cg_adaptive(A, div, x0, rtol, atol, max_iter, None)
    p = info['x'].reshape(res)
    grad = O.gradient_faces(p, dx, O.pressure_bc(kinds), kinds)
    hard = O.hard_bcs_faces(accessible, kinds)
    v_new = [a - g * h for a, g, h in zip(v, grad, hard)]
    return v_new, p, info


class MaskedMethodEngine(OracleEngine):
    @classmethod
    def make_incompressible_masked(cls, dom, vspec, v, p, prm, accessible):
        comps = dom.faces_to_numpy(v, vspec, squeeze=False)
        p0, acc = dom.centered_to_numpy(p, squeeze=False), dom.centered_to_numpy(accessible, squeeze=False)
        method = 'CG-adaptive' if prm.method == 1 else 'CG'
        outs, ps, infos = [], [], []
        for b in range(dom.batch):
            vb, pb, info = make_incompressible_obstacles([c[b] for c in comps], vspec, dom.res, dom.dx, acc[b], None, prm.rtol, prm.atol,
                                                         prm.max_iter, x0=p0[b], method=method)
            outs.append(vb); ps.append(pb); infos.append(info)
        new = dom.faces_from_numpy([np.stack([o[c] for o in outs]) for c in range(dom.dim)], vspec)
        for c in range(dom.dim):
            v[c].copy_(new[c])
        p.copy_(dom.centered_from_numpy(np.stack(ps)))
        cls._record(dom, infos)
