"""
Fp64OracleEngine: tests/oracle_engine.OracleEngine for float64 domains (math.set_global_precision(64) in the mirror), with every
oracle function evaluated under oracle_np.precision(64) and PhiCgResult64 records.  Host tests run the mirror's fp64 path and
examples/taylor_green.py over it without a GPU; the GPU tests use its step as the yardstick of the Taylor-Green run.
"""
import numpy as np
import torch

from oracle import oracle_np as O
from oracle_engine import OracleEngine
from phiflow_b200 import _ops


def taylor_green_step(v, p, dt, viscosity, vbc, res, dx, lower, upper, rtol=1e-12, atol=1e-12, max_iter=1000):
    """The notebook step on NumPy arrays in float64: diffuse.explicit, semi_lagrangian, make_incompressible(Solve('CG', x0=p))."""
    with O.precision(64):
        v = O.diffuse_explicit(v, vbc, dx, viscosity, dt)
        v = O.semi_lagrangian_staggered(v, vbc, v, vbc, res, lower, upper, dt)
        return O.make_incompressible(v, vbc, res, dx, rtol, atol, max_iter, x0=p, use_matrix_offset=False)


class Fp64OracleEngine(OracleEngine):
    @staticmethod
    def _f64(dom):
        assert dom.dtype == torch.float64, "Fp64OracleEngine serves float64 domains"

    @classmethod
    def _record(cls, dom, infos):
        rec = np.zeros(dom.batch, dtype=_ops._RESULT_DTYPE64)
        for b, info in enumerate(infos):
            rec[b] = (info['iterations'], int(info['converged']), int(info['diverged']), info['residual_sq'], info['tol_sq'], 0.0)
        cls.last = rec

    @classmethod
    def laplace_axpy(cls, dom, bc, x, coeff, out=None):
        cls._f64(dom)
        a = dom.centered_to_numpy(x, squeeze=False)
        with O.precision(64):
            res = dom.centered_from_numpy(np.stack([a[b] + coeff * O.laplace(a[b], dom.dx, bc) for b in range(dom.batch)]))
        if out is not None:
            out.copy_(res)
            return out
        return res

    @classmethod
    def laplace(cls, dom, spec, x):
        cls._f64(dom)
        with O.precision(64):
            return super().laplace(dom, spec, x)

    @classmethod
    def divergence(cls, dom, vspec, v):
        cls._f64(dom)
        with O.precision(64):
            return super().divergence(dom, vspec, v)

    @classmethod
    def grad_sub(cls, dom, vspec, v, p, accessible=None):
        cls._f64(dom)
        with O.precision(64):
            return super().grad_sub(dom, vspec, v, p, accessible)

    @classmethod
    def advect_staggered(cls, dom, vspec, v, fspec, f, dt):
        cls._f64(dom)
        with O.precision(64):
            return super().advect_staggered(dom, vspec, v, fspec, f, dt)

    @classmethod
    def advect_centered(cls, dom, vspec, v, sspec, s, dt):
        cls._f64(dom)
        with O.precision(64):
            return super().advect_centered(dom, vspec, v, sspec, s, dt)

    @classmethod
    def make_incompressible(cls, dom, vspec, v, p=None, prm=None, accessible=None):
        cls._f64(dom)
        assert accessible is None and isinstance(prm, _ops.PhiCgParams64) and prm.method == 0
        comps = dom.faces_to_numpy(v, vspec, squeeze=False)
        p0 = dom.centered_to_numpy(p, squeeze=False)
        outs, ps, infos = [], [], []
        with O.precision(64):
            for b in range(dom.batch):
                vb, pb, info = O.make_incompressible([c[b] for c in comps], vspec, dom.res, dom.dx, prm.rtol, prm.atol, prm.max_iter,
                                                     x0=p0[b], use_matrix_offset=False)
                outs.append(vb); ps.append(pb); infos.append(info)
        for c, t in enumerate(dom.faces_from_numpy([np.stack([o[c] for o in outs]) for c in range(dom.dim)], vspec)):
            v[c].copy_(t)
        p.copy_(dom.centered_from_numpy(np.stack(ps)))
        cls._record(dom, infos)
        return v, p
