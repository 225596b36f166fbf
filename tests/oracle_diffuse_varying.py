"""
diffuse.implicit with a spatially varying diffusivity (phi/physics/diffuse.py:48-59, 90-95, 129-141) restated on the oracle's pieces
(oracle/oracle_np.py) - test infrastructure only.

The reference solves sharpen(x) = explicit(x, k, -dt) = y; traced by jit_compile_linear, solve_linear solves the affine system
M x = y - bias (PhiML/phiml/math/_optimize.py:616-645) with M = I + D0, the face-minimum stencil of w = -dt k (varying_system below).
Pinned against PhiML 1.7.2 by tests/golden/phiml_diffuse_varying.npz (tests/golden/make_diffuse_varying_golden.py).

VaryingDiffuseOracleEngine is tests/oracle_diffuse.DiffuseOracleEngine plus the engine's diffuse_implicit_varying, for the host tests
of the mirror and the facade.
"""
import numpy as np
import scipy.sparse as sp

from oracle import oracle_np as O
from oracle_diffuse import DiffuseOracleEngine
from phiflow_b200 import _ops


def _flat_index(res, idx):
    return np.ravel_multi_index(tuple(idx), res)


def varying_system(u, k, bc, dx, dt, face='w', coef_bc=None):
    """(M, y - bias) of diffuse.implicit(u, k, dt) with a spatially varying diffusivity k (phi/physics/diffuse.py:129-141):
        sharpen(x) = x + sum_d [f_{i+1/2} (x_{i+1} - x_i) - f_{i-1/2} (x_i - x_{i-1})] / dx_d^2,
        f = min(w_lo, w_hi), w = fl(-dt * k) with u's boundary as its ghosts (constants c unscaled: f_b = min(w_edge, c)),
    traced as M x = y - bias: M = I + D0 (value ghosts of constant sides 0, their coefficient ghosts keep c), bias = sharpen(0) =
    sum over constant sides of f_b c / dx^2.  face='k' builds the faces as fl(-dt * min(k_lo, k_hi)) instead - not the reference;
    the host tests use it to show that the golden data tells the two rules apart (for dt > 0 it takes the face MINIMUM of k where
    the reference's min(-dt k) is the face MAXIMUM).  coef_bc: another boundary for the coefficient ghosts (default: bc, as in the
    reference) - also only for showing what the golden data pins."""
    u = np.asarray(u, np.float32)
    k = np.asarray(k, np.float32)
    res, n_cells = u.shape, u.size
    w = (np.float32(-dt) * k).astype(np.float32)
    rows, cols, vals = [], [], []
    diag = np.ones(n_cells, np.float64)
    bias = np.zeros(n_cells, np.float64)
    idx = np.indices(res)
    for ax in range(u.ndim):
        n = res[ax]
        lo, hi = bc[ax]
        inv = 1.0 / float(np.float32(dx[ax]) ** 2)
        if face == 'w':
            wp = O.pad_axis(w, ax, 1, 1, (coef_bc or bc)[ax])
            f = np.minimum(np.take(wp, np.arange(0, n + 1), axis=ax), np.take(wp, np.arange(1, n + 2), axis=ax))
        else:
            kp = O.pad_axis(k, ax, 1, 1, tuple(s if isinstance(s, str) else np.float32(s) / np.float32(-dt) for s in bc[ax]))
            f = (np.float32(-dt) * np.minimum(np.take(kp, np.arange(0, n + 1), axis=ax), np.take(kp, np.arange(1, n + 2), axis=ax))).astype(np.float32)
        f = f.astype(np.float64)
        for j in range(n + 1):                                      # face j lies between cells j - 1 and j
            fj = np.take(f, j, axis=ax)
            if 0 < j < n:
                a = _flat_index(res, [np.take(idx[d], j - 1, axis=ax) for d in range(u.ndim)]).ravel()
                b = _flat_index(res, [np.take(idx[d], j, axis=ax) for d in range(u.ndim)]).ravel()
                c = fj.ravel() * inv
                rows += [a, b]; cols += [b, a]; vals += [c, c]
                np.subtract.at(diag, a, c); np.subtract.at(diag, b, c)
                continue
            cell = 0 if j == 0 else n - 1
            side = lo if j == 0 else hi
            me = _flat_index(res, [np.take(idx[d], cell, axis=ax) for d in range(u.ndim)]).ravel()
            c = fj.ravel() * inv
            if side == O.PERIODIC:
                if j == 0:                                          # the wrapped face, counted once for each of its two cells
                    other = _flat_index(res, [np.take(idx[d], n - 1, axis=ax) for d in range(u.ndim)]).ravel()
                    rows += [me, other]; cols += [other, me]; vals += [c, c]
                    np.subtract.at(diag, me, c); np.subtract.at(diag, other, c)
            elif side != O.ZG:                                      # constant: value ghost 0 in D0, c in the bias
                np.subtract.at(diag, me, c)
                np.add.at(bias, me, c * float(side))
    rows.append(np.arange(n_cells)); cols.append(np.arange(n_cells)); vals.append(diag)
    M = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n_cells, n_cells))
    M.sum_duplicates()
    M = M.astype(np.float32)
    M.sort_indices()
    return M, (u.ravel() - bias.astype(np.float32)).astype(np.float32)


def sharpen_varying(x, k, bc, dx, dt):
    """sharpen(x) = explicit(x, k, -dt) evaluated directly on padded arrays (the same restatement as
    tests/golden/make_diffuse_varying_golden.py), for checking varying_system."""
    x = np.asarray(x, np.float32)
    w = (np.float32(-dt) * np.asarray(k, np.float32)).astype(np.float32)
    total = x.copy()
    for ax in range(x.ndim):
        n = x.shape[ax]
        wp, xp = O.pad_axis(w, ax, 1, 1, bc[ax]), O.pad_axis(x, ax, 1, 1, bc[ax])
        f = np.minimum(np.take(wp, np.arange(0, n + 1), axis=ax), np.take(wp, np.arange(1, n + 2), axis=ax))
        grad = (np.take(xp, np.arange(1, n + 2), axis=ax) - np.take(xp, np.arange(0, n + 1), axis=ax)) / np.float32(dx[ax])
        flux = f * grad
        total = total + (np.take(flux, np.arange(1, n + 1), axis=ax) - np.take(flux, np.arange(0, n), axis=ax)) / np.float32(dx[ax])
    return total


def diffuse_implicit_varying(u, k, bc, dx, dt, rtol=1e-5, atol=1e-5, max_iter=1000, x0=None, face='w', coef_bc=None):
    """One system: u, k centred arrays of the same shape.  Returns (x, oracle_np.cg info)."""
    M, y = varying_system(u, k, bc, dx, dt, face, coef_bc)
    info = O.cg(M, y, np.asarray(u if x0 is None else x0, np.float32).ravel(), rtol, atol, max_iter)
    return info['x'].reshape(np.shape(u)), info


class VaryingDiffuseOracleEngine(DiffuseOracleEngine):
    @classmethod
    def diffuse_implicit_varying(cls, dom, spec, u, k, dt, rtol=1e-5, atol=1e-5, max_iter=1000, x0=None):
        us = dom.centered_to_numpy(u, squeeze=False)
        kd = _ops.Domain(dom.res, dom.dx, k.shape[0], device='cpu')
        ks = kd.centered_to_numpy(k, squeeze=False)
        starts = None if x0 is None else dom.centered_to_numpy(x0, squeeze=False)
        outs, rec = [], np.zeros(dom.batch, dtype=_ops._RESULT_DTYPE)
        for b in range(dom.batch):
            x, info = diffuse_implicit_varying(us[b], ks[b if ks.shape[0] > 1 else 0], spec, dom.dx, dt, rtol, atol, max_iter,
                                               None if starts is None else starts[b])
            outs.append(x)
            rec[b] = (info['iterations'], int(info['converged']), int(info['diverged']), info['residual_sq'], info['tol_sq'], 0.0)
        cls.last = rec
        return dom.centered_from_numpy(np.stack(outs))
