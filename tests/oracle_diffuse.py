"""
diffuse.implicit (phi/physics/diffuse.py:63-95) restated on the oracle's pieces (oracle/oracle_np.py) - test infrastructure only.

The reference traces sharpen(x) = x - a L_bc(x) with jit_compile_linear and solve_linear solves the affine system M x = y - bias
(PhiML/phiml/math/_optimize.py:616-645):
    M    = I - a L0, L0 = laplace with every constant ghost 0 = oracle_np.poisson_matrix(res, dx, bc) (constant sides keep [-2 1]),
    bias = sharpen(0) = -a L_bc(0)  (non-zero next to constant sides with a non-zero value).
The components of a vector field are separate systems: the reference's tracer keeps the uncoupled vector dim out of the matrix and
solve_linear treats it as a batch dim (per-component iteration counts in tests/golden/phiml_diffuse_implicit.npz).  Pinned against
PhiML 1.7.2 by that file.

DiffuseOracleEngine is tests/oracle_engine.OracleEngine plus the engine's diffuse_implicit, for the host tests of the mirror and
the facade.
"""
import numpy as np
import scipy.sparse as sp

from oracle import oracle_np as O
from oracle_engine import OracleEngine
from phiflow_b200 import _ops


def helmholtz_system(u, bc, dx, amount):
    """(M, y - bias) of one centred array with boundary spec `bc`."""
    a = np.float32(amount)
    L0 = O.poisson_matrix(u.shape, dx, bc)
    M = (sp.identity(u.size, dtype=np.float32, format='csr') - L0 * a).astype(np.float32).tocsr()
    M.sort_indices()
    bias = (-a * O.laplace(np.zeros(u.shape, np.float32), dx, bc)).astype(np.float32)
    return M, (np.asarray(u, np.float32) - bias).ravel()


def diffuse_implicit(u, bc, dx, amount, rtol=1e-5, atol=1e-5, max_iter=1000, x0=None):
    """u: centred array with boundary spec `bc`, or a list of same-shaped component arrays with one spec or a list of specs.
    Returns (x of the same form, oracle_np.cg info - a list with one info per component for a list)."""
    if isinstance(u, (list, tuple)):
        bcs = bc if isinstance(bc, list) else [bc] * len(u)
        outs = [diffuse_implicit(c, bcs[i], dx, amount, rtol, atol, max_iter, None if x0 is None else x0[i]) for i, c in enumerate(u)]
        return [o[0] for o in outs], [o[1] for o in outs]
    M, y = helmholtz_system(u, bc, dx, amount)
    info = O.cg(M, y, np.asarray(u if x0 is None else x0, np.float32).ravel(), rtol, atol, max_iter)
    return info['x'].reshape(u.shape), info


class DiffuseOracleEngine(OracleEngine):
    @classmethod
    def diffuse_implicit(cls, dom, spec, u, amount, rtol=1e-5, atol=1e-5, max_iter=1000, x0=None):
        is_list = isinstance(u, (list, tuple))
        comps = [dom.centered_to_numpy(t, squeeze=False) for t in (u if is_list else [u])]
        starts = None if x0 is None else [dom.centered_to_numpy(t, squeeze=False) for t in (x0 if is_list else [x0])]
        bcs = spec if isinstance(spec, list) else [spec] * len(comps)
        outs, infos = [], []
        for b in range(dom.batch):
            xs, info = diffuse_implicit([c[b] for c in comps], bcs, dom.dx, amount, rtol, atol, max_iter,
                                        x0=[s[b] for s in starts] if starts is not None else None)
            outs.append(xs)
            infos += info                                       # entry b * C + c
        rec = np.zeros(len(infos), dtype=_ops._RESULT_DTYPE)
        for i, info in enumerate(infos):
            rec[i] = (info['iterations'], int(info['converged']), int(info['diverged']), info['residual_sq'], info['tol_sq'], 0.0)
        cls.last = rec
        res = [dom.centered_from_numpy(np.stack([o[c] for o in outs])) for c in range(len(comps))]
        return res if is_list else res[0]

    @classmethod
    def read_results(cls, dom, components=1):
        return cls.last
