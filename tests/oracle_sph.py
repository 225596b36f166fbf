"""
NumPy float32 restatement of one SPH substep of the SPH notebook (examples/particles/SPH.ipynb, phi/physics/sph.py:23-64, 116-185)
with the hash-grid neighbour search of PhiML's find_neighbors_sparse / build_hash_grid (PhiML/phiml/backend/_partition.py:116-240),
operation for operation as phiflow_b200/csrc/sph_kernels.cu forms it (include/phicuda.h, N12):

  1. hash grid: res = max(1, ceil(max(upper - lower, s) / s)), edge = (s res) / res, cell = trunc((x - lower) / edge) clamped into
     [0, res - 1] (NaN -> 0; the reference clamps above only);
  2. pairs (i, j) with sqrt(r2) < s, delta = x_j - x_i, r2 = (d0 d0 + d1 d1) + d2 d2, self included; the stored order of row i is the
     3^d neighbour cells in PhiML's offset order (x outermost), each cell's particles by ascending index;
  3. W = norm ((s s - r2)^2 (s s - r2)), rho_i = (sum_j W) m, p = iso (rho - base);
  4. d = sqrt(max(r2, 1e-5)), u = delta / d, gap = h - d;
  5. F_i = sum_j (P (((-u) avg) gap^2) + V (((v_j - v_i) / rho_j) gap)), avg = (p_i + p_j) / (2 rho_j); a = F / rho + g, v += a dt,
     x += dt v;
  6. c = clip(x, lower, upper); v *= damping where c != x (per component); x = c.

Every sum is sequential in the stored order (np.add.at in row order), every operation one float32 rounding.  Where this differs
from PhiML's NumPy backend, tests/test_sph_host.py states the tolerance: NumPy's unstable argsort orders a cell's particles, and
np.power rounds x ** 3 and s ** 9 differently from (x x) x.
"""
import numpy as np

F = np.float32


def hash_grid(lower, upper, s, d):
    """(res, edge) of PhiML's build_hash_grid in float32."""
    lo, up, s = np.asarray(lower, F)[:d], np.asarray(upper, F)[:d], F(s)
    size = np.maximum(up - lo, s)
    res = np.maximum(1, np.ceil(size / s).astype(np.int64))
    edge = (s * res.astype(F)) / res.astype(F)
    return res, edge.astype(F)


def cells(x, lower, res, edge):
    """Integer cell coordinates (n, d), truncated toward zero and clamped into [0, res - 1]; NaN -> 0."""
    d = x.shape[1]
    t = (x - np.asarray(lower, F)[:d]) / edge
    t = np.where(np.isnan(t), F(0), t)
    t = np.clip(t, F(-1), res.astype(F))
    return np.clip(np.trunc(t).astype(np.int64), 0, res - 1)


def kernel_norm(s, d):
    """PhiML's poly6 normalisation const / s ** (d + 6) (np.power, as PhiML's NumPy backend rounds it)."""
    const = 315 / 64 / np.pi if d == 3 else 4 / np.pi
    return F(F(const) / np.power(np.asarray(s, F), d + 6))


def pairs(x, lower, upper, s, rows=None):
    """(i, j) of every stored pair whose row i is in `rows` (all particles by default), rows ascending, each row in stored order."""
    n, d = x.shape
    res, edge = hash_grid(lower, upper, s, d)
    c = cells(x, lower, res, edge)
    lin = np.ravel_multi_index(tuple(c.T), tuple(res))
    order = np.argsort(lin, kind='stable')
    start = np.searchsorted(lin[order], np.arange(np.prod(res) + 1))
    rows = np.arange(n) if rows is None else np.asarray(rows)
    offsets = np.stack(np.meshgrid(*[(-1, 0, 1)] * d, indexing='ij'), -1).reshape(-1, d)
    I, K, J = [], [], []
    for k, off in enumerate(offsets):
        nc = c[rows] + off
        ok = np.all((nc >= 0) & (nc < res), axis=1)
        cid = np.where(ok, np.ravel_multi_index(tuple(np.clip(nc, 0, res - 1).T), tuple(res)), 0)
        cnt = np.where(ok, start[cid + 1] - start[cid], 0)
        r = np.repeat(rows, cnt)
        first = np.repeat(start[cid], cnt)
        t = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        I.append(r)
        K.append(np.full(len(r), k))
        J.append(order[first + t])
    I, K, J = np.concatenate(I), np.concatenate(K), np.concatenate(J)
    srt = np.lexsort((K, I))           # stable: (row, offset), then the cell's ascending order
    I, J = I[srt], J[srt]
    delta, r2 = _delta(x, I, J)
    keep = np.sqrt(r2) < F(s)
    return I[keep], J[keep]


def _delta(x, I, J):
    delta = x[J] - x[I]
    r2 = delta[:, 0] * delta[:, 0]
    for a in range(1, x.shape[1]):
        r2 = r2 + delta[:, a] * delta[:, a]
    return delta, r2


def density(x, I, J, s, norm, m, n=None):
    """rho for every row: (sequential sum of W over the row's pairs) * m."""
    _, r2 = _delta(x, I, J)
    diff = F(s) * F(s) - r2
    w = F(norm) * ((diff * diff) * diff)
    acc = np.zeros(len(x) if n is None else n, F)
    np.add.at(acc, I, w)
    return acc * F(m), w


def forces(x, v, rho, I, J, h, P, V, iso, base):
    """F for every row (n, d); rho must hold every row and column of the pairs."""
    delta, r2 = _delta(x, I, J)
    p = F(iso) * (rho - F(base))
    dist = np.sqrt(np.maximum(r2, F(1e-5)))
    gap = F(h) - dist
    avg = (p[I] + p[J]) / (F(2) * rho[J])
    u = delta / dist[:, None]
    pf = ((-u) * avg[:, None]) * (gap * gap)[:, None]
    vf = ((v[J] - v[I]) / rho[J][:, None]) * gap[:, None]
    term = F(P) * pf + F(V) * vf
    f = np.zeros_like(x)
    np.add.at(f, I, term)
    return f


def integrate(x, v, f, rho, dt, gravity, lower, upper, damping):
    d = x.shape[1]
    a = f / rho[:, None] + np.asarray(gravity, F)[:d]
    v = v + a * F(dt)
    x = x + F(dt) * v
    lo, up = np.asarray(lower, F)[:d], np.asarray(upper, F)[:d]
    c = np.where(x < lo, lo, np.where(x > up, up, x))
    v = np.where(c == x, v, v * F(damping))
    return c.astype(F), v.astype(F)


def sph_substep(x, v, prm, rows=None):
    """One substep.  prm: dict(lower, upper, s, h, norm, m, P, V, iso, base, dt, gravity, damping).  Returns (x, v, rho, f);
    with `rows`, only those particles' (x, v, rho, f) are formed, from the density of every particle they interact with."""
    x, v = np.asarray(x, F), np.asarray(v, F)
    if rows is None:
        I, J = pairs(x, prm['lower'], prm['upper'], prm['s'])
        rho, _ = density(x, I, J, prm['s'], prm['norm'], prm['m'])
        idx = slice(None)
    else:
        I, J = pairs(x, prm['lower'], prm['upper'], prm['s'], rows)
        need = np.unique(np.concatenate([np.asarray(rows), J]))
        I2, J2 = pairs(x, prm['lower'], prm['upper'], prm['s'], need)
        rho, _ = density(x, I2, J2, prm['s'], prm['norm'], prm['m'])
        idx = np.asarray(rows)
    f = forces(x, v, rho, I, J, prm['h'], prm['P'], prm['V'], prm['iso'], prm['base'])
    xn, vn = integrate(x[idx], v[idx], f[idx], rho[idx], prm['dt'], prm['gravity'], prm['lower'], prm['upper'], prm['damping'])
    return xn, vn, rho[idx], f[idx]


def sph(x, v, prm, substeps=1):
    """`substeps` substeps; returns (x, v, rho of the last substep)."""
    x, v = np.asarray(x, F), np.asarray(v, F)
    rho = None
    for _ in range(substeps):
        x, v, rho, _ = sph_substep(x, v, prm)
    return x, v, rho


def notebook_params(d=3, h=0.8, lower=None, upper=None):
    """The notebook's constants as its PhiML tensors round them: Sphere(volume=h ** d) stores radius_from_volume(volume) and reports
    volume_from_radius(radius); desired_neighbors = volume_from_radius(h) / volume, s = radius_from_volume(volume desired_neighbors)
    (phi/geom/_sphere.py:69-90, phi/physics/sph.py:71-98); m = 0.01 volume, P = -(45 m) / (pi h^6), V = (45 0.025 m) / (pi h^6).
    The domain defaults to the notebook's Box(x=80, y=80, z=80)."""
    vol = np.asarray(h ** d, F)
    if d == 3:
        volume = F(4 / 3 * np.pi) * np.power(np.power(F(.75 / np.pi) * vol, 1 / 3), 3)
        s = np.power(F(.75 / np.pi) * (volume * (F(4 / 3 * np.pi * h ** 3) / volume)), 1 / 3)
    else:
        volume = F(np.pi) * np.power(np.sqrt(vol / F(np.pi)), 2)
        s = np.sqrt((volume * (F(np.pi * h ** 2) / volume)) / F(np.pi))
    m = F(0.01) * volume
    P = -(F(45.0) * m) / F(np.pi * h ** 6)
    V = (F(45.0 * 0.025) * m) / F(np.pi * h ** 6)
    g = (0., 0., -0.1) if d == 3 else (0., -0.1)
    return dict(lower=tuple(lower or (0.,) * d), upper=tuple(upper or (80.,) * d), s=F(s), h=F(h), norm=kernel_norm(s, d), m=F(m),
                P=F(P), V=F(V), iso=F(20.), base=F(1.), dt=F(0.01 * h), gravity=tuple(F(c) for c in g), damping=F(-0.95))


def notebook_lattice(nx=25, ny=100, nz=25, h=0.8, seed=0, d=3):
    """The notebook's initial positions: meshgrid(x=nx, y=ny, z=nz) packed x-major, * h, + 0.001 h N(0, 1) (seeded here)."""
    dims = (nx, ny, nz)[:d]
    grid = np.stack(np.meshgrid(*[np.arange(k) for k in dims], indexing='ij'), -1).reshape(-1, d).astype(F) * F(h)
    rng = np.random.default_rng(seed)
    return (grid + F(0.001 * h) * rng.standard_normal(grid.shape).astype(F)).astype(F)
