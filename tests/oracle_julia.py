"""
NumPy restatement of the Julia_Set notebook's escape counts (examples/grids/Julia_Set.ipynb) with the rounding of PhiML 1.7.2's
NumPy backend on a CPU whose NumPy dispatches to its AVX-512 loops (complex64):

    next_z = z ** 2 + c         z ** 2 = np.power(z, 2):  re = a * a - b * b,  im = a * b + b * a;  then + c per component
    counter += abs(z) < 2       abs(z) = big * sqrt(fma(r, r, 1)),  r = small / big,  big / small = max / min(|a|, |b|)

Every operation is one float32 rounding; `fma32` is the exact fused multiply-add (tests/golden/phiml_julia.npz pins all of it).
PhiML's `**` calls np.power, whose complex loop multiplies without fma; NumPy's own `z ** 2` on an array would call np.square, whose
AVX-512 loop rounds re as fma(a, a, -(b * b)) instead (about a third of all inputs differ in the last bit).
`band_decision` is the kernel's shortcut for abs(z) < 2 (phiflow_b200/csrc/julia_kernels.cu): s = fma(a, a, b * b) decides outside
[JULIA_LO, JULIA_HI] and the exact formula inside.  The float32 operations are correctly rounded on every CPU, so the oracle does not
depend on NumPy's SIMD dispatch; only NumPy's own complex64 loops do.
"""
import numpy as np

F32 = np.float32
JULIA_LO = F32(4.0 - 2.0 ** -18)          # 4 (1 - 2^-20)
JULIA_HI = F32(4.0 + 2.0 ** -18)          # 4 (1 + 2^-20)


def fma32(a, b, c):
    """Correctly rounded float32 a * b + c: a * b is exact in float64, the sum is rounded once to float64 and once to float32.  The
    two roundings differ from one only where the float64 sum is a float32 midpoint; there the exact remainder (TwoSum) decides."""
    a, b, c = (np.asarray(v, F32) for v in (a, b, c))
    with np.errstate(all='ignore'):
        p = a.astype(np.float64) * b.astype(np.float64)
        c64 = c.astype(np.float64)
        s = p + c64
        bb = s - p
        err = (p - (s - bb)) + (c64 - bb)
        f = s.astype(F32)
        other = np.where(s > f, np.nextafter(f, F32(np.inf)), np.nextafter(f, F32(-np.inf)))
        tie = np.isfinite(s) & (s != f) & ((f.astype(np.float64) + other.astype(np.float64)) * 0.5 == s) & (err != 0)
        up = np.maximum(f, other)
        down = np.minimum(f, other)
        return np.where(tie, np.where(err > 0, up, down), f).astype(F32)


def square_plus(a, b, cr, ci):
    """z ** 2 + c for z = a + ib, c = cr + i ci (float32 arrays), as PhiML rounds it."""
    with np.errstate(all='ignore'):
        a, b = np.asarray(a, F32), np.asarray(b, F32)
        re = a * a - b * b
        ab = a * b
        return (re + F32(cr)).astype(F32), ((ab + b * a) + F32(ci)).astype(F32)


def abs32(a, b):
    """abs(a + ib) as NumPy's complex64 loop computes it (0 for z = 0, inf / nan for non-finite z)."""
    with np.errstate(all='ignore'):
        x, y = np.abs(np.asarray(a, F32)), np.abs(np.asarray(b, F32))
        big, small = np.maximum(x, y), np.minimum(x, y)
        r = small / big
        out = (big * np.sqrt(fma32(r, r, F32(1)))).astype(F32)
        out = np.where(big == 0, F32(0), out)
        return np.where(np.isinf(x) | np.isinf(y), F32(np.inf), out).astype(F32)


def band_decision(a, b):
    """The kernel's abs(z) < 2: fma(a, a, b * b) < JULIA_LO is inside, > JULIA_HI outside, the exact abs32 in between (nan: outside)."""
    with np.errstate(all='ignore'):
        a, b = np.asarray(a, F32), np.asarray(b, F32)
        s = fma32(a, a, b * b)
        return np.where(s < JULIA_LO, True, np.where(s > JULIA_HI, False, abs32(a, b) < F32(2)))


def julia_counts(xc, yc, c, iterations: int) -> np.ndarray:
    """Counts (batch, nx, ny) as int32: for every constant c[k] (complex) and cell (i, j), z0 = xc[i] + i yc[j] and the number of
    iterations t < `iterations` with abs(z_t) < 2."""
    xc, yc = np.asarray(xc, F32), np.asarray(yc, F32)
    c = np.atleast_1d(np.asarray(c, np.complex64))
    out = np.zeros((len(c), len(xc), len(yc)), np.int32)
    for k, ck in enumerate(c):
        a, b = np.meshgrid(xc, yc, indexing='ij')
        cnt = np.zeros(a.shape, np.int32)
        for _ in range(iterations):
            cnt += abs32(a, b) < F32(2)
            a, b = square_plus(a, b, F32(ck.real), F32(ck.imag))
        out[k] = cnt
    return out


class JuliaOracleEngine:
    """Stand-in for phiflow_b200._ops in host tests of the mirror: `julia` computed by julia_counts, in the library's layout."""
    from phiflow_b200._ops import Domain, stored_faces

    @staticmethod
    def julia(dom, centres, c, iterations, out=None):
        import torch
        counts = julia_counts(centres[:dom.res[0]], centres[dom.res[0]:], c, iterations)
        t = torch.zeros(dom._shape(dom.cext), dtype=torch.int32, device=dom.device)
        t[:, :dom.res[1], :dom.res[0]] = torch.from_numpy(np.ascontiguousarray(counts.transpose(0, 2, 1)))
        return t
