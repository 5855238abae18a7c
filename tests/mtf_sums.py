"""Restatement of the sums of rt_grid_mtf (include/b200rt.h, DESIGN.md section 4) in numpy, written
with explicit sequential chains, shift by shift: for one tile's pupil function P [n, n] (x outer)

    Cx(k) = sum over lines j (in order, from +0.0) of
            sum over i = 0 ... n-k-1 (in order, from +0.0) of P[i+k, j]*conj(P[i, j])
    Cy(k)   the same with the roles of i and j exchanged
    S       = sum over lines j of sum over i of P[i, j]

with a*conj(b) = (ar*br + ai*bi, ai*br - ar*bi), every real product rounded once.  The real and
imaginary parts are separate chains.  The mistake switches change one rule each, for the test that
the restatement is sensitive to them."""
import math
from fractions import Fraction

import numpy as np

U = 2.0**-53


def chain(v):
    """sum over axis 0 from +0.0 in increasing index (np.add.accumulate is a sequential chain)"""
    v = np.asarray(v, dtype=np.float64)
    return np.add.accumulate(np.concatenate([np.zeros((1,) + v.shape[1:]), v]), axis=0)[-1]


def _fma(a, b, c):
    """a*b + c rounded once (exact rational arithmetic)"""
    return np.array([float(Fraction(x)*Fraction(y) + Fraction(z)) for x, y, z in
                     zip(np.ravel(a), np.ravel(np.broadcast_to(b, np.shape(a))), np.ravel(c))]).reshape(np.shape(a))


def mul_conj(a, b, fma=False, conj_first=False):
    """(re, im) of a*conj(b); ``fma``: re contracted to fma(ar, br, ai*bi), im to
    fma(ai, br, -(ar*bi)); ``conj_first``: conj(a)*b instead"""
    ar, ai, br, bi = a.real, a.imag, b.real, b.imag
    if conj_first:
        return ar*br + ai*bi, ar*bi - ai*br
    if fma:
        return _fma(ar, br, ai*bi), _fma(ai, br, -(ar*bi))
    return ar*br + ai*bi, ai*br - ar*bi


def autocorr(P, axis, reverse_lines=False, fma=False, conj_first=False):
    """``[n]`` complex C(k) along ``axis`` (0: Cx, 1: Cy)"""
    Q = np.asarray(P, dtype=np.complex128)
    Q = Q if axis == 0 else Q.T
    n = Q.shape[0]
    out = np.zeros(n, dtype=np.complex128)
    for k in range(n):
        re, im = mul_conj(Q[k:], Q[:n - k], fma, conj_first)      # [n - k, lines]
        lr, li = chain(re), chain(im)                              # one sum per line
        if reverse_lines:
            lr, li = lr[::-1], li[::-1]
        out[k] = complex(chain(lr), chain(li))
    return out


def autocorr_at(P, axis, shifts):
    """C(k) of ``autocorr`` at the given shifts only"""
    Q = np.asarray(P, dtype=np.complex128)
    Q = Q if axis == 0 else Q.T
    n = Q.shape[0]
    out = []
    for k in shifts:
        re, im = mul_conj(Q[k:], Q[:n - k])
        out.append(complex(chain(chain(re)), chain(chain(im))))
    return np.array(out)


def pupil_sum(P):
    P = np.asarray(P, dtype=np.complex128)
    return complex(chain(chain(P.real)), chain(chain(P.imag)))


def sums(P):
    """(Cx [n], Cy [n], S) of one tile"""
    return autocorr(P, 0), autocorr(P, 1), pupil_sum(P)


def exact_autocorr(P, axis):
    """(exactly rounded C(k) of the same rounded product terms (math.fsum), sum of |terms|) ``[n]``"""
    Q = np.asarray(P, dtype=np.complex128)
    Q = Q if axis == 0 else Q.T
    n = Q.shape[0]
    ex = np.zeros(n, dtype=np.complex128)
    ab = np.zeros((n, 2))
    for k in range(n):
        re, im = mul_conj(Q[k:], Q[:n - k])
        ex[k] = complex(math.fsum(re.ravel()), math.fsum(im.ravel()))
        ab[k] = np.abs(re).sum(), np.abs(im).sum()
    return ex, ab


def gamma(m):
    return m*U/(1 - m*U)


def depth(n, k):
    """additions in the longest chain of shift k: n - k in a line, n for the lines"""
    return (n - k) + n


def disk_mask(n, holes=False, rng=None):
    """used-ray mask of an n x n grid over [-1, 1]^2: the unit disk (inclusive), optionally with
    random holes (failed rays)"""
    g = np.linspace(-1.0, 1.0, n) if n > 1 else np.zeros(1)
    x, y = np.meshgrid(g, g, indexing='ij')
    m = x*x + y*y <= 1.0
    if holes:
        m &= rng.random((n, n)) > 0.1
    return m, x, y


def phasors(w, mask):
    """exp(2 pi i w) where mask, else 0 (numpy; the device's are sincospi(2w))"""
    r = 2.0*np.pi*(w - np.rint(w))
    return np.where(mask, np.cos(r) + 1j*np.sin(r), 0.0 + 0.0j)
