"""Host model of ``rq_h`` / ``rq_dphi_dalpha`` in ``stheno_b200/csrc/kernel_matrix_bwd.cu`` (test infrastructure).

``h(w) = log1p(w) - w / (1 + w)``, so that ``d/d alpha (1 + w)^-alpha = -(1 + w)^-alpha h(w)`` at fixed ``d2``
(``w = d2 / (2 alpha)``).  The model restates the device function operation for operation: ``+ - * /`` on Python floats
round like the device's double operations, every ``fma`` is evaluated exactly and rounded once (through
``fractions.Fraction``), and the ``1 / (2j + 3)`` constants are the correctly rounded doubles the compiler folds.  The one
library call, ``log1p`` (only for ``w > 3``), is taken correctly rounded here; the device's is within 1 ulp of that.

``exact_h`` is ``h`` from ``mpmath`` at 50 significant digits: the series ``sum_{k>=2} t^k / k`` (``t = w / (1 + w)``) for
``t < 0.1``, where the direct form would cancel, and the direct form above it (at most a factor 20 lost to the
subtraction, 48 digits left)."""
import math
from fractions import Fraction

import mpmath

SPLIT = 3.0  # RQ_H_SPLIT
TERMS = 36  # RQ_H_TERMS


def fma(a, b, c):
    """``a * b + c`` with one rounding (finite arguments)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _log1p_cr(w):
    with mpmath.workdps(50):
        return float(mpmath.log1p(mpmath.mpf(w)))


def rq_h(w):
    w = float(w)
    if not w <= SPLIT:
        if w != w:
            return w
        if math.isinf(w):
            return math.nan  # inf - inf / inf: the caller returns 0 where phi is 0
        return _log1p_cr(w) - w / (1.0 + w)
    u2 = 2.0 + w
    s = w / u2
    e2 = 2.0 - (u2 - w) if w >= 2.0 else w - (u2 - 2.0)
    ds = fma(-s, e2, fma(-s, u2, w)) / u2
    s2 = s * s
    p = 1.0 / (2 * (TERMS - 1) + 3)
    for j in range(TERMS - 2, -1, -1):
        p = fma(p, s2, 1.0 / (2 * j + 3))
    c = s2 * s
    corr = 4.0 * s * ds / ((1.0 - s) * (1.0 + s) * (1.0 + s))
    return fma(c + c, p, (s2 + s2) / (1.0 + s)) + corr


def rq_dphi_dalpha(w, phi):
    """``-phi h(w)``, 0 where ``phi`` is 0."""
    return 0.0 if phi == 0.0 else -phi * rq_h(w)


def exact_h(w):
    """``h(w)`` from mpmath at 50 digits (an mpf)."""
    with mpmath.workdps(50):
        w = mpmath.mpf(w)
        if w == 0:
            return w
        t = w / (1 + w)
        if t < mpmath.mpf("0.1"):
            s, tk, k = mpmath.mpf(0), t * t, 2
            while True:
                term = tk / k
                s += term
                if term < s * mpmath.mpf(10) ** -52:
                    return s
                tk *= t
                k += 1
        return mpmath.log1p(w) - t


def exact_dphi_dalpha(d2, alpha):
    """``d/d alpha (1 + d2 / (2 alpha))^-alpha`` at 50 digits (an mpf)."""
    with mpmath.workdps(50):
        a = mpmath.mpf(alpha)
        w = mpmath.mpf(d2) / (2 * a)
        return -mpmath.power(1 + w, -a) * exact_h(w)


def ulps(got, want):
    """``|got - want|`` in units of the last place of ``want`` (a float64 normal number)."""
    wf = float(want)
    with mpmath.workdps(50):
        return float(abs(mpmath.mpf(got) - want) / mpmath.mpf(math.ulp(wf)))
