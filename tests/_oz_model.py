"""NumPy integer model of the int8-slice fp64 emulation in ``stheno_b200/csrc/gemm_oz.cu`` (test infrastructure).

It restates, operation for operation, what ``oz_slice_kernel`` and ``oz_gemm_kernel`` compute: the power-of-two row scaling,
the round-to-nearest 7-bit slicing (error-free: every step is exact in fp64), the exact integer slice products grouped by
``s + t``, the fp64 Horner recombination and the scaling.  Because every inexact step of the kernel is a single correctly
rounded fp64 operation, the kernel's output must equal this model BIT FOR BIT (``tests/test_emulation.py``).

Semantics at the edges: a row's exponent ``e = ilogb(max |x|) + 1`` covers every finite magnitude (subnormal rows give
``e`` down to -1073, rows near the overflow threshold 1024); a row holding a NaN or an infinity gets zero slices and makes
its whole row / column of the product NaN.  The result is ``(v alpha) 2^E`` with ``E = e_row + e_col - (12 + 7 (S-1))``
summed as an integer and applied as at most two normal powers of two."""
import numpy as np

#: row exponent the kernel gives a row with a NaN or an infinity
E_NONFINITE = 1 << 20


def _pow2(e):
    """``2^e`` for integer ``e`` in [-1022, 1023] (exact normal doubles)."""
    return np.ldexp(1.0, np.asarray(e, np.int64))


def _clamp(e):
    return np.clip(e, -1022, 1023)


def slice_rows(X, S):
    """``X [rows, K]`` -> (``e [rows]``, list of ``S`` int64 arrays ``q_s [rows, K]``, remainder) with
    ``X = 2^e * sum_s q_s 2^-(6 + 7 s) + 2^e * remainder``, ``|q_s| <= 64``, ``|remainder| <= 2^-7S`` for finite rows."""
    X = np.asarray(X, np.float64)
    finite = np.isfinite(X).all(axis=1)
    with np.errstate(invalid="ignore"):
        m = np.where(finite, np.abs(np.where(np.isfinite(X), X, 0.0)).max(axis=1, initial=0.0), 0.0)
    _, ex = np.frexp(m)  # m = f * 2^ex, f in [0.5, 1)  ->  ilogb(m) + 1 = ex (subnormal m included)
    e = np.where(m > 0, ex, 0).astype(np.int64)
    s1 = _clamp(-e)
    Xf = np.where(finite[:, None], X, 0.0)
    r = Xf * _pow2(s1)[:, None] * _pow2(-e - s1)[:, None]  # two exact scalings, like the kernel
    e = np.where(finite, e, E_NONFINITE)
    qs, pw = [], 64.0
    for _ in range(S):
        t = np.rint(r * pw)  # round half to even, like the device rint()
        r = r - t / pw  # exact
        qs.append(t.astype(np.int64))
        pw *= 128.0
    return e, qs, r


def gemm(A, B, C0, alpha, beta, S):
    """``beta * C0 + alpha * A @ B.T`` the way the kernel forms it (A: [M, K], B: [N, K])."""
    ea, qa, _ = slice_rows(A, S)
    eb, qb, _ = slice_rows(B, S)
    acc = [sum(qa[s] @ qb[d - s].T for s in range(d + 1)) for d in range(S)]  # exact integers, diagonal d = s + t
    v = acc[0].astype(np.float64)
    for d in range(1, S):
        v = v * 128.0 + acc[d].astype(np.float64)  # v * 128 is exact: one rounding per step, like the device fma
    E = ea[:, None] + eb[None, :] - (12 + 7 * (S - 1))
    e1 = _clamp(E)
    e2 = _clamp(E - e1)
    with np.errstate(over="ignore", under="ignore"):
        out = v * alpha * _pow2(e1) * _pow2(e2)
    out = np.where(E > E_NONFINITE // 2, np.nan, out)
    if beta == 0.0:
        return out
    base = C0 if beta == 1.0 else C0 * beta
    return base + out
