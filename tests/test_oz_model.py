"""CPU checks of the NumPy integer model of the fp64 emulation (``tests/_oz_model.py``): the slicing is error-free and the
modelled product has the accuracy the design claims.  (The GPU kernel is compared with this model bit for bit in
``tests/test_emulation.py``.)"""
from fractions import Fraction

import numpy as np
import pytest

from tests._oz_model import gemm, slice_rows


@pytest.mark.parametrize("S", [5, 6, 7, 8])
def test_slicing_is_error_free(S):
    rng = np.random.default_rng(S)
    X = rng.standard_normal((64, 256)) * np.exp(4 * rng.standard_normal((64, 1)))
    X[3] = 0.0  # an all-zero row (identity padding)
    X[5, 7] = 2.0 ** 10  # an exact power of two as the row maximum
    e, qs, rem = slice_rows(X, S)
    assert all(np.abs(q).max() <= 64 for q in qs)
    recon = sum(q.astype(np.float64) * 2.0 ** -(6 + 7 * s) for s, q in enumerate(qs)) * np.ldexp(1.0, e)[:, None]
    scale = np.ldexp(1.0, e)[:, None]
    # the first S slices carry 6 + 7 (S - 1) bits below the row's power-of-two scale; what is left is the remainder, exactly
    # (at 8 slices that is 55 bits, i.e. the reconstruction sum itself rounds at the last bit of the 53-bit mantissa)
    assert np.all(np.abs(X - recon) <= scale * 2.0 ** -(7 * S) * (1 + 1e-9) + np.abs(X) * 2.0 ** -52)
    assert np.all(np.abs(rem) <= 2.0 ** -(7 * S) * (1 + 1e-9))
    assert np.all(recon[3] == 0.0)


@pytest.mark.parametrize("S,tol", [(6, 2e-11), (7, 2e-13), (8, 5e-15)])
def test_model_product_accuracy(S, tol):
    rng = np.random.default_rng(10 + S)
    M, N, K = 96, 80, 512
    A = rng.standard_normal((M, K)) * np.exp(3 * rng.standard_normal((M, 1)))
    B = rng.standard_normal((N, K))
    ref = A @ B.T
    got = gemm(A, B, None, 1.0, 0.0, S)
    scale = np.abs(A).max(1)[:, None] * np.abs(B).max(1)[None, :] * np.sqrt(K)
    assert np.max(np.abs(got - ref) / scale) < tol


def test_model_is_exact_on_small_integers():
    rng = np.random.default_rng(0)
    A = rng.integers(-1000, 1000, (32, 128)).astype(np.float64)
    B = rng.integers(-1000, 1000, (48, 128)).astype(np.float64)
    assert np.array_equal(gemm(A, B, None, 1.0, 0.0, 7), A @ B.T)


def _exact_product(A, B):
    """``A @ B.T`` in exact rational arithmetic."""
    Af = [[Fraction(float(v)) for v in row] for row in A]
    Bf = [[Fraction(float(v)) for v in row] for row in B]
    return [[sum(a * b for a, b in zip(ra, rb)) for rb in Bf] for ra in Af]


# 2^k on the rows of A, 2^-k on the rows of B (capped at 2^1020 so that B stays finite): products of O(1), operands from
# subnormal to near overflow.  (Before the exponents were summed as integers, alpha = -1/3 lost 1e-11 of the bound at
# k = -980, 1e-5 at -1000 and everything below; rows beyond +-1000 were clamped.)
EXTREME_K = [0, -1070, -1020, -1000, -980, 980, 1000, 1020]


@pytest.mark.parametrize("alpha", [1.0, -1.0 / 3.0])
@pytest.mark.parametrize("k", EXTREME_K)
def test_model_exact_at_extreme_row_magnitudes(k, alpha):
    """The model (= the kernel, bit for bit) against exact rational products, at the design bound of 8 slices."""
    S, M, N, K = 8, 6, 5, 128
    rng = np.random.default_rng(abs(k) + 7)
    A = np.ldexp(rng.standard_normal((M, K)), k)
    B = np.ldexp(rng.standard_normal((N, K)), min(-k, 1020))
    got = gemm(A, B, None, alpha, 0.0, S)
    exact = _exact_product(A, B)
    rowmax, colmax = np.abs(A).max(1), np.abs(B).max(1)
    for i in range(M):
        for j in range(N):
            want = Fraction(alpha) * exact[i][j]
            err = abs(Fraction(float(got[i, j])) - want)
            scale = Fraction(float(rowmax[i])) * Fraction(float(colmax[j])) * Fraction(np.sqrt(K))
            assert float(err / scale) < 5e-15, (i, j, float(err / scale))


@pytest.mark.parametrize("alpha", [1.0, -1.0 / 3.0])
def test_model_subnormal_results(alpha):
    """Products of two small rows land in the subnormal range: the error stays within the bound plus a few subnormal ulps
    (the one place where the final scaling may round twice)."""
    S, K = 8, 128
    rng = np.random.default_rng(1)
    A = np.ldexp(rng.standard_normal((4, K)), -560)
    B = np.ldexp(rng.standard_normal((3, K)), -490)
    got = gemm(A, B, None, alpha, 0.0, S)
    exact = _exact_product(A, B)
    tiny = Fraction(2) ** -1074
    for i in range(4):
        for j in range(3):
            want = Fraction(alpha) * exact[i][j]
            scale = Fraction(float(np.abs(A[i]).max())) * Fraction(float(np.abs(B[j]).max())) * Fraction(np.sqrt(K))
            assert abs(Fraction(float(got[i, j])) - want) <= Fraction(5e-15) * scale + 2 * tiny
    assert np.all(np.abs(got) < 2.0**-1000) and np.any(got != 0)


def test_model_nonfinite_rows():
    """A row holding a NaN, +inf or -inf makes its whole row (column) of the product NaN, where fp64 is non-finite too; every
    other element equals the product with those rows set to zero, bit for bit."""
    rng = np.random.default_rng(2)
    A = rng.standard_normal((8, 256))
    B = rng.standard_normal((6, 256))
    C0 = rng.standard_normal((8, 6))
    A[1, 5], A[4, 200], A[6, 0] = np.nan, np.inf, -np.inf
    B[2, 17], B[5, 255] = -np.inf, np.nan
    bad_a, bad_b = [1, 4, 6], [2, 5]
    with np.errstate(invalid="ignore"):
        ref = A @ B.T
    for alpha, beta in ((1.0, 0.0), (-1.5, 0.5), (-1.0, 1.0)):
        got = gemm(A, B, C0, alpha, beta, 7)
        assert not np.isfinite(ref[bad_a]).any() and not np.isfinite(ref[:, bad_b]).any()
        assert np.isnan(got[bad_a]).all() and np.isnan(got[:, bad_b]).all()
        A0, B0 = A.copy(), B.copy()
        A0[bad_a], B0[bad_b] = 0.0, 0.0
        clean = gemm(A0, B0, C0, alpha, beta, 7)
        keep = np.ones(got.shape, bool)
        keep[bad_a] = False
        keep[:, bad_b] = False
        assert np.array_equal(got[keep], clean[keep])


def test_slicing_full_exponent_range():
    """Row exponents are exact over the whole finite range: no clamp at +-1000, no cap at 1e300."""
    X = np.zeros((5, 128))
    X[0, 3] = 5e-324  # the smallest subnormal
    X[1, 9] = np.ldexp(1.5, -1060)
    X[2, 0] = np.finfo(np.float64).max
    X[3, 4] = 1e305
    X[4, 7] = -np.ldexp(1.0, -1010)
    e, qs, rem = slice_rows(X, 8)
    assert list(e) == [-1073, -1059, 1024, 1014, -1009]
    recon = sum(q.astype(np.float64) * 2.0 ** -(6 + 7 * s) for s, q in enumerate(qs))
    assert np.array_equal(np.ldexp(recon, e[:, None]), X)


def test_auto_slice_count_heuristic():
    """``B.precision = "auto"``: 7 slices only for factorisations that are well conditioned by construction."""
    from stheno_b200 import B, ops

    eq = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    eq_delta = ops.FlatKernel([(2.0, [("eq", 0)]), (0.1, [("delta", 0)])], 1)
    lin = ops.FlatKernel([(1.0, [("linear", 0)])], 1)
    assert ops._well_conditioned(eq, 0.1, None, 1e-12)
    assert ops._well_conditioned(eq_delta, 0.0, None, 1e-12)  # the Delta term is the noise
    assert not ops._well_conditioned(eq, 0.0, None, 1e-12)  # noise-free: only the jitter
    assert not ops._well_conditioned(eq, 1e-9, None, 0.0)
    assert not ops._well_conditioned(eq, 1e-4, None, 0.0)  # measured: the 7-slice log-pdf error reaches 1e-10 near 1e-4
    assert not ops._well_conditioned(eq, 0.1, object(), 0.0)  # per-point noise: smallest entry unknown on the host
    assert not ops._well_conditioned(lin, 0.1, None, 0.0)  # unbounded kernel
    before = B.precision
    try:
        B.precision = "auto"
        assert ops._oz_slices(True) == 7 and ops._oz_slices(False) == 8
        B.precision = "int8x6"
        assert ops._oz_slices(True) == 6 and ops._oz_slices(False) == 6
        B.precision = "fp64"
        assert ops._oz_slices(True) == 0
        B.precision = "tf32x3"
        assert ops._oz_slices(False) == 0
    finally:
        B.precision = before
