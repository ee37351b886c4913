"""The fp32 route against fp64 references at its edges: the 3xTF32 tensor-core GEMM and the FFMA GEMM, the fp32 Cholesky with
its fused and separate triangular solves at the benchmarked shape (BASELINE config 3: batches of n = 2048), the opt-in
``B.precision = "tf32x3"`` fp64 Cholesky, and the fp32 row reductions behind posterior variances and log-pdfs.

Bounds, with u = 2^-24 (fp32's unit roundoff) and S = |alpha| |A| |B|^T:

- 3xTF32 GEMM, per entry: ``(6 K + 48) u S + 2 u (|ref| + |beta C|)`` (:func:`tc_bound`).  The split drops ``lo_a lo_b`` and the
  tensor core reads each ``lo`` truncated to TF32 again: each of these three losses is below 2^-20 |a||b| = 16 u |a||b|, so
  48 u S in all.  The 3 K partial products are then added into fp32 accumulators; with round toward zero (the worst case a
  tensor core may use) each addition errs by less than 2 u of the running sum, 6 K u S over 3 K additions.  The epilogue
  rounds ``alpha acc`` and the fused ``beta C`` once each.
- FFMA GEMM: ``2 K u S`` plus the same epilogue term, as ``tests/test_gpu_primitives.py`` uses.
- Cholesky: the backward error ``max |K - L L^T| / (n u max |K|)`` of every batch member, and the residuals of the solves
  ``|b - L x| <= c n u |L| |x|``, all computed in fp64 from the fp32 outputs: they do not depend on conditioning.  ``logdet``
  and the log-pdf against fp64 values of the same fp32 matrix, within the first-order effect of the measured backward error.
- Row reductions: a few u of the fp64 sum of the same fp32 values -- what an fp64 accumulator and one final rounding give.
"""
import math

import numpy as np
import pytest
import torch

from tests import _tf32x3_model as T

U = 2.0**-24


# ---- A. the host model of the 3xTF32 split (no GPU) -------------------------------------------------------------------


def _floats_every_low_pattern():
    """Every sign, every exponent field (0: subnormals, up to 254: the largest finite binade) and every pattern of the 13 low
    mantissa bits -- the bits the split acts on -- under four patterns of the 10 high mantissa bits (incl. +-max)."""
    low = np.arange(1 << 13, dtype=np.uint32)
    high = np.array([0, 1, 0x2AA, 0x3FF], dtype=np.uint32) << 13
    exp = np.arange(255, dtype=np.uint32) << 23
    bits = (exp[:, None, None] | high[None, :, None] | low[None, None, :]).ravel()
    bits = np.concatenate([bits, bits | np.uint32(0x80000000)])
    return bits.view(np.float32)


def test_split_is_exact_for_every_finite_float():
    a = _floats_every_low_pattern()
    assert np.isfinite(a).all() and np.float32(np.finfo(np.float32).max) in a and np.float32(2.0**-149) in a
    hi, lo = T.split(a)
    assert ((hi.view(np.uint32) & np.uint32(0x1FFF)) == 0).all()  # hi is a TF32 value
    assert np.array_equal(hi + lo, a)  # fp32 addition, exact
    assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), a.astype(np.float64))
    # normal a: |lo| < ulp_tf32(a) <= 2^-10 |a|, what the error bound assumes (a subnormal a may be all lo)
    normal = np.abs(a) >= 2.0**-126
    assert (np.abs(lo[normal]) < np.abs(a[normal]) * 2.0**-10).all()


def test_model_reproduces_the_probe_identity():
    """``a = 1 + 2^-11``: the split gives ``a^2 - 2^-22 = 1 + 2^-10`` (``lo_a lo_b = 2^-22`` is dropped), FFMA ``a^2``."""
    a = np.array([[1.0 + 2.0**-11]], np.float32)
    assert T.gemm_nt(a, a)[0, 0] == np.float32(1.0 + 2.0**-10)
    assert T.ffma_gemm_nt(a, a)[0, 0] == np.float32(1.0 + 2.0**-10 + 2.0**-22)
    hi, lo = T.split(a)
    assert hi[0, 0] == 1.0 and lo[0, 0] == 2.0**-11


def test_split_of_infinities_and_nans():
    """``lo = inf - inf = NaN``: a row holding +-inf makes its whole row of the product NaN (FFMA: +-inf).  A NaN whose
    payload lies only in the low 13 bits truncates to an infinity, but its ``lo`` is NaN, so it stays NaN.  Selecting
    ``lo = 0`` for infinities would not give fp32's answer either: ``hi_a lo_b`` is then ``inf * 0 = NaN`` for every ``b``
    that TF32 holds exactly (1, 0.5, ...)."""
    bits = np.array([0x7F800000, 0xFF800000, 0x7F800001, 0x7F801FFF, 0x7FC00000, 0xFFC00001], np.uint32)
    a = bits.view(np.float32)
    hi, lo = T.split(a)
    assert hi[0] == np.inf and hi[1] == -np.inf and np.isnan(lo[:2]).all()
    assert (hi[2:4].view(np.uint32) == 0x7F800000).all()  # low-payload NaNs: masking yields +inf
    assert np.isnan(hi[4:]).all() and np.isnan(lo[2:]).all()
    b = np.array([[2.0, 1.0 + 2.0**-11, -3.0]], np.float32)  # one k: each entry of a meets each entry of b
    tc = T.gemm_nt(a[:, None], b.T)
    assert np.isnan(tc).all()
    ffma = T.ffma_gemm_nt(a[:2, None], b.T)
    assert np.array_equal(ffma, np.array([[np.inf, np.inf, -np.inf], [-np.inf, -np.inf, np.inf]], np.float32))
    with np.errstate(invalid="ignore"):
        assert np.isnan(np.float64(np.inf) * T.split(np.float32(1.0))[1])


def test_model_bound_covers_the_split_loss():
    """The 48 u |a||b| of the split (three losses below 2^-20 |a||b| each) bounds the model's error on random 24-bit
    operands; and the model is 2^-21-level, not FFMA's 2^-24 (the bound is not vacuous)."""
    rng = np.random.default_rng(0)
    a = rng.standard_normal((512, 1)).astype(np.float32)
    b = rng.standard_normal((512, 1)).astype(np.float32)
    exact = a.astype(np.float64) @ b.astype(np.float64).T
    err = np.abs(T.gemm_nt(a, b).astype(np.float64) - exact)
    assert (err <= 48 * U * np.abs(exact) + U * np.abs(exact)).all()
    assert (err / np.abs(exact)).max() > 2 * U


# ---- B. the fp32 GEMM on both kernels -----------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def ops():
    from stheno_b200 import ops

    return ops


def _probe(ops, M, N, K, batch=1, lower=False):
    from tests.test_gpu_primitives import tc32_probe

    return tc32_probe(ops, M, N, K, batch, lower)


def tc_bound(K, alpha, absprod, ref, beta=0.0, Cabs=0.0, eta=0.0):
    """Per-entry bound of the 3xTF32 GEMM (module docstring); ``eta``: absolute error allowed per partial product for
    results in or below the subnormal range."""
    return (6 * K + 48) * U * abs(alpha) * absprod + 2 * U * (ref.abs() + abs(beta) * Cabs) + 3 * K * eta


def ffma_bound(K, alpha, absprod, ref, beta=0.0, Cabs=0.0, eta=0.0):
    return 2 * K * U * abs(alpha) * absprod + 2 * U * (ref.abs() + abs(beta) * Cabs) + K * eta


#: the tensor cores keep subnormal operands and subnormal products (measured on H100: the one-k products below agree with the
#: model without flushing, bit for bit), so an underflowing partial product errs by at most half the smallest subnormal
ETA = 2.0**-149


def _one_k_operands(rows, K, seed):
    """Rows ``r`` with a single non-zero at column ``r % K``: rows 0-5 special (+inf, -inf, a NaN with a low payload, a quiet
    NaN, two subnormals), 8-39 tiny (3 significant bits, 2^-72 .. 2^-60: products of two go subnormal), 40-55 huge (2^56 ..
    2^62: products reach 2^124), the rest 13 significant bits at 2^0 .. 2^40.  Every product is exact in fp32 or
    underflows to 0 whatever the rounding, so the one-k model is bit exact."""
    rng = np.random.default_rng(seed)
    v = np.ldexp(rng.integers(2**12, 2**13, rows).astype(np.float64), rng.integers(0, 41, rows) - 12)
    v[8:40] = np.ldexp(rng.integers(4, 8, 32).astype(np.float64), rng.integers(-72, -59, 32) - 2)
    v[40:56] = np.ldexp(rng.integers(4, 8, 16).astype(np.float64), rng.integers(56, 63, 16) - 2)
    v *= rng.choice([-1.0, 1.0], rows)
    v = v.astype(np.float32)
    v[:6] = np.array([0x7F800000, 0xFF800000, 0x7F800001, 0x7FC00000, 0x00300000, 0x80280000], np.uint32).view(np.float32)
    M = np.zeros((rows, K), np.float32)
    M[np.arange(rows), np.arange(rows) % K] = v
    return M


def _same(out, want):
    """Bit for bit up to the sign of zero; NaN where and only where expected."""
    nan = np.isnan(want)
    return np.array_equal(np.isnan(out), nan) and np.array_equal(out[~nan], want[~nan])


@pytest.mark.gpu
@pytest.mark.parametrize("K,kernel", [(128, "tc32"), (256, "tc32"), (96, "ffma")])
def test_one_k_products_bit_exact(ops, K, kernel):
    """Non-finite, subnormal, tiny and huge operands through each kernel, against the host model bit for bit.  3xTF32: a row
    holding +-inf or NaN gives a NaN row (``lo = inf - inf``), subnormal operands and products are kept.  FFMA: IEEE fp32."""
    M = N = 256
    assert _probe(ops, M, N, K) == kernel
    A, Bm = _one_k_operands(M, K, 1), _one_k_operands(N, K, 2)
    out = ops.gemm_nt(torch.as_tensor(A, device="cuda")[None], torch.as_tensor(Bm, device="cuda")[None])[0].cpu().numpy()
    if kernel == "ffma":
        assert _same(out, T.ffma_gemm_nt(A, Bm))
        return
    want = T.gemm_nt(A, Bm)
    flushed = T.gemm_nt(A, Bm, ftz_products=True)
    assert not _same(want, flushed)  # the data has subnormal products: the test tells the two apart
    assert _same(out, want), ("flushes subnormal products" if _same(out, flushed) else "differs from the model",
                              int((out != want).sum()))
    assert np.isnan(out[:4]).all() and np.isnan(out[:, :4]).all()
    ffma = T.ffma_gemm_nt(A, Bm)
    assert np.isinf(ffma[:2, :2]).any()  # where FFMA gives +-inf the tensor-core kernel gives NaN


def _randn(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g)


@pytest.mark.gpu
def test_tc_alpha_beta_and_beta0_over_nan(ops):
    Bn, M, N, K = 2, 256, 384, 512
    assert _probe(ops, M, N, K, Bn) == "tc32"
    A, Bm, C = _randn((Bn, M, K), 1), _randn((Bn, N, K), 2), _randn((Bn, M, N), 3)
    Ad, Bd, Cd = A.double(), Bm.double(), C.double()
    S = Ad.abs() @ Bd.abs().transpose(1, 2)
    ref = 0.5 * Cd - 1.25 * (Ad @ Bd.transpose(1, 2))
    out = ops.gemm_nt(A, Bm, C.clone(), alpha=-1.25, beta=0.5)
    assert ((out.double() - ref).abs() <= tc_bound(K, -1.25, S, ref, 0.5, Cd.abs())).all()
    out = ops.gemm_nt(A, Bm, torch.full_like(C, float("nan")), alpha=-0.75, beta=0.0)
    ref = -0.75 * (Ad @ Bd.transpose(1, 2))
    assert out.isfinite().all()
    assert ((out.double() - ref).abs() <= tc_bound(K, -0.75, S, ref)).all()


@pytest.mark.gpu
def test_tc_strided_batches_with_an_unusual_batch_stride(ops):
    """Offset views whose batch stride is not ``rows * ld`` (the TMA descriptors take the batch stride as their third
    dimension's stride), C likewise."""
    Bn, M, N, K, ld, ldc = 3, 256, 384, 256, 320, 448
    a_bs, b_bs, c_bs = M * ld + 132, N * ld + 36, M * ldc + 68
    bufA, bufB = _randn((Bn * a_bs + 1024,), 4), _randn((Bn * b_bs + 1024,), 5)
    bufC = _randn((Bn * c_bs + 1024,), 6)
    A = bufA.as_strided((Bn, M, K), (a_bs, ld, 1), 64)
    Bm = bufB.as_strided((Bn, N, K), (b_bs, ld, 1), 32)
    C = bufC.as_strided((Bn, M, N), (c_bs, ldc, 1), 16)
    A_, B_ = A.contiguous(), Bm.contiguous()
    assert _probe(ops, M, N, K, Bn) == "tc32"
    before = bufC.clone()
    Cd = C.double()
    ops.gemm_nt(A, Bm, C, alpha=1.5, beta=-0.5)
    ref = -0.5 * Cd + 1.5 * (A_.double() @ B_.double().transpose(1, 2))
    S = A_.double().abs() @ B_.double().abs().transpose(1, 2)
    assert ((C.double() - ref).abs() <= tc_bound(K, 1.5, S, ref, 0.5, Cd.abs())).all()
    touched = torch.zeros_like(bufC, dtype=torch.bool)
    touched.as_strided((Bn, M, N), (c_bs, ldc, 1), 16).fill_(True)
    assert torch.equal(bufC[~touched], before[~touched])  # nothing outside the view is written


def _lower_mask(M, N):
    tr = torch.arange(M, device="cuda")[:, None] // 128
    tc = torch.arange(N, device="cuda")[None, :] // 128
    return tc <= tr


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(640, 384, 256), (128 * 515, 256, 128)], ids=["lower_m_gt_n", "tall_ragged_swizzle"])
def test_tc_lower_sentinel_and_tall(ops, M, N, K):
    """Lower mode with a sentinel above the diagonal tiles, M > N; and a tall product: 515 tile rows (M > 65535), so the
    tile swizzle (groups of 8 tile rows) runs over 65 groups and ends on a ragged one of 3.  Both modes on both shapes."""
    assert _probe(ops, M, N, K) == "tc32" and _probe(ops, M, N, K, lower=True) == "tc32"
    A, Bm, C = _randn((1, M, K), M), _randn((1, N, K), N), _randn((1, M, N), K)
    Ad, Bd, Cd = A.double(), Bm.double(), C.double()
    prod = Ad @ Bd.transpose(1, 2)
    S = Ad.abs() @ Bd.abs().transpose(1, 2)
    out = ops.gemm_nt(A, Bm, C.clone(), alpha=-1.0, beta=1.0)
    ref = Cd - prod
    assert ((out.double() - ref).abs() <= tc_bound(K, -1.0, S, ref, 1.0, Cd.abs())).all()
    mask = _lower_mask(M, N)
    Cs = torch.where(mask, C, torch.full_like(C, 31.25))
    out = ops.gemm_nt(A, Bm, Cs.clone(), alpha=-1.0, beta=1.0, lower=True)
    assert torch.equal(out[:, ~mask], Cs[:, ~mask])
    ok = (out.double() - ref).abs() <= tc_bound(K, -1.0, S, ref, 1.0, Cd.abs())
    assert ok[:, mask].all()


#: the normwise error ``max |err| / max S`` of the 3xTF32 kernel per K on these seeds (random normal operands), measured on an
#: H100 80GB HBM3 at 700 W: it grows like sqrt(K), far inside the worst-case bound.  The test allows twice that (the numbers are
#: recorded next to gpk_gemm_nt_f32 in include/gpk.h).
TC_MEASURED = {4096: 3.1e-6, 8192: 4.3e-6, 16384: 6.1e-6}


@pytest.mark.gpu
@pytest.mark.parametrize("K", [4096, 8192, 16384, 8208])
def test_long_k_per_entry(ops, K):
    """Long reductions: per-entry bound on both kernels (K = 8208 is not a multiple of 32: FFMA), and the measured growth of
    the 3xTF32 kernel's error with K."""
    M = N = 256
    kernel = _probe(ops, M, N, K)
    assert kernel == ("ffma" if K % 32 else "tc32")
    A, Bm = _randn((1, M, K), K), _randn((1, N, K), K + 1)
    Ad, Bd = A.double(), Bm.double()
    ref = Ad @ Bd.transpose(1, 2)
    S = Ad.abs() @ Bd.abs().transpose(1, 2)
    err = (ops.gemm_nt(A, Bm).double() - ref).abs()
    bound = (tc_bound if kernel == "tc32" else ffma_bound)(K, 1.0, S, ref)
    assert (err <= bound).all()
    normwise = err.max().item() / S.max().item()
    print(f"K={K} {kernel}: max|err|/max S = {normwise:.3e}, max err/S per entry = {(err / S).max().item():.3e}")
    if kernel == "tc32":
        assert normwise <= 2 * TC_MEASURED[K], normwise


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["tc32", "ffma"])
def test_non_finite_rows(ops, kernel):
    """Random operands with a NaN and a +inf in two rows of A and a -inf in a row of B.  FFMA: what fp64 gives (NaN or +-inf
    per entry).  3xTF32: the row of A (column of B) holding the NaN or infinity is NaN throughout, the rest is untouched by
    it (include/gpk.h)."""
    M, N, K = 256, 256, (128 if kernel == "tc32" else 96)
    assert _probe(ops, M, N, K) == kernel
    A, Bm = _randn((1, M, K), 7), _randn((1, N, K), 8)
    A[0, 3, 5], A[0, 7, 9], Bm[0, 11, 40] = float("nan"), float("inf"), float("-inf")
    out = ops.gemm_nt(A, Bm).double()[0].cpu()
    Ad, Bd = A[0].double().cpu().numpy(), Bm[0].double().cpu().numpy()
    ref = torch.as_tensor((Ad[:, None, :] * Bd[None, :, :]).sum(-1))  # IEEE products and sums, no BLAS
    bad = torch.zeros(M, N, dtype=torch.bool)
    bad[[3, 7], :] = True
    bad[:, 11] = True
    if kernel == "tc32":
        assert out[bad].isnan().all()
    else:
        assert torch.equal(out[bad].isnan(), ref[bad].isnan())
        assert torch.equal(out[bad][ref[bad].isinf()], ref[bad][ref[bad].isinf()])
        assert ref[bad].isinf().any()
    S = torch.as_tensor(np.abs(Ad) @ np.abs(Bd).T)
    bound = (tc_bound if kernel == "tc32" else ffma_bound)(K, 1.0, S, ref)
    assert ((out - ref).abs() <= bound)[~bad].all()


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["tc32", "ffma"])
def test_extreme_row_magnitudes(ops, kernel):
    """Rows of A scaled by 2^-70 .. 2^60 and of B by 2^-70 .. 2^50: products from deep in the subnormal range to 2^110, per
    entry against fp64 with the subnormal term of the bound."""
    M, N, K = 384, 256, (256 if kernel == "tc32" else 144)
    assert _probe(ops, M, N, K) == kernel
    g = torch.Generator(device="cuda").manual_seed(9)
    ea = torch.randint(-70, 61, (1, M, 1), device="cuda", generator=g).float()
    eb = torch.randint(-70, 51, (1, N, 1), device="cuda", generator=g).float()
    A, Bm = _randn((1, M, K), 10) * torch.exp2(ea), _randn((1, N, K), 11) * torch.exp2(eb)
    Ad, Bd = A.double(), Bm.double()
    ref = Ad @ Bd.transpose(1, 2)
    S = Ad.abs() @ Bd.abs().transpose(1, 2)
    out = ops.gemm_nt(A, Bm).double()
    assert out.isfinite().all()
    bound = (tc_bound if kernel == "tc32" else ffma_bound)(K, 1.0, S, ref, eta=ETA)
    assert ((out - ref).abs() <= bound).all()
    assert (ref.abs() < 2.0**-126).any() and (ref.abs() > 2.0**100).any()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [513, 640, 4096])
def test_tf32x3_fp64_cholesky(ops, n, monkeypatch):
    """``B.precision = "tf32x3"``: the fp64 Cholesky's trailing updates on ``gemm_nt_f32_tc_kernel<double>``, from n_pad > 512
    (n = 513: a single row past the first panel).  L against torch's fp64 Cholesky with the fp32-level bounds of
    ``tests/test_cholesky_schedules.py`` (u = 2^-22), and different bits from the native fp64 factor (the path was taken)."""
    from stheno_b200 import B
    from tests.test_cholesky_schedules import spd

    A = spd(1, n, n)
    monkeypatch.setattr(B, "precision", "tf32x3")
    L = ops.chol_from_dense(A).check().L()
    monkeypatch.setattr(B, "precision", "fp64")
    L64 = ops.chol_from_dense(A).check().L()
    assert not torch.equal(L, L64)
    u = 2.0**-22
    d = A.diagonal(dim1=1, dim2=2).sqrt()
    back = (A - L @ L.transpose(1, 2)).abs() / (d[:, :, None] * d[:, None, :])
    assert back.max().item() <= 4 * n * u, back.max().item()
    Lref = torch.linalg.cholesky(A)
    assert ((L - Lref).abs().max() / Lref.abs().max()).item() <= 200 * n * u


# ---- C. the fp32 Cholesky and its solves at the benchmarked shape --------------------------------------------------------


def _config3_problem(ops, batch, n, seed):
    """EQ kernel matrices of ``batch`` sets of n standard-normal points in 8 dimensions, noise 0.1 and jitter 1e-6 on the
    diagonal (BASELINE config 3), in fp32, and one right-hand side per member."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(batch, n, 8, device="cuda", generator=g)
    y = torch.randn(batch, 1, n, device="cuda", generator=g)
    flat = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    K = ops.kernel_matrix(flat, x[None], noise_scalar=0.1, jitter=1e-6)
    return K, y


@pytest.mark.gpu
@pytest.mark.parametrize("batch,n", [(64, 2048), (8, 2047), (8, 2049), (1, 8192)])
def test_fp32_cholesky_every_member(ops, batch, n):
    K, y = _config3_problem(ops, batch, n, n)
    ch = ops.chol_from_dense(K, rhs_t=y).check()
    g = torch.Generator(device="cuda").manual_seed(1)
    R = torch.randn(batch, 130, n, device="cuda", generator=g)
    X = ch.half_solve(R).double()  # X L^T = R
    buf = ch.new_rows(130)
    buf[:, :130, :n] = R
    Xt = ch.solve_rows_t_(buf)[:, :130, :n].double()  # Xt L = R
    logdet32, lp32 = ch.logdet.double(), ch.logpdf()[:, 0].double()
    h = ch.rhs_half()[:, 0].double()
    Lall = ch.L()
    for b in range(batch):
        Kd, L = K[b].double(), Lall[b].double()
        E = Kd - L @ L.T
        back = E.abs().max().item() / (n * U * Kd.abs().max().item())
        assert back <= 4, (b, back)
        aL = L.abs()
        # residuals of the fused forward solve and of the two separate triangular solves
        r = y[b, 0].double() - L @ h[b]
        assert (r.abs() <= 4 * n * U * (aL @ h[b].abs())).all(), b
        assert ((R[b].double() - X[b] @ L.T).abs() <= 4 * n * U * (X[b].abs() @ aL.T)).all(), b
        assert ((R[b].double() - Xt[b] @ L).abs() <= 4 * n * U * (Xt[b].abs() @ aL)).all(), b
        # logdet and log-pdf against fp64 values of the same fp32 matrix, within the first-order effect of E
        L64 = torch.linalg.cholesky(Kd)
        Kinv = torch.cholesky_inverse(L64)
        alpha = Kinv @ y[b, 0].double()
        ld64 = 2 * L64.diagonal().log().sum().item()
        quad64 = (y[b, 0].double() @ alpha).item()
        lp64 = -0.5 * (ld64 + n * math.log(2 * math.pi) + quad64)
        eps = E.abs().max().item()
        ld_bound = 1.5 * eps * Kinv.abs().sum().item() + 4 * U * abs(ld64)
        assert abs(logdet32[b].item() - ld64) <= ld_bound, (b, logdet32[b].item(), ld64, ld_bound)
        Linv_r = torch.linalg.solve_triangular(L, r[:, None], upper=False)[:, 0]
        quad_bound = 1.5 * eps * alpha.abs().sum().item() ** 2 + 2 * h[b].norm().item() * Linv_r.norm().item() + Linv_r.norm().item() ** 2
        lp_bound = 0.5 * (ld_bound + quad_bound) + 4 * U * (abs(lp64) + abs(ld64) + n * math.log(2 * math.pi) + quad64)
        assert abs(lp32[b].item() - lp64) <= lp_bound, (b, lp32[b].item(), lp64, lp_bound)


# ---- D. the fp32 row reductions --------------------------------------------------------------------------------------


def _rows(n_cols, seed):
    """Two rows: ``1`` followed by ``2^-13`` (each squared term is below half an ulp of 1: an fp32 accumulator that starts at
    1 loses all of them) and a random normal row."""
    adv = torch.full((n_cols,), 2.0**-13, device="cuda")
    adv[0] = 1.0
    return torch.stack([adv, _randn((n_cols,), seed)])


@pytest.mark.gpu
@pytest.mark.parametrize("n_cols", [128, 65536, 262144])
def test_row_dot_sq_fp32_sums_in_fp64(ops, n_cols):
    V = _rows(n_cols, n_cols)[None]
    b = _randn((1, n_cols), n_cols + 1)
    dot, sq = ops.row_dot_sq(V, 2, n_cols, b)
    Vd, bd = V.double(), b.double()
    sq_ref = (Vd * Vd).sum(-1)
    dot_ref = (Vd * bd[:, None, :]).sum(-1)
    sq_err = ((sq.double() - sq_ref).abs() / (U * sq_ref)).max().item()
    dot_err = ((dot.double() - dot_ref).abs() / (U * (Vd * bd[:, None, :]).abs().sum(-1))).max().item()
    assert sq_err <= 2, sq_err  # errors in units of u: one final rounding of an fp64 sum
    assert dot_err <= 2, dot_err


@pytest.mark.gpu
@pytest.mark.parametrize("n_cols", [128, 65536, 262144])
def test_logpdf_finish_fp32_sums_in_fp64(ops, n_cols):
    """``gpk_logpdf_finish_f32`` on constructed rows, ``n = 0`` and ``logdet = -1`` so that the output is the quadratic form's
    excess over 1 and every lost term shows."""
    rows = _rows(n_cols, n_cols + 2)[None]
    logdet = torch.full((1,), -1.0, device="cuda")
    out = torch.empty(1, 2, device="cuda")
    ops.check(ops._fn("gpk_logpdf_finish", torch.float32)(ops._ptr(rows), rows.stride(1), rows.stride(0), 0, n_cols, 2,
                                                          ops._ptr(logdet), ops._ptr(out), 1, ops._stream()),
              "gpk_logpdf_finish")
    ref = -0.5 * (-1.0 + (rows.double() ** 2).sum(-1))
    err = ((out.double() - ref).abs() / (U * ref.abs())).max().item()
    assert err <= 2, err
    # with n: -0.5 (logdet + n log 2 pi + sum) rounded once
    out_n = torch.empty(1, 2, device="cuda")
    ops.check(ops._fn("gpk_logpdf_finish", torch.float32)(ops._ptr(rows), rows.stride(1), rows.stride(0), n_cols, n_cols, 2,
                                                          ops._ptr(logdet), ops._ptr(out_n), 1, ops._stream()),
              "gpk_logpdf_finish")
    ref_n = ref - 0.5 * n_cols * math.log(2 * math.pi)
    assert ((out_n.double() - ref_n).abs() <= 2 * U * ref_n.abs()).all()


@pytest.mark.gpu
def test_fp32_posterior_variance_on_the_training_inputs(ops):
    """End to end at n = 16384, noise 1e-3: the fp32 exact-posterior variance at test points placed on training inputs (the
    variance is the small difference of two values near 1) against the fp64 posterior.  With ``v`` the fp32 solved rows and
    ``w`` the fp64 ones, ``var32 - var64 = -(sq32 - |v|^2) - (|v|^2 - |w|^2)``: the bound is the second term, which the fp32
    solve alone makes, plus one rounding of the sum and of the subtraction."""
    n, m, d = 16384, 512, 4
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(n, d, device="cuda", generator=g)
    flat = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    xg, xsg = x[None, None], x[None, None, :m]
    ch = ops.chol_from_kernel(flat, xg, noise_scalar=1e-3).check()
    _, sq = ops.posterior_marginals(flat, xsg, xg, ch)
    var32 = (ops.kernel_diag(flat, xsg)[0] - sq).double()
    V = ch.solve_rows_(ops.kernel_rows_padded(flat, xsg, xg, ch))
    assert torch.equal(ops.row_dot_sq(V, m, ch.n_pad)[1][0], sq)  # the same two steps
    v = V[0, :m, :n].double()
    del V, ch
    xg64, xsg64 = xg.double(), xsg.double()
    L64 = torch.linalg.cholesky(ops.kernel_matrix(flat, xg64, noise_scalar=1e-3)[0])
    w = torch.linalg.solve_triangular(L64, ops.kernel_matrix(flat, xg64, xsg64, same=False)[0], upper=False).T
    var64 = ops.kernel_diag(flat, xsg64)[0] - (w * w).sum(-1)
    del L64
    sq_v = (v * v).sum(-1)
    bound = ((v - w) * (v + w)).sum(-1).abs() + 2 * U * sq_v + U * var32.abs()
    assert ((var32 - var64).abs() <= bound).all()
    assert (var64 < 2e-3).all()  # near the data: the variance is at the noise level
