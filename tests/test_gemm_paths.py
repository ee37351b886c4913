"""The fp64 GEMM ``C = beta C + alpha A B^T`` on every launch path, against a NumPy fp64 reference:

  v2<16,4>    K % 32 != 0                     (generic entry, native fp64)
  v2<32,3>    K < 512, K % 32 == 0
  v3          K >= 512, K % 32 == 0
  emulated    generic entry under B.precision = "auto", M N K >= 1.5e9 (int8-slice emulation, 8 slices)
  oz5 .. oz8  gpk_gemm_nt_f64_oz called directly with 5 .. 8 slices

Every call checks the path it took through the in-situ launch profile (kind 0 = the v3 kernel, kind 1 = the emulation;
v2 launches are not profiled).  Cases: alpha / beta, beta = 0 over a NaN-filled C, batches of strided offset views, lower
mode with a sentinel above the diagonal tiles, a tall product (M > 65535) with a general beta, NaN / inf rows and rows of
extreme magnitude."""
import contextlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0**-53
# emulation bound per slice count, relative to rowmax(A) colmax(B) sqrt(K) (as in tests/test_emulation.py)
TOL = {5: 2e-9, 6: 2e-11, 7: 2e-13, 8: 5e-15}

#: path -> (M, N, K, slices of the emulation or 0 for native fp64)
PATHS = {
    "v2_16x4": (256, 256, 144, 0),
    "v2_32x3": (256, 128, 256, 0),
    "v3_k512": (256, 256, 512, 0),
    "v3_k1024": (128, 256, 1024, 0),
    "emulated": (1152, 1024, 1280, 8),
    "oz5": (256, 192, 384, 5),
    "oz6": (256, 192, 384, 6),
    "oz7": (256, 192, 384, 7),
    "oz8": (256, 192, 384, 8),
}


@pytest.fixture(scope="module")
def ops():
    from stheno_b200 import ops

    return ops


@contextlib.contextmanager
def _precision(mode):
    from stheno_b200 import B

    before = B.precision
    B.precision = mode
    try:
        yield
    finally:
        B.precision = before


def _direct(path):
    return path.startswith("oz")


def gemm(ops, path, A, Bm, C, alpha, beta, lower=False):
    """``C`` ``[batch, M, N]`` (views allowed) <- beta C + alpha A Bm^T on ``path``; asserts that ``path`` ran."""
    ops.gemm_profile(True)
    try:
        if _direct(path):
            assert A.shape[0] == 1
            ops.gemm_nt_oz(A[0], Bm[0], C[0], alpha=alpha, beta=beta, lower=lower, slices=PATHS[path][3])
        else:
            with _precision("auto" if path == "emulated" else "fp64"):
                ops.gemm_nt(A, Bm, C, alpha=alpha, beta=beta, lower=lower)
        n_v3 = ops.gemm_profile_read(0)[2]
        n_oz = ops.gemm_profile_read(1)[2]
    finally:
        ops.gemm_profile(False)
    if path.startswith("v2"):
        assert (n_v3, n_oz) == (0, 0), (path, n_v3, n_oz)
    elif path.startswith("v3"):
        assert (n_v3, n_oz) == (1, 0), (path, n_v3, n_oz)
    else:
        assert n_v3 == 0 and n_oz >= 1, (path, n_v3, n_oz)
    return C


def bound(path, A, Bm, C0, alpha, beta, ref):
    """Elementwise error bound: K u |alpha| |A| |B|^T for native fp64, the slicing bound for the emulation; plus the
    rounding of the result and of beta C0."""
    K = A.shape[-1]
    S = PATHS[path][3]
    with np.errstate(over="ignore"):
        if S == 0:
            prod = 2 * K * U * abs(alpha) * (np.abs(A) @ np.abs(np.swapaxes(Bm, -1, -2)))
        else:
            scale = np.abs(A).max(-1)[..., :, None] * np.abs(Bm).max(-1)[..., None, :] * np.sqrt(K)
            prod = TOL[S] * abs(alpha) * scale
        return prod + 4 * U * (np.abs(ref) + np.abs(beta * C0)) + 2.0**-1070


def _rand(rng, *shape):
    return rng.standard_normal(shape)


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda")


def _ref(A, Bm, C0, alpha, beta):
    with np.errstate(invalid="ignore", over="ignore"):
        p = alpha * (A @ np.swapaxes(Bm, -1, -2))
        return p if beta == 0.0 else beta * C0 + p


@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (-1.0, 1.0), (-1.5, 0.5), (-1.0 / 3.0, 0.0)])
@pytest.mark.parametrize("path", list(PATHS))
def test_alpha_beta(ops, path, alpha, beta):
    M, N, K, _ = PATHS[path]
    rng = np.random.default_rng(M + N + K)
    A = _rand(rng, 1, M, K) * np.exp(2 * rng.standard_normal((1, M, 1)))
    Bm = _rand(rng, 1, N, K)
    C0 = _rand(rng, 1, M, N)
    got = gemm(ops, path, _dev(A), _dev(Bm), _dev(C0), alpha, beta).cpu().numpy()
    ref = _ref(A, Bm, C0, alpha, beta)
    err = np.abs(got - ref) / bound(path, A, Bm, C0, alpha, beta, ref)
    assert err.max() <= 1.0, err.max()


@pytest.mark.parametrize("path", list(PATHS))
def test_beta_zero_ignores_nan_c(ops, path):
    M, N, K, _ = PATHS[path]
    rng = np.random.default_rng(1)
    A, Bm = _rand(rng, 1, M, K), _rand(rng, 1, N, K)
    C = torch.full((1, M, N), float("nan"), device="cuda", dtype=torch.float64)
    got = gemm(ops, path, _dev(A), _dev(Bm), C, -0.75, 0.0).cpu().numpy()
    ref = -0.75 * (A @ Bm.transpose(0, 2, 1))
    assert np.isfinite(got).all()
    assert (np.abs(got - ref) <= bound(path, A, Bm, 0.0, -0.75, 0.0, ref)).all()


@pytest.mark.parametrize("path", list(PATHS))
def test_batched_strided_views(ops, path):
    """Offset views into larger buffers (row strides != K, N), batch 3 on the native paths (the emulation serves single
    problems: batch 1 there); what lies outside the view of C stays untouched."""
    M, N, K, _ = PATHS[path]
    batch = 1 if PATHS[path][3] else 3
    rng = np.random.default_rng(2)
    Abuf, Bbuf = _dev(_rand(rng, batch, M + 128, K + 48)), _dev(_rand(rng, batch, N + 64, K + 32))
    Cbuf = _dev(_rand(rng, batch, M + 128, N + 96))
    A, Bm, C = Abuf[:, 64 : 64 + M, 16 : 16 + K], Bbuf[:, 32 : 32 + N, 8 : 8 + K], Cbuf[:, 128 : 128 + M, 32 : 32 + N]
    An, Bn, Cn, Cbuf0 = A.cpu().numpy(), Bm.cpu().numpy(), C.cpu().numpy(), Cbuf.clone()
    gemm(ops, path, A, Bm, C, -1.5, 0.5)
    ref = _ref(An, Bn, Cn, -1.5, 0.5)
    assert (np.abs(C.cpu().numpy() - ref) <= bound(path, An, Bn, Cn, -1.5, 0.5, ref)).all()
    outside = torch.ones_like(Cbuf, dtype=torch.bool)
    outside[:, 128 : 128 + M, 32 : 32 + N] = False
    assert torch.equal(Cbuf[outside], Cbuf0[outside])


LOWER_SHAPES = {"emulated": (1536, 1024, 1024)}


@pytest.mark.parametrize("beta", [0.0, 1.0, 0.5])
@pytest.mark.parametrize("path", list(PATHS))
def test_lower_mode_sentinel(ops, path, beta):
    """lower = 1, M > N: the tiles that touch the lower triangle (row i: columns below 128 (i // 128 + 1)) get
    beta C + alpha A B^T; every element above them keeps its sentinel bit for bit, whatever beta."""
    M, N, K, _ = PATHS[path]
    M, N, K = LOWER_SHAPES.get(path, (M + 128, N, K))
    rng = np.random.default_rng(3)
    A, Bm, C0 = _rand(rng, 1, M, K), _rand(rng, 1, N, K), _rand(rng, 1, M, N)
    i, j = np.arange(M)[:, None], np.arange(N)[None, :]
    touched = j < 128 * (i // 128 + 1)
    C0 = np.where(touched, C0, 31.25)
    got = gemm(ops, path, _dev(A), _dev(Bm), _dev(C0), -1.0, beta, lower=True).cpu().numpy()
    ref = _ref(A, Bm, C0, -1.0, beta)
    assert np.array_equal(got[0][~touched], C0[0][~touched])
    ok = np.abs(got - ref) <= bound(path, A, Bm, C0, -1.0, beta, ref)
    assert ok[0][touched].all()


@pytest.mark.parametrize("path", ["emulated", "oz8"])
def test_tall_product_general_beta(ops, path):
    """M = 65664 rows (more than a CUDA grid's y extent) with beta = 0.5 on the emulated paths: computed, not refused."""
    M, N, K = 65664, 256, 256
    rng = np.random.default_rng(4)
    A, Bm, C0 = _rand(rng, 1, M, K), _rand(rng, 1, N, K), _rand(rng, 1, M, N)
    got = gemm(ops, path, _dev(A), _dev(Bm), _dev(C0), 2.0, 0.5).cpu().numpy()
    ref = _ref(A, Bm, C0, 2.0, 0.5)
    assert (np.abs(got - ref) <= bound(path, A, Bm, C0, 2.0, 0.5, ref)).all()


@pytest.mark.parametrize("path", list(PATHS))
def test_nonfinite_rows(ops, path):
    """NaN, +inf and -inf in chosen rows of A and of B: wherever the fp64 product is non-finite the result is non-finite
    (NaN may stand for +-inf), and every other element is bit-identical to the same call with those rows set to zero."""
    M, N, K, _ = PATHS[path]
    rng = np.random.default_rng(5)
    A, Bm, C0 = _rand(rng, 1, M, K), _rand(rng, 1, N, K), _rand(rng, 1, M, N)
    bad_a, bad_b = [3, M // 2 + 2, M - 1], [0, 77, N - 2]
    A[0, 3, 5], A[0, M // 2 + 2, K - 1], A[0, M - 1, 40] = np.nan, np.inf, -np.inf
    Bm[0, 0, 0], Bm[0, 77, 17], Bm[0, N - 2, K - 3] = -np.inf, np.nan, np.inf
    got = gemm(ops, path, _dev(A), _dev(Bm), _dev(C0), -1.0, 0.5).cpu().numpy()
    ref = _ref(A, Bm, C0, -1.0, 0.5)
    A0, B0 = A.copy(), Bm.copy()
    A0[0, bad_a], B0[0, bad_b] = 0.0, 0.0
    clean = gemm(ops, path, _dev(A0), _dev(B0), _dev(C0), -1.0, 0.5).cpu().numpy()
    nonfinite = ~np.isfinite(ref)
    assert nonfinite[0][bad_a].all() and nonfinite[0][:, bad_b].all()
    assert not np.isfinite(got[nonfinite]).any()
    assert np.array_equal(got[~nonfinite], clean[~nonfinite])


EXTREME_K = [-1070, -1020, -1000, -980, 980, 1000, 1020]


@pytest.mark.parametrize("alpha", [1.0, -1.0 / 3.0])
@pytest.mark.parametrize("k", EXTREME_K)
@pytest.mark.parametrize("path", list(PATHS))
def test_extreme_row_magnitudes(ops, path, k, alpha):
    """A rows scaled by 2^k, B rows by 2^-k (at most 2^1020, so that B stays finite): products of O(1) from operands that
    range from subnormal to near overflow.  The emulation meets its rowmax colmax sqrt(K) bound."""
    M, N, K, _ = PATHS[path]
    rng = np.random.default_rng(abs(k))
    A = np.ldexp(_rand(rng, 1, M, K), k)
    Bm = np.ldexp(_rand(rng, 1, N, K), min(-k, 1020))
    C0 = np.zeros((1, M, N))
    got = gemm(ops, path, _dev(A), _dev(Bm), _dev(C0), alpha, 0.0).cpu().numpy()
    ref = _ref(A, Bm, C0, alpha, 0.0)
    err = np.abs(got - ref) / bound(path, A, Bm, C0, alpha, 0.0, ref)
    assert err.max() <= 1.0, err.max()
