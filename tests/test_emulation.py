"""fp64 emulated on the int8 tensor cores (wgmma .s32.s8.s8, error-free 7-bit slicing, exact int32 products):
the GEMM kernel against torch fp64, and the factorisation / solves that use it against the native fp64 (DMMA) path and
the NumPy oracle.  ``B.precision = "auto"`` (the default) means 7 slices."""
import numpy as np
import pytest
import torch

from oracle import gp_oracle as O

pytestmark = pytest.mark.gpu

from tests._oz_model import gemm as oz_model_gemm  # noqa: E402  (NumPy integer model of the kernel)


@pytest.fixture(scope="module")
def S():
    import stheno_b200.torch as S

    return S


@pytest.fixture(scope="module")
def ops():
    from stheno_b200 import ops

    return ops


# measured: 6 slices 3e-12 .. 4.4e-12, 7 slices 2.6e-14 .. 3.8e-14, 8 slices 5e-16 .. 8e-16 (Frobenius-relative)
TOL = {5: 2e-9, 6: 2e-11, 7: 2e-13, 8: 5e-15}


@pytest.mark.parametrize("slices", [5, 6, 7, 8])
@pytest.mark.parametrize("M,N,K", [(128, 64, 128), (384, 320, 640), (1024, 1024, 512), (256, 512, 4096)])
def test_gemm_oz_vs_torch(ops, slices, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M + N + K + slices)
    # rows with very different magnitudes: the per-row power-of-two scaling has to cope
    A = torch.randn(M, K, device="cuda", dtype=torch.float64, generator=g)
    A *= torch.exp(3 * torch.randn(M, 1, device="cuda", dtype=torch.float64, generator=g))
    Bm = torch.randn(N, K, device="cuda", dtype=torch.float64, generator=g)
    C0 = torch.randn(M, N, device="cuda", dtype=torch.float64, generator=g)
    for alpha, beta in ((1.0, 0.0), (-1.0, 1.0), (-1.5, 0.5)):
        ref = beta * C0 + alpha * (A @ Bm.T)
        C = ops.gemm_nt_oz(A, Bm, C0.clone(), alpha=alpha, beta=beta, slices=slices)
        # error model: slicing error relative to the row maxima, accumulated over K
        scale = A.abs().amax(1, keepdim=True) * Bm.abs().amax(1)[None, :] * np.sqrt(K)
        # (+ the fp64 rounding of the result itself, which matters for the 8-slice variant)
        bound = TOL[slices] * scale + 4e-16 * (ref.abs() + (beta * C0).abs())
        assert ((C - ref).abs() <= bound).all().item(), ((alpha, beta), ((C - ref).abs() / bound).max().item())


def test_gemm_oz_exact_on_integers(ops):
    """Small integers fit the first slices exactly: the result must be bit-identical to the exact product."""
    g = torch.Generator(device="cuda").manual_seed(0)
    A = torch.randint(-1000, 1000, (256, 256), device="cuda", generator=g).double()
    Bm = torch.randint(-1000, 1000, (128, 256), device="cuda", generator=g).double()
    C = ops.gemm_nt_oz(A, Bm, slices=7)
    assert torch.equal(C, A @ Bm.T)


def test_gemm_oz_lower_and_zero_rows(ops):
    g = torch.Generator(device="cuda").manual_seed(3)
    P = torch.randn(512, 256, device="cuda", dtype=torch.float64, generator=g)
    P[100:140] = 0.0  # all-zero rows (identity padding produces them)
    C0 = torch.randn(512, 512, device="cuda", dtype=torch.float64, generator=g)
    mask = torch.ones(512, 512, device="cuda", dtype=torch.bool).tril()
    above = torch.arange(512, device="cuda")[None, :] >= 128 * (torch.arange(512, device="cuda")[:, None] // 128 + 1)
    for beta in (1.0, 0.5):
        C = ops.gemm_nt_oz(P, P, C0.clone(), alpha=-1.0, beta=beta, lower=True, slices=7)
        ref = beta * C0 - P @ P.T
        assert ((C - ref)[mask].abs().max() / ref.abs().max()).item() < 1e-13
        # tiles strictly above the diagonal (128 x 64 granularity) are not touched, whatever beta
        assert torch.equal(C[above], C0[above])


@pytest.mark.parametrize("n,k", [(2048, 1), (3000, 3), (4480, 1)])
def test_emulated_cholesky_vs_native(S, ops, n, k):
    rng = np.random.default_rng(n)
    x = torch.as_tensor(rng.uniform(0, 4, (n, 3)), device="cuda")
    y = torch.as_tensor(rng.standard_normal((n, k)), device="cuda")
    f = S.GP(2.0 * S.EQ().stretch(0.7) + 0.5 * S.Matern32())
    out = {}
    before = S.B.precision
    try:
        for prec in ("fp64", "int8x6", "auto", "int8x8"):
            S.B.precision = prec
            out[prec] = f(x, 0.05).logpdf(y).cpu().numpy().ravel()
    finally:
        S.B.precision = before
    ref = out["fp64"]
    assert np.max(np.abs(out["auto"] - ref) / np.abs(ref)) < 1e-11
    assert np.max(np.abs(out["int8x8"] - ref) / np.abs(ref)) < 1e-12
    assert np.max(np.abs(out["int8x6"] - ref) / np.abs(ref)) < 1e-7
    assert not np.array_equal(out["int8x6"], ref)  # it really took the emulated path


def test_emulated_logpdf_and_posterior_vs_oracle(S):
    """The default path at a size where the emulation is active (n_pad >= 2048) against the NumPy oracle: the 1e-10 bar."""
    rng = np.random.default_rng(11)
    n, m, d = 2500, 300, 4
    x = rng.uniform(0, 3, (n, d))
    xs = rng.uniform(0, 3, (m, d))
    y = np.sin(x.sum(1)) + 0.1 * rng.standard_normal(n)
    spec = ("sum", ("stretched", 0.8, ("eq",)), ("scaled", 0.3, ("stretched", 2.0, ("matern52",))))
    assert S.B.precision == "auto"
    f = S.GP(S.EQ().stretch(0.8) + 0.3 * S.Matern52().stretch(2.0))
    lp = f(x, 0.2).logpdf(y)
    want = float(np.ravel(O.fdd_logpdf(spec, x, 0.2, y))[0])
    assert abs(float(lp) - want) / abs(want) < 1e-10
    post = f | (f(x, 0.2), y)
    mean, var = post(xs).marginals()
    mo, vo = O.posterior_marginals(spec, x, 0.2, y, xs)
    assert np.max(np.abs(np.ravel(mean) - np.ravel(mo))) < 1e-9
    assert np.max(np.abs(np.ravel(var) - np.ravel(vo))) < 1e-9


def test_emulated_solves_vs_native(S):
    """Posterior with enough test points that the triangular solves' GEMMs go through the emulation."""
    rng = np.random.default_rng(5)
    n, m = 4096, 1024
    x = torch.as_tensor(rng.uniform(0, 5, (n, 2)), device="cuda")
    xs = torch.as_tensor(rng.uniform(0, 5, (m, 2)), device="cuda")
    y = torch.as_tensor(rng.standard_normal(n), device="cuda")
    f = S.GP(S.EQ())
    res = {}
    before = S.B.precision
    try:
        for prec in ("fp64", "auto"):
            S.B.precision = prec
            post = f | (f(x, 0.1), y)
            fdd = post(xs)
            res[prec] = (fdd.mean.squeeze().clone(), S.B.dense(fdd.var).clone())
    finally:
        S.B.precision = before
    assert (res["auto"][0] - res["fp64"][0]).abs().max().item() < 1e-10
    assert (res["auto"][1] - res["fp64"][1]).abs().max().item() < 1e-10


def test_emulation_switch_is_per_call(S, ops):
    """Switching B.precision back to "fp64" really returns to the native kernels (bit-identical results)."""
    rng = np.random.default_rng(2)
    x = torch.as_tensor(rng.standard_normal((2304, 2)), device="cuda")
    y = torch.as_tensor(rng.standard_normal(2304), device="cuda")
    f = S.GP(S.EQ())
    before = S.B.precision
    try:
        S.B.precision = "fp64"
        a = f(x, 0.1).logpdf(y).item()
        S.B.precision = "auto"
        b = f(x, 0.1).logpdf(y).item()
        S.B.precision = "fp64"
        c = f(x, 0.1).logpdf(y).item()
    finally:
        S.B.precision = before
    assert a == c
    assert abs(a - b) / abs(a) < 1e-11


def test_long_reduction_runs_in_k_chunks(S, ops):
    """K > 65536 (the sparse path's n = 262144 reductions): the emulated GEMM behind ``gemm_nt`` splits K into passes that
    each keep the int32 accumulation exact."""
    g = torch.Generator(device="cuda").manual_seed(9)
    M, N, K = 256, 384, 131072 + 128
    A = torch.randn(1, M, K, device="cuda", dtype=torch.float64, generator=g)
    Bm = torch.randn(1, N, K, device="cuda", dtype=torch.float64, generator=g)
    C0 = torch.randn(1, M, N, device="cuda", dtype=torch.float64, generator=g)
    ref = 0.5 * C0 + 2.0 * (A @ Bm.transpose(1, 2))
    before = S.B.precision
    try:
        S.B.precision = "fp64"
        native = ops.gemm_nt(A, Bm, C0.clone(), alpha=2.0, beta=0.5)
        S.B.precision = "auto"
        emu = ops.gemm_nt(A, Bm, C0.clone(), alpha=2.0, beta=0.5)
    finally:
        S.B.precision = before
    scale = ref.abs().max().item()
    assert (native - ref).abs().max().item() / scale < 1e-13
    assert (emu - ref).abs().max().item() / scale < 1e-12
    assert not torch.equal(emu, native)  # it really took the emulated path


@pytest.mark.parametrize("slices", [6, 7, 8])
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (-1.0, 1.0), (-1.5, 0.5)])
def test_gemm_oz_bit_exact_vs_integer_model(ops, slices, alpha, beta):
    """Every inexact step of the emulation is ONE correctly rounded fp64 operation (the slice products are exact integers),
    so the kernel must reproduce the NumPy integer model bit for bit."""
    rng = np.random.default_rng(slices)
    M, N, K = 256, 192, 384
    A = rng.standard_normal((M, K)) * np.exp(2 * rng.standard_normal((M, 1)))
    B = rng.standard_normal((N, K))
    C0 = rng.standard_normal((M, N))
    # rows from subnormal to near overflow (their products with each other O(1), with the other rows anything from zero
    # through subnormal to inf), and rows holding a NaN or an infinity
    for r, k in enumerate((-1070, -1020, -1000, -980, 980, 1000, 1020)):
        A[200 + r] = np.ldexp(rng.standard_normal(K), k)
        B[100 + r] = np.ldexp(rng.standard_normal(K), min(-k, 1020))
    A[220, 7], A[221, 300], B[120, 0] = np.nan, np.inf, -np.inf
    want = oz_model_gemm(A, B, C0, alpha, beta, slices)
    dev = lambda a: torch.as_tensor(a, device="cuda")
    got = ops.gemm_nt_oz(dev(A), dev(B), dev(C0).clone(), alpha=alpha, beta=beta, slices=slices).cpu().numpy()
    assert np.array_equal(got, want, equal_nan=True), np.nanmax(np.abs(got - want))
    normal = np.ones((M, N), bool)
    normal[200:], normal[:, 100:121] = False, False
    assert np.isfinite(got[normal]).all() and np.isnan(got[220:222]).all() and np.isnan(got[:, 120]).all()


def test_auto_picks_slices_by_conditioning(S):
    """"auto" = 7 slices when the matrix is well conditioned by construction (known scalar noise), 8 slices (the accuracy of
    the fp64 tensor-core kernel itself) for factorisations that may be numerically singular: noise-free kernels with the
    1e-12 jitter lose positive definiteness under the 100x larger backward error of 7 slices (tools/oz_illcond.py)."""
    rng = np.random.default_rng(4)
    n = 2304
    x = torch.as_tensor(rng.uniform(0, 10, (n, 2)), device="cuda")
    y = torch.as_tensor(rng.standard_normal(n), device="cuda")
    f = S.GP(S.EQ().stretch(0.1))  # short length scale: the noise-free matrix is comfortably positive definite
    before = S.B.precision
    out = {}
    try:
        for prec in ("auto", "int8x7", "int8x8"):
            S.B.precision = prec
            out[prec] = (f(x).logpdf(y).item(), f(x, 0.1).logpdf(y).item())
    finally:
        S.B.precision = before
    assert out["auto"][0] == out["int8x8"][0]  # noise-free: 8 slices
    assert out["auto"][1] == out["int8x7"][1]  # known noise: 7 slices
    assert out["int8x7"][1] != out["int8x8"][1]


@pytest.mark.parametrize("n", [4096, 4700, 5250, 6400])
def test_pair_scheme_vs_native(S, n):
    """n_pad >= 4096: the emulated factorisation updates the far trailing matrix once per PAIR of 512-panels with K = 1024
    (``potrf_driver_pairs``).  Ragged tails (a last pair with a short or missing second panel) against the native fp64 path."""
    rng = np.random.default_rng(n)
    x = torch.as_tensor(rng.uniform(0, 4, (n, 3)), device="cuda")
    y = torch.as_tensor(rng.standard_normal((n, 2)), device="cuda")  # two right-hand sides ride along as extra rows
    f = S.GP(S.EQ().stretch(0.7) + 0.5 * S.Matern32())
    out = {}
    before = S.B.precision
    try:
        for prec in ("fp64", "int8x8", "auto"):
            S.B.precision = prec
            out[prec] = f(x, 0.05).logpdf(y).cpu().numpy()
    finally:
        S.B.precision = before
    assert np.max(np.abs(out["int8x8"] - out["fp64"]) / np.abs(out["fp64"])) < 1e-12
    assert np.max(np.abs(out["auto"] - out["fp64"]) / np.abs(out["fp64"])) < 1e-11
