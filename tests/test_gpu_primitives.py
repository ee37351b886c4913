"""GPU parity of the C-ABI primitives (libgpk) against the NumPy oracle / torch fp64 on the same seeded inputs."""
import numpy as np
import pytest
import torch

from oracle import gp_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from stheno_b200 import ops

    return ops


def dev(a, dtype=torch.float64):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device="cuda")


def groups(x, scales, dtype=torch.float64):
    """[G, B=1, n, d] stretched inputs."""
    x = np.asarray(x, np.float64)
    if x.ndim == 1:
        x = x[:, None]
    return torch.stack([dev(x / s, dtype)[None] for s in scales])


KERNELS = [
    ("eq", [(1.0, [("eq", 0)])], [1.0], ("eq",)),
    ("m12", [(1.0, [("matern12", 0)])], [1.0], ("matern12",)),
    ("m32", [(1.0, [("matern32", 0)])], [1.0], ("matern32",)),
    ("m52", [(1.0, [("matern52", 0)])], [1.0], ("matern52",)),
    ("lin", [(1.0, [("linear", 0)])], [1.0], ("linear",)),
    ("eq_stretch_plus_delta", [(1.0, [("eq", 0)]), (0.1, [("delta", 0)])], [2.0],
     ("sum", ("stretched", 2.0, ("eq",)), ("scaled", 0.1, ("delta",)))),
    ("composite", [(2.0, [("eq", 0)]), (0.5, [("matern32", 1), ("linear", 1)]), (0.3, [("one", 0)])], [2.0, 0.7],
     ("sum", ("sum", ("scaled", 2.0, ("stretched", 2.0, ("eq",))),
              ("scaled", 0.5, ("product", ("stretched", 0.7, ("matern32",)), ("stretched", 0.7, ("linear",))))),
      ("scaled", 0.3, ("one",)))),
]


@pytest.mark.parametrize("name,terms,scales,spec", KERNELS, ids=[k[0] for k in KERNELS])
@pytest.mark.parametrize("n,m,d", [(5, 3, 1), (100, 77, 1), (130, 64, 8), (333, 200, 3), (64, 64, 2)])
def test_kernel_matrix_vs_oracle(ops, name, terms, scales, spec, n, m, d):
    rng = np.random.default_rng(n * 1000 + m + d)
    x = rng.standard_normal((n, d))
    y = rng.standard_normal((m, d))
    y[: min(2, m)] = x[: min(2, m)]  # exact repeats exercise Delta's non-same branch
    flat = ops.FlatKernel(terms, len(scales))
    K = ops.kernel_matrix(flat, groups(x, scales), groups(y, scales), same=False)[0].cpu().numpy()
    ref = O.kernel_matrix(spec, x, y)
    # Matern12 is not smooth at r = 0: for d > 1 the reference's GEMM-expansion distance leaves +-1e-15 of rounding
    # noise in r^2 on coincident points, i.e. r ~ 3e-8 instead of 0 and exp(-r) off by ~6e-8 there (the direct
    # difference form used on the GPU gives exactly 0).  Everything else agrees to rounding.
    atol = 2e-7 if (name == "m12" and d > 1) else 1e-13
    np.testing.assert_allclose(K, ref, rtol=1e-12, atol=atol)
    Ks = ops.kernel_matrix(flat, groups(x, scales), noise_scalar=0.25, jitter=1e-3)[0].cpu().numpy()
    refs = O.kernel_matrix(spec, x) + (0.25 + 1e-3) * np.eye(n)
    np.testing.assert_allclose(Ks, refs, rtol=1e-12, atol=atol)
    kd = ops.kernel_diag(flat, groups(x, scales))[0].cpu().numpy()
    np.testing.assert_allclose(kd, O.kernel_elwise(spec, x)[:, 0], rtol=1e-12, atol=atol)


def test_kernel_matrix_fp32_and_batch(ops):
    rng = np.random.default_rng(0)
    x = rng.standard_normal((3, 150, 4))
    xg = dev(x, torch.float32)[None]
    flat = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    nv = dev(rng.uniform(0.1, 0.2, (3, 150)), torch.float32)
    K = ops.kernel_matrix(flat, xg, noise_vec=nv).cpu().numpy()
    for b in range(3):
        ref = O.kernel_matrix(("eq",), x[b]) + np.diag(nv[b].cpu().numpy().astype(np.float64))
        np.testing.assert_allclose(K[b], ref, rtol=2e-6, atol=2e-6)


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-12), (torch.float32, 2e-4)])
def test_gemm_nt(ops, dtype, tol):
    g = torch.Generator(device="cuda").manual_seed(1)
    A = torch.randn(2, 256, 160, device="cuda", dtype=dtype, generator=g)
    Bm = torch.randn(2, 384, 160, device="cuda", dtype=dtype, generator=g)
    C = torch.randn(2, 256, 384, device="cuda", dtype=dtype, generator=g)
    ref = 0.5 * C.double() - 1.5 * A.double() @ Bm.double().transpose(1, 2)
    out = ops.gemm_nt(A, Bm, C.clone(), alpha=-1.5, beta=0.5)
    assert (out.double() - ref).abs().max().item() < tol * 200
    out0 = ops.gemm_nt(A, Bm)
    assert (out0.double() - A.double() @ Bm.double().transpose(1, 2)).abs().max().item() < tol * 200
    # K = 0: exactly beta C.  Called through the C ABI with the operands' own pointers: torch reports a null data pointer
    # for a zero-width view, which the library rejects.
    outk0 = C.clone()
    ops.check(ops._fn("gpk_gemm_nt", dtype)(256, 384, 0, -1.5, ops._ptr(A), A.stride(1), A.stride(0), ops._ptr(Bm),
                                            Bm.stride(1), Bm.stride(0), 0.5, ops._ptr(outk0), outk0.stride(1),
                                            outk0.stride(0), 0, 2, ops._stream()), "gpk_gemm_nt")
    assert torch.equal(outk0, 0.5 * C)
    if dtype == torch.float64:
        # lower mode over 3600 tile rows (450 groups of 8), K = 128: the fp64 tensor-core kernel, not the emulation
        A3 = torch.randn(1, 460800, 128, device="cuda", dtype=dtype, generator=g)
        B3 = torch.randn(1, 256, 128, device="cuda", dtype=dtype, generator=g)
        C3 = torch.full((1, 460800, 256), float("nan"), device="cuda", dtype=dtype)
        ops.gemm_nt(A3, B3, C3, lower=True)
        ref = A3[0] @ B3[0].T
        assert (C3[0, :, :128] - ref[:, :128]).abs().max().item() < tol * 200
        assert (C3[0, 128:, 128:] - ref[128:, 128:]).abs().max().item() < tol * 200
        assert C3[0, :128, 128:].isnan().all()  # tile (0, 1), above the diagonal, is untouched
        del A3, B3, C3, ref
    # lower: only tiles on/below the diagonal are touched
    S = torch.randn(1, 384, 144, device="cuda", dtype=dtype, generator=g)
    C2 = torch.zeros(1, 384, 384, device="cuda", dtype=dtype)
    ops.gemm_nt(S, S, C2, alpha=1.0, beta=1.0, lower=True)
    full = (S.double() @ S.double().transpose(1, 2))[0]
    got = C2[0].double()
    for ti in range(3):
        for tj in range(3):
            blk = got[ti * 128:(ti + 1) * 128, tj * 128:(tj + 1) * 128]
            if tj <= ti:
                assert (blk - full[ti * 128:(ti + 1) * 128, tj * 128:(tj + 1) * 128]).abs().max().item() < tol * 200
            else:
                assert blk.abs().max().item() == 0.0


@pytest.mark.parametrize("K", [16, 48, 96, 144])
def test_gemm_nt_f32_ffma(ops, K):
    """The fp32 FFMA kernel (``gemm_nt_f32_kernel``): the 3xTF32 kernel takes only K >= 128 with K % 32 == 0, so these K
    (the Schur-complement GEMM of a fp32 Woodbury matrix with n <= 96 has K = round_up(n, 32) < 128) run on FFMA.
    alpha / beta, beta = 0 over a NaN-filled C, lower mode with a sentinel above the diagonal tiles, batch 2.
    Bound: 2 K u_32 |alpha| |A| |B|^T plus the rounding of the result and of beta C."""
    u = 2.0**-24
    g = torch.Generator(device="cuda").manual_seed(K)
    A = torch.randn(2, 384, K, device="cuda", generator=g) * torch.exp(torch.randn(2, 384, 1, device="cuda", generator=g))
    Bm = torch.randn(2, 256, K, device="cuda", generator=g)
    C0 = torch.randn(2, 384, 256, device="cuda", generator=g)
    Ad, Bd, Cd = A.double(), Bm.double(), C0.double()
    absprod = Ad.abs() @ Bd.abs().transpose(1, 2)

    def check(out, alpha, beta, mask=None):
        ref = alpha * (Ad @ Bd.transpose(1, 2)) + (beta * Cd if beta else 0.0)
        bound = 2 * K * u * abs(alpha) * absprod + 2 * u * (ref.abs() + abs(beta) * Cd.abs())
        ok = (out.double() - ref).abs() <= bound
        assert (ok if mask is None else ok[:, mask]).all()

    launches = ops.launch_count()
    check(ops.gemm_nt(A, Bm, C0.clone(), alpha=-1.5, beta=0.5), -1.5, 0.5)
    assert ops.launch_count() == launches + 1  # one kernel, no split or copy
    nan_c = torch.full_like(C0, float("nan"))
    out = ops.gemm_nt(A, Bm, nan_c, alpha=-0.75, beta=0.0)
    assert out.isfinite().all()
    check(out, -0.75, 0.0)
    # lower: the tiles on / below the diagonal get beta C + alpha A B^T, the tiles above keep their sentinel bit for bit
    tr = torch.arange(384, device="cuda")[:, None] // 128
    tc = torch.arange(256, device="cuda")[None, :] // 128
    touched = tc <= tr
    Cs = torch.where(touched, C0, torch.full_like(C0, 31.25))
    out = ops.gemm_nt(A, Bm, Cs.clone(), alpha=1.0, beta=1.0, lower=True)
    assert torch.equal(out[:, ~touched], Cs[:, ~touched])
    Cd = Cs.double()
    check(out, 1.0, 1.0, touched)


def _spd(n, B=1, seed=0, dtype=torch.float64, cond_shift=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(B, n, n, device="cuda", dtype=torch.float64, generator=g)
    K = A @ A.transpose(1, 2) / n + (cond_shift if cond_shift is not None else 0.5) * torch.eye(n, device="cuda", dtype=torch.float64)
    return K.to(dtype)


@pytest.mark.parametrize("n", [3, 128, 300, 1000, 1280, 2500])
def test_potrf_dense_vs_torch(ops, n):
    K = _spd(n, B=2, seed=n)
    g = torch.Generator(device="cuda").manual_seed(7)
    rhs = torch.randn(2, 3, n, device="cuda", dtype=torch.float64, generator=g)
    ch = ops.chol_from_dense(K, jitter=1e-12, rhs_t=rhs).check()
    Lref = torch.linalg.cholesky(K + 1e-12 * torch.eye(n, device="cuda", dtype=torch.float64))
    assert (ch.L() - Lref).abs().max().item() < 1e-11
    ld_ref = 2 * torch.log(torch.diagonal(Lref, dim1=1, dim2=2)).sum(-1)
    assert ((ch.logdet - ld_ref).abs() / ld_ref.abs().clamp_min(1)).max().item() < 1e-12
    half_ref = torch.linalg.solve_triangular(Lref, rhs.transpose(1, 2), upper=False).transpose(1, 2)
    assert (ch.rhs_half() - half_ref).abs().max().item() < 1e-10
    lp = ch.logpdf()
    lp_ref = -0.5 * (ld_ref[:, None] + n * np.log(2 * np.pi) + (half_ref ** 2).sum(-1))
    assert ((lp - lp_ref).abs() / lp_ref.abs()).max().item() < 1e-12
    # separate solves
    hs = ch.half_solve(rhs)
    assert (hs - half_ref).abs().max().item() < 1e-10
    fs = ch.full_solve(rhs)
    full_ref = torch.cholesky_solve(rhs.transpose(1, 2), Lref).transpose(1, 2)
    assert (fs - full_ref).abs().max().item() < 1e-9


def test_potrf_on_two_devices(ops):
    """CUDA applies a kernel's opt-in to more than 48 KB of shared memory per device: a factorisation on cuda:0, then one
    on cuda:1 in the same process (the leaf, the tensor-core TRSM and the emulated GEMM all launch above 48 KB)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for i in range(2):
        with torch.cuda.device(i):  # ops launches on the current device's stream
            K = _spd(4096, seed=i)
            ch = ops.chol_from_dense(K).check()
            assert ch.L().device == torch.device("cuda", i)
            assert (ch.L() - torch.linalg.cholesky(K)).abs().max().item() < 1e-10


def test_potrf_not_pd_reports_info(ops):
    K = _spd(200, B=1, seed=3)
    K[0, 150, 150] = -1.0
    ch = ops.chol_from_dense(K)
    assert int(ch.info[0]) == 151
    with pytest.raises(torch.linalg.LinAlgError):
        ch.check()


def test_potrf_fp32_batched(ops):
    K = _spd(384, B=5, seed=11, dtype=torch.float32)
    ch = ops.chol_from_dense(K, jitter=1e-6).check()
    Lref = torch.linalg.cholesky(K.double() + 1e-6 * torch.eye(384, device="cuda", dtype=torch.float64))
    assert (ch.L().double() - Lref).abs().max().item() < 5e-5
    ld_ref = 2 * torch.log(torch.diagonal(Lref, dim1=1, dim2=2)).sum(-1)
    assert ((ch.logdet.double() - ld_ref).abs() / ld_ref.abs()).max().item() < 1e-4


def test_config1_logpdf_vs_oracle(ops):
    # BASELINE config 1: EQ GP, n=1000, d=1, fp64 (SURVEY 8d: x = linspace(0, 10, 1000), noise 0.1)
    rng = np.random.default_rng(1)
    x = np.linspace(0, 10, 1000)
    y = rng.standard_normal((1000, 2))
    flat = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    ch = ops.chol_from_kernel(flat, groups(x, [1.0]), noise_scalar=0.1, jitter=1e-12, rhs_t=dev(y.T)[None]).check()
    lp = ch.logpdf()[0].cpu().numpy()
    ref = O.fdd_logpdf(("eq",), x, 0.1, y)
    np.testing.assert_allclose(lp, ref, rtol=1e-10)


def test_posterior_pieces_vs_oracle(ops):
    rng = np.random.default_rng(2)
    n, m, d = 700, 300, 3
    x = rng.standard_normal((n, d))
    xs = rng.standard_normal((m, d))
    y = rng.standard_normal(n)
    spec = ("stretched", 1.5, ("matern52",))
    flat = ops.FlatKernel([(1.0, [("matern52", 0)])], 1)
    xg, xsg = groups(x, [1.5]), groups(xs, [1.5])
    ch = ops.chol_from_kernel(flat, xg, noise_scalar=0.2, jitter=1e-12, rhs_t=dev(y)[None, None]).check()
    V = ops.kernel_rows_padded(flat, xsg, xg, ch)
    ch.solve_rows_(V)
    b = torch.zeros(1, ch.n_pad, device="cuda", dtype=torch.float64)
    b[:, :n] = ch.rhs_half()[:, 0]
    dot, sq = ops.row_dot_sq(V, m, ch.n_pad, b)
    mean_ref, var_ref = O.posterior(spec, x, 0.2, y, xs)
    np.testing.assert_allclose(dot[0].cpu().numpy(), mean_ref[:, 0], rtol=1e-9, atol=1e-10)
    vd = ops.kernel_diag(flat, xsg)[0] - sq[0]
    np.testing.assert_allclose(vd.cpu().numpy(), np.diag(var_ref), rtol=1e-8, atol=1e-10)
    # full covariance: K** - V V^T on the tensor cores, lower tiles + mirror
    m_pad = V.shape[1]
    Kss = torch.zeros(1, m_pad, m_pad, device="cuda", dtype=torch.float64)
    Kss[:, :m, :m] = ops.kernel_matrix(flat, xsg)
    ops.gemm_nt(V, V, Kss, alpha=-1.0, beta=1.0, lower=True)
    ops.symmetrize_(Kss, m)
    np.testing.assert_allclose(Kss[0, :m, :m].cpu().numpy(), var_ref, rtol=1e-8, atol=1e-9)


def test_transpose_and_symmetrize(ops):
    A = torch.randn(2, 70, 45, device="cuda", dtype=torch.float64)
    assert torch.equal(ops.transpose(A, 70, 45), A.transpose(1, 2).contiguous())
    S = torch.randn(1, 100, 100, device="cuda", dtype=torch.float32)
    ref = torch.tril(S) + torch.tril(S, -1).transpose(1, 2)
    assert torch.equal(ops.symmetrize_(S.clone(), 100), ref)


def tc32_probe(ops, M, N, K, batch=1, lower=False, gemm=None):
    """Which kernel an fp32 ``gemm_nt`` of this shape runs on: "tc32" (3xTF32 wgmma) or "ffma".

    The probe puts a single ``a = 1 + 2^-11`` at the same k in the last row of A and the first row of B (a tile on or below
    the diagonal).  The 3xTF32 split drops the ``a_lo b_lo`` term and gives exactly ``a^2 - 2^-22 = 1 + 2^-10``; FFMA gives
    ``a^2 = 1 + 2^-10 + 2^-22`` exactly.  A kernel that silently falls back to FFMA therefore shows here."""
    gemm = ops.gemm_nt if gemm is None else gemm
    A = torch.zeros(batch, M, K, device="cuda", dtype=torch.float32)
    Bm = torch.zeros(batch, N, K, device="cuda", dtype=torch.float32)
    a = 1.0 + 2.0**-11
    A[:, M - 1, K - 1] = a
    Bm[:, 0, K - 1] = a
    C = gemm(A, Bm, torch.zeros(batch, M, N, device="cuda", dtype=torch.float32), alpha=-1.0, beta=1.0, lower=lower)
    got = {float(v) for v in C[:, M - 1, 0].cpu()}
    if got == {-(1.0 + 2.0**-10)}:
        return "tc32"
    assert got == {-(1.0 + 2.0**-10 + 2.0**-22)}, got
    return "ffma"


@pytest.mark.parametrize("M,N,K,batch,lower", [(128, 128, 128, 1, False), (256, 384, 512, 2, False), (384, 384, 256, 3, True),
                                                 (1024, 512, 1024, 1, False)])
def test_gemm_f32_tensor_core_3xtf32(ops, M, N, K, batch, lower):
    """fp32 GEMM on wgmma (3xTF32 split): fp32-level accuracy against an fp64 reference, incl. strided views; the probe proves
    the shape runs on the 3xTF32 kernel (FFMA would pass the accuracy bar too)."""
    assert tc32_probe(ops, M, N, K, batch, lower) == "tc32"
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    big = torch.randn(batch, M + 128, K + 64, device="cuda", generator=g)
    A = big[:, 64:64 + M, 32:32 + K]  # a strided view: ld = K + 64, non-zero offset
    Bm = torch.randn(batch, N, K, device="cuda", generator=g)
    C = torch.randn(batch, M, N, device="cuda", generator=g)
    ref = 0.5 * C.double() - 1.25 * A.double() @ Bm.double().transpose(1, 2)
    out = ops.gemm_nt(A, Bm, C.clone(), alpha=-1.25, beta=0.5, lower=lower)
    scale = (A.double().abs() @ Bm.double().abs().transpose(1, 2)).max().item()
    err = (out.double() - ref).abs()
    if lower:
        tr = torch.arange(M, device="cuda")[:, None] // 128
        tc = torch.arange(N, device="cuda")[None, :] // 128
        mask = tc <= tr
        assert torch.equal(out[:, ~mask], C[:, ~mask])  # tiles above the diagonal untouched
        err = err * mask
    # plain TF32 would be ~1e-3 relative; the split recovers fp32-level accuracy.  Measured (tools/f32_gemm_accuracy.py):
    # max |err| / sum|a||b| = 8e-7 (K=128) .. 3.9e-6 (K=4096), zero-mean, vs 2.3e-7 for the FFMA kernel.
    assert err.max().item() < 6e-6 * scale
