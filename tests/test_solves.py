"""Triangular solves with the padded factor (``gpk_trsm_right`` / ``gpk_trsm_right_t``, the recursive
``solve_many_rows_t_``) and the one-call posterior (``gpk_posterior_marginals``) against fp64 references: forward error
against ``solve_triangular`` on a well-conditioned ``L``, and a normwise backward error with the residual formed on the host
in extended precision."""
import numpy as np
import pytest
import scipy.linalg as sla
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from stheno_b200 import ops

    return ops


def chol_of(ops, batch, n, dtype, seed):
    """Factor of a well-conditioned SPD matrix (G G^T / 64 + I) of size n = n_pad."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    G = torch.randn(batch, n, 64, device="cuda", dtype=torch.float64, generator=g)
    A = G @ G.transpose(1, 2) / 64 + torch.eye(n, device="cuda", dtype=torch.float64)
    ch = ops.chol_from_dense(A.to(dtype))
    assert not ch.info.any()
    return ch


def backward_error(L, X, Bt, transpose, rows=(0, 1, 63, 64, 127, 128, -2, -1)):
    """max over some rows (first / last of each 128-row block among them) of |x L^T - b| / (|L| |x| + |b|) (resp. x L),
    residual in np.longdouble (no BLAS: a sample of rows keeps it fast)."""
    rows = sorted({r % X.shape[-2] for r in rows})
    L = L.astype(np.longdouble)
    X, Bt = X[..., rows, :].astype(np.longdouble), Bt[..., rows, :].astype(np.longdouble)
    Lop = L if transpose else np.swapaxes(L, -1, -2)
    r = np.abs(X @ Lop - Bt).max(-1)
    scale = (np.abs(X) @ np.abs(Lop)).max(-1) + np.abs(Bt).max(-1)
    return float((r / scale).max())


U = {torch.float64: 2.0**-53, torch.float32: 2.0**-24}


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("n", [128, 896, 4096])
def test_trsm_right(ops, n, batch, dtype):
    """Bt <- Bt L^-T: 896 is a recursion that does not halve into powers of two; at 4096 with 384 rows the (batch-1,
    fp64) solve's largest GEMM (384 x 2048 x 2048 >= 1.5e9) goes through the emulation under the default precision --
    checked on the launch profile, as is its absence everywhere else."""
    ch = chol_of(ops, batch, n, dtype, n + batch)
    g = torch.Generator(device="cuda").manual_seed(1)
    Bt = torch.randn(batch, 384, n, device="cuda", dtype=torch.float64, generator=g).to(dtype)
    ops.gemm_profile(True)
    try:
        X = ch.solve_rows_(Bt.clone())
        n_oz = ops.gemm_profile_read(1)[2]
    finally:
        ops.gemm_profile(False)
    emulated = n == 4096 and batch == 1 and dtype == torch.float64
    assert (n_oz > 0) == emulated, (n_oz, emulated)
    L, Xn, Bn = ch.L().double().cpu().numpy(), X.double().cpu().numpy(), Bt.double().cpu().numpy()
    want = np.stack([sla.solve_triangular(L[b], Bn[b].T, lower=True).T for b in range(batch)])
    u = U[dtype]
    assert np.abs(Xn - want).max() / np.abs(want).max() <= 100 * n * u
    assert backward_error(L, Xn, Bn, transpose=False) <= 4 * n * u


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("rows", [64, 192])
def test_trsm_right_t_ragged_rows(ops, rows, batch, dtype):
    """Bt <- Bt L^-1 (backward substitution) with a row count that is not a multiple of 128."""
    n = 896
    ch = chol_of(ops, batch, n, dtype, rows + batch)
    g = torch.Generator(device="cuda").manual_seed(2)
    Bt = torch.randn(batch, rows, n, device="cuda", dtype=torch.float64, generator=g).to(dtype)
    guard = torch.randn(batch, 64, n, device="cuda", dtype=dtype, generator=None)
    buf = torch.cat([Bt, guard], dim=1)  # rows below the problem: must stay untouched
    ch.solve_rows_t_(buf[:, :rows])
    assert torch.equal(buf[:, rows:], guard)
    L, Xn, Bn = ch.L().double().cpu().numpy(), buf[:, :rows].double().cpu().numpy(), Bt.double().cpu().numpy()
    want = np.stack([sla.solve_triangular(L[b], Bn[b].T, lower=True, trans="T").T for b in range(batch)])
    u = U[dtype]
    assert np.abs(Xn - want).max() / np.abs(want).max() <= 100 * n * u
    assert backward_error(L, Xn, Bn, transpose=True) <= 4 * n * u


def test_solve_many_rows_t_small_blocks(ops):
    """The recursive transposed solve with 256-column leaves and 128-column panels against the plain substitution."""
    n = 1664
    ch = chol_of(ops, 1, n, torch.float64, 5)
    g = torch.Generator(device="cuda").manual_seed(3)
    Bt = torch.randn(1, 384, n, device="cuda", dtype=torch.float64, generator=g)
    X = ch.solve_many_rows_t_(Bt.clone(), leaf=256, panel=128)
    Y = ch.solve_rows_t_(Bt.clone())
    assert ((X - Y).abs().max() / Y.abs().max()).item() < 1e-12
    L = ch.L().cpu().numpy()[0]
    want = sla.solve_triangular(L, Bt[0].cpu().numpy().T, lower=True, trans="T").T
    assert np.abs(X[0].cpu().numpy() - want).max() / np.abs(want).max() < 1e-12


@pytest.mark.parametrize("want_dot,want_sq", [(True, True), (True, False), (False, True)])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_posterior_marginals_chunks(ops, dtype, want_dot, want_sq):
    """``gpk_posterior_marginals`` streamed in chunks of 128 test points (m = 389: three full chunks and a ragged one)
    against a NumPy reference, and bit for bit against a single chunk (n = 1000: no emulation anywhere)."""
    rng = np.random.default_rng(8)
    n, m, d = 1000, 389, 2
    x, xs = rng.uniform(0, 4, (n, d)), rng.uniform(0, 4, (m, d))
    y = rng.standard_normal(n)
    flat = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    xg = torch.as_tensor(x, device="cuda", dtype=dtype)[None, None]
    xsg = torch.as_tensor(xs, device="cuda", dtype=dtype)[None, None]
    ch = ops.chol_from_kernel(flat, xg, noise_scalar=0.1, rhs_t=torch.as_tensor(y, device="cuda", dtype=dtype)[None, None])
    half_y = ch.rhs_half()[0, 0] if want_dot else None
    dot, sq = ops.posterior_marginals(flat, xsg, xg, ch, half_y, want_sq=want_sq, chunk=128)
    dot1, sq1 = ops.posterior_marginals(flat, xsg, xg, ch, half_y, want_sq=want_sq, chunk=4096)
    assert (dot is None) == (not want_dot) and (sq is None) == (not want_sq)
    # reference in fp64 on the host
    xr, xsr = np.asarray(xg[0, 0].cpu(), np.float64), np.asarray(xsg[0, 0].cpu(), np.float64)
    d2 = lambda a, b: ((a[:, None, :] - b[None, :, :]) ** 2).sum(-1)
    K = np.exp(-0.5 * d2(xr, xr)) + 0.1 * np.eye(n)
    Ks = np.exp(-0.5 * d2(xsr, xr))
    L = np.linalg.cholesky(K)
    V = sla.solve_triangular(L, Ks.T, lower=True)
    tol = 1e-10 if dtype == torch.float64 else 2e-3
    if want_dot:
        ref_dot = V.T @ sla.solve_triangular(L, np.asarray(torch.as_tensor(y, dtype=dtype).double()), lower=True)
        assert np.abs(dot.double().cpu().numpy() - ref_dot).max() <= tol * max(1.0, np.abs(ref_dot).max())
        assert torch.equal(dot, dot1)
    if want_sq:
        ref_sq = (V**2).sum(0)
        assert np.abs(sq.double().cpu().numpy() - ref_sq).max() <= tol
        assert torch.equal(sq, sq1)
