"""TEST-ONLY stand-in for ``stheno_b200.ops`` so that the host-side model layer (kernel algebra, lazy measure graph,
FDD / Normal / Observations plumbing, multi-output block assembly) can be exercised on a machine without a GPU.

It mirrors the *storage conventions* of the CUDA ops (padded workspaces, right-hand sides as rows) with plain torch
CPU linear algebra.  It is never importable from the product: ``stheno_b200`` has no CPU path and raises without CUDA.
"""
import math

import torch

from stheno_b200 import ops as real_ops

TILE = 128
round_up = real_ops.round_up
FlatKernel = real_ops.FlatKernel
LOG_2_PI = math.log(2 * math.pi)


def _factor(kind, x, y, same_obj, param=None):
    # x: [B, n, d], y: [B, m, d]
    d = x.shape[-1]
    diff = x[:, :, None, :] - y[:, None, :, :]
    d2 = (diff * diff).sum(-1)
    if kind == "eq":
        return torch.exp(-0.5 * d2)
    if kind == "rq":
        return torch.exp(-param * torch.log1p(d2 / (2.0 * param)))
    if kind in ("matern12", "matern32", "matern52"):
        r = torch.sqrt(d2) if d == 1 else torch.sqrt(torch.clamp_min(d2, 1e-30))
        if kind == "matern12":
            return torch.exp(-r)
        if kind == "matern32":
            s = math.sqrt(3.0) * r
            return (1 + s) * torch.exp(-s)
        s = math.sqrt(5.0) * r
        return (1 + s + 5.0 / 3.0 * d2) * torch.exp(-s)
    if kind == "linear":
        return x @ y.transpose(1, 2)
    if kind == "delta":
        if same_obj:
            return torch.eye(x.shape[1], dtype=x.dtype).expand(x.shape[0], -1, -1).clone()
        return (d2 < 1e-10).to(x.dtype)
    if kind == "one":
        return torch.ones_like(d2)
    raise ValueError(kind)


def _eval(flat, xg, yg, same):
    out = torch.zeros(xg.shape[1], xg.shape[2], yg.shape[2], dtype=xg.dtype)
    for coef, fs in flat.terms:
        prod = torch.full_like(out, coef)
        for fac in fs:
            prod = prod * _factor(fac[0], xg[fac[1]], yg[fac[1]], same, fac[2] if len(fac) > 2 else None)
        out = out + prod
    return out


def kernel_matrix(flat, xg, yg=None, *, same=None, noise_scalar=0.0, noise_vec=None, jitter=0.0):
    if yg is None:
        yg, same = xg, (True if same is None else same)
    K = _eval(flat, xg, yg, bool(same))
    if same:
        n = K.shape[1]
        idx = torch.arange(n)
        K[:, idx, idx] += noise_scalar
        if noise_vec is not None:
            K[:, idx, idx] += noise_vec.reshape(-1, n)
        K[:, idx, idx] += jitter
    return K


KM_LOWER, KM_SAME, KM_PAD_IDENTITY, KM_PAD_ZERO = 1, 2, 4, 8


def _km_launch(flat, xg, yg, n, n2, d, flags, noise_scalar, noise_vec, jitter, out, ldo, o_bstride, batch):
    """Stand-in of the raw K1 launch: ``out`` is a (possibly strided) view ``[B, >= n, >= n2]`` written in place."""
    same = bool(flags & KM_SAME)
    K = kernel_matrix(flat, xg, None if (same and yg is xg) else yg, same=same, noise_scalar=noise_scalar if same else 0.0,
                      noise_vec=noise_vec if same else None, jitter=jitter if same else 0.0)
    out[:, :n, :n2] = K


def _new_workspace(B, n, k, device, dtype, rhs_t):
    n_pad = round_up(max(n, 1))
    extra = round_up(k) if k > 0 else 0
    W = torch.zeros(B, n_pad + extra, n_pad, dtype=dtype)
    if extra:
        W[:, n_pad : n_pad + k, :n] = rhs_t
    return W, n_pad, extra


def _potrf(W, n, n_pad, extra, k, well_conditioned=False):
    Kp = torch.tril(W[:, :n_pad]) + torch.tril(W[:, :n_pad], -1).transpose(1, 2)
    rhs = W[:, n_pad : n_pad + k, :n].clone() if k else None
    return _finish(Kp, n, rhs)


def kernel_diag(flat, xg, yg=None, *, same=None):
    if yg is None:
        yg, same = xg, (True if same is None else same)
    B, n = xg.shape[1], xg.shape[2]
    out = torch.zeros(B, n, dtype=xg.dtype)
    for coef, fs in flat.terms:
        prod = torch.full_like(out, coef)
        for fac in fs:
            kind, g = fac[0], fac[1]
            param = fac[2] if len(fac) > 2 else None
            x, y = xg[g], yg[g]
            d2 = ((x - y) ** 2).sum(-1)
            if kind == "linear":
                v = (x * y).sum(-1)
            elif kind == "delta":
                v = torch.ones_like(d2) if same else (d2 < 1e-10).to(x.dtype)
            else:
                v = torch.diagonal(_factor(kind, x, y, same), dim1=1, dim2=2) if False else None
                if v is None:
                    xx = x.reshape(-1, 1, x.shape[-1])
                    yy = y.reshape(-1, 1, y.shape[-1])
                    v = _factor(kind, xx, yy, False, param).reshape(B, n)
            prod = prod * v
        out = out + prod
    return out


def gemm_nt(A, Bm, C=None, *, alpha=1.0, beta=0.0, lower=False):
    P = alpha * (A @ Bm.transpose(1, 2))
    if C is None:
        return P
    if lower:
        M, N = P.shape[1], P.shape[2]
        tr = torch.arange(M)[:, None] // TILE
        tc = torch.arange(N)[None, :] // TILE
        mask = (tc <= tr)
        C[:] = torch.where(mask, beta * C + P, C)
    else:
        C[:] = beta * C + P
    return C


def symmetrize_(A, n):
    sub = A[:, :n, :n]
    low = torch.tril(sub)
    A[:, :n, :n] = low + torch.tril(sub, -1).transpose(1, 2)
    return A


def transpose(src, rows, cols, out=None):
    if out is None:
        out = torch.empty(src.shape[0], cols, rows, dtype=src.dtype)
    out[:, :cols, :rows] = src[:, :rows, :cols].transpose(1, 2)
    return out


def row_dot_sq(V, rows, n_cols, b=None, want_dot=True, want_sq=True):
    Vv = V[:, :rows, :n_cols]
    dot = (Vv * b[:, None, :n_cols]).sum(-1) if (b is not None and want_dot) else None
    sq = (Vv * Vv).sum(-1) if want_sq else None
    return dot, sq


class Chol:
    def __init__(self, W, n, k, logdet, info):
        self.W, self.n, self.k, self.logdet, self.info = W, n, k, logdet, info
        self.n_pad, self.batch = W.shape[2], W.shape[0]

    dtype = property(lambda self: self.W.dtype)
    device = property(lambda self: self.W.device)

    def check(self):
        if bool(self.info.any()):
            raise torch.linalg.LinAlgError("not positive definite")
        return self

    def L_padded(self):
        return self.W[:, : self.n_pad, :]

    def L(self):
        return torch.tril(self.W[:, : self.n, : self.n])

    def L_lower_(self):
        self.W[:, : self.n_pad, :].tril_()
        return self.W[:, : self.n_pad, :]

    def rhs_half(self):
        return self.W[:, self.n_pad : self.n_pad + self.k, : self.n]

    def logpdf(self):
        h = self.W[:, self.n_pad : self.n_pad + self.k, :]
        return -0.5 * (self.logdet[:, None] + self.n * LOG_2_PI + (h * h).sum(-1))

    def new_rows(self, rows, zero=True):
        return torch.zeros(self.batch, round_up(rows), self.n_pad, dtype=self.dtype)

    def _Lfull(self):
        return torch.tril(self.W[:, : self.n_pad, :])

    def solve_rows_(self, Bt):
        Bt[:] = torch.linalg.solve_triangular(self._Lfull(), Bt.transpose(1, 2), upper=False).transpose(1, 2)
        return Bt

    def solve_rows_t_(self, Bt):
        Bt[:] = torch.linalg.solve_triangular(self._Lfull().transpose(1, 2), Bt.transpose(1, 2), upper=True).transpose(1, 2)
        return Bt

    def half_solve(self, bt):
        m = bt.shape[1]
        buf = self.new_rows(m)
        buf[:, :m, : self.n] = bt
        return self.solve_rows_(buf)[:, :m, : self.n]

    def full_solve(self, bt):
        m = bt.shape[1]
        buf = self.new_rows(m)
        buf[:, :m, : self.n] = bt
        self.solve_rows_(buf)
        return self.solve_rows_t_(buf)[:, :m, : self.n]


def _finish(Kp, n, rhs_t):
    B, n_pad = Kp.shape[0], Kp.shape[1]
    k = 0 if rhs_t is None else rhs_t.shape[1]
    extra = round_up(k) if k else 0
    W = torch.zeros(B, n_pad + extra, n_pad, dtype=Kp.dtype)
    L, info = torch.linalg.cholesky_ex(Kp)
    W[:, :n_pad] = L
    logdet = 2 * torch.log(torch.diagonal(L, dim1=1, dim2=2)).sum(-1)
    if k:
        R = torch.zeros(B, extra, n_pad, dtype=Kp.dtype)
        R[:, :k, :n] = rhs_t
        W[:, n_pad:] = torch.linalg.solve_triangular(L, R.transpose(1, 2), upper=False).transpose(1, 2)
    return Chol(W, n, k, logdet, info.to(torch.int32))


def _pad_identity(K, n):
    B = K.shape[0]
    n_pad = round_up(max(n, 1))
    Kp = torch.eye(n_pad, dtype=K.dtype).expand(B, -1, -1).clone()
    Kp[:, :n, :n] = K
    return Kp


def chol_from_kernel(flat, xg, *, noise_scalar=0.0, noise_vec=None, jitter=0.0, rhs_t=None, full_precision=False):
    K = kernel_matrix(flat, xg, noise_scalar=noise_scalar, noise_vec=noise_vec, jitter=jitter)
    n = K.shape[1]
    return _finish(_pad_identity(K, n), n, rhs_t)


def chol_from_dense(K, *, jitter=0.0, rhs_t=None):
    n = K.shape[1]
    K = torch.tril(K) + torch.tril(K, -1).transpose(1, 2)
    K = K + jitter * torch.eye(n, dtype=K.dtype)
    return _finish(_pad_identity(K, n), n, rhs_t)


def kernel_rows_padded(flat, xsg, xg, chol):
    B, m = xsg.shape[1], xsg.shape[2]
    n = xg.shape[2]
    out = torch.zeros(B, round_up(max(m, 1)), chol.n_pad, dtype=xg.dtype)
    out[:, :m, :n] = _eval(flat, xsg, xg, False)
    return out


def posterior_marginals(flat, xsg, xg, chol, half_y=None, want_sq=True, chunk=4096):
    V = kernel_rows_padded(flat, xsg, xg, chol)
    chol.solve_rows_(V)
    m = xsg.shape[2]
    dot = (V[0, :m] * half_y[None, :]).sum(-1) if half_y is not None else None
    sq = (V[0, :m] ** 2).sum(-1) if want_sq else None
    return dot, sq


class SparseAccumulator:
    """torch-CPU stand-in of ``ops.SparseAccumulator`` (same interface and accumulation semantics, chunk by chunk)."""

    def __init__(self, flat, zg, ch_z, method, chunk=16384):
        self.flat, self.zg, self.ch, self.method, self.chunk = flat, zg, ch_z, method, int(chunk)
        self.m, self.m_pad = ch_z.n, ch_z.n_pad
        self.A = torch.eye(self.m_pad, dtype=ch_z.dtype).reshape(1, self.m_pad, self.m_pad).clone()
        self.prod = torch.zeros(self.m_pad, dtype=ch_z.dtype)
        self.scalars = torch.zeros(3, dtype=ch_z.dtype)

    def add(self, xg_chunk, kdiag, kn, ybar):
        c = xg_chunk.shape[2]
        Wt = torch.zeros(1, c, self.m_pad, dtype=self.ch.dtype)
        Wt[:, :, : self.m] = _eval(self.flat, xg_chunk, self.zg, False)
        self.ch.solve_rows_(Wt)
        W = Wt[0].T  # [m_pad, c]
        kn = kn.clone()
        if self.method in ("vfe", "fitc"):
            corr = kdiag - (W * W).sum(0)
            if self.method == "vfe":
                self.scalars[2] += (corr / kn).sum()
            else:
                kn = kn + corr
        Ws = W / kn
        upd = Ws @ W.T
        tr = torch.arange(self.m_pad)[:, None] // TILE
        tc = torch.arange(self.m_pad)[None, :] // TILE
        self.A[0] += torch.where(tc <= tr, upd, torch.zeros_like(upd))  # lower 128-tiles only, like the SYRK
        self.prod += Ws @ ybar
        self.scalars[0] += torch.log(2 * math.pi * kn).sum()
        self.scalars[1] += (ybar * ybar / kn).sum()


def launch_count(reset=False):
    return 0


product_slices = real_ops.product_slices


def install(monkeypatch):
    """Swap the CUDA ops for this module and pin the compute device to the CPU."""
    import sys

    import stheno_b200
    from stheno_b200 import _util, autograd, kernels, matrix, pathwise
    from stheno_b200 import random as random_mod
    from stheno_b200.model import observations

    me = sys.modules[__name__]
    monkeypatch.setattr(_util, "_device_fn", lambda: torch.device("cpu"))
    # autograd and pathwise too (imported here, before the swap): a module first imported while the stand-ins are installed
    # would keep them after the test, and a GPU test later in the session would run on them
    for mod in (kernels, matrix, observations, random_mod, autograd, pathwise, stheno_b200):
        monkeypatch.setattr(mod, "ops", me, raising=False)
