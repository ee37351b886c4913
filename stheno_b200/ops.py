"""Tensor-level operations of the GP hot path, executed by the hand-written sm_90a kernels of ``libgpk``.

Everything here takes and returns CUDA ``torch`` tensors (PyTorch = device memory + streams; the arithmetic is
in ``csrc/*.cu``).  There is no CPU implementation: calling an op with a CPU tensor raises.

Storage conventions (see ``include/gpk.h``): row-major, batch-major ``[B, rows, cols]``; matrices that get
factorised live in a workspace ``W[B, n_pad + extra, n_pad]`` padded to multiples of 128 with the identity, the
``extra`` rows below the matrix carrying right-hand sides ``b^T`` that leave the factorisation as ``(L^-1 b)^T``.
"""
import ctypes
import math
import threading

import torch

from . import _lib
from ._lib import KIND, KM_LOWER, KM_PAD_IDENTITY, KM_PAD_ZERO, KM_SAME, GpkError, KernelDesc, check

__all__ = [
    "FlatKernel",
    "Chol",
    "round_up",
    "kernel_matrix",
    "kernel_diag",
    "chol_from_kernel",
    "chol_from_dense",
    "gemm_nt",
    "launch_count",
]

TILE = 128


def round_up(n, m=TILE):
    return (int(n) + m - 1) // m * m


def _suffix(dtype):
    if dtype == torch.float64:
        return "f64"
    if dtype == torch.float32:
        return "f32"
    raise TypeError(f"stheno_b200 computes in float64 or float32, got {dtype}")


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "stheno_b200.ops: CUDA tensor required -- the hot path runs only on the sm_90a kernels "
                "(there is no CPU fallback)"
            )


def _fn(name, dtype):
    """``name_f64`` / ``name_f32`` of libgpk.  An fp64 call that leaves out the emulation arguments ``(slices, ws, ws_bytes)``
    before the stream runs on the fp64 tensor cores, as with ``(0, NULL, 0)``."""
    fn = getattr(_lib.load(), f"{name}_{_suffix(dtype)}")
    if dtype != torch.float64 or "OZ" not in _lib._SIGNATURES.get(name, ()):
        return fn
    native = len(fn.argtypes) - 3
    return lambda *args: fn(*args[:-1], 0, None, 0, args[-1]) if len(args) == native else fn(*args)


def launch_count(reset=False):
    lib = _lib.load()
    c = int(lib.gpk_launch_count())
    if reset:
        lib.gpk_launch_count_reset()
    return c


class FlatKernel:
    """A kernel flattened to a sum of products of elementary kernels on pre-stretched inputs:
    ``sum_t coef_t * prod_f kind_f(x / scale[group_f], y / scale[group_f])``.

    ``terms`` is a list of ``(coef: float, [(kind: str, group: int), ...])``."""

    def __init__(self, terms, n_groups):
        # a factor is (kind, group) or (kind, group, param) -- param = the shape parameter of kinds that have one (rq: alpha)
        self.terms = [(float(c), [tuple([str(f[0]), int(f[1])] + [float(v) for v in f[2:3]]) for f in fs]) for c, fs in terms]
        self.n_groups = max(int(n_groups), 1)
        if len(self.terms) > _lib.GPK_MAX_TERMS:
            raise GpkError(f"kernel expands to {len(self.terms)} product terms (limit {_lib.GPK_MAX_TERMS})")
        if sum(len(fs) for _, fs in self.terms) > _lib.GPK_MAX_FACTORS:
            raise GpkError(f"kernel has more than {_lib.GPK_MAX_FACTORS} elementary factors")
        if self.n_groups > _lib.GPK_MAX_GROUPS:
            raise GpkError(f"kernel uses more than {_lib.GPK_MAX_GROUPS} distinct length scales")

    def desc(self):
        d = KernelDesc()
        d.n_terms = len(self.terms)
        d.n_groups = self.n_groups
        f = 0
        for t, (coef, fs) in enumerate(self.terms):
            d.term_begin[t] = f
            d.coef[t] = coef
            for fac in fs:
                d.fac_kind[f] = KIND[fac[0]]
                d.fac_group[f] = fac[1]
                d.fac_param[f] = fac[2] if len(fac) > 2 else 0.0
                f += 1
        d.term_begin[len(self.terms)] = f
        return d


def _check_groups(xg, flat):
    if xg.dim() != 4:
        raise ValueError("scaled inputs must have shape [groups, batch, n, d]")
    if xg.shape[0] < flat.n_groups:
        raise ValueError("not enough input groups for the kernel")


def _km_launch(flat, xg, yg, n, n2, d, flags, noise_scalar, noise_vec, jitter, out, ldo, o_bstride, batch):
    _require_cuda(xg, yg, out, noise_vec)
    xg = xg.contiguous()
    yg = xg if yg is xg else yg.contiguous()
    if noise_vec is not None:
        noise_vec = noise_vec.contiguous()
    desc = flat.desc()
    rc = _fn("gpk_kernel_matrix", out.dtype)(
        ctypes.byref(desc), _ptr(xg), xg.stride(0), xg.stride(1), n, _ptr(yg), yg.stride(0), yg.stride(1), n2, d,
        float(noise_scalar), _ptr(noise_vec), (noise_vec.stride(0) if noise_vec is not None else 0), float(jitter),
        flags, _ptr(out), ldo, o_bstride, batch, _stream(),
    )
    check(rc, "gpk_kernel_matrix")


def kernel_matrix(flat, xg, yg=None, *, same=None, noise_scalar=0.0, noise_vec=None, jitter=0.0):
    """Full ``[B, n, n2]`` kernel matrix ``k(x, y)`` (+ noise on the diagonal when ``same``).

    ``xg``/``yg``: ``[G, B, n, d]`` pre-stretched inputs; ``yg=None`` means the same object as ``xg``."""
    _check_groups(xg, flat)
    if yg is None:
        yg = xg
        same = True if same is None else same
    same = bool(same)
    B, n, d = xg.shape[1], xg.shape[2], xg.shape[3]
    n2 = yg.shape[2]
    out = torch.empty(B, n, n2, device=xg.device, dtype=xg.dtype)
    if n == 0 or n2 == 0:
        return out
    _km_launch(flat, xg, yg, n, n2, d, KM_SAME if same else 0, noise_scalar, noise_vec, jitter, out, n2, n * n2, B)
    return out


def kernel_diag(flat, xg, yg=None, *, same=None):
    """``k.elwise(x, y)`` -> ``[B, n]``."""
    _check_groups(xg, flat)
    if yg is None:
        yg, same = xg, (True if same is None else same)
    _require_cuda(xg, yg)
    xg = xg.contiguous()
    yg = xg if yg is xg else yg.contiguous()
    B, n, d = xg.shape[1], xg.shape[2], xg.shape[3]
    out = torch.empty(B, n, device=xg.device, dtype=xg.dtype)
    if n == 0:
        return out
    desc = flat.desc()
    rc = _fn("gpk_kernel_diag", xg.dtype)(
        ctypes.byref(desc), _ptr(xg), xg.stride(0), xg.stride(1), _ptr(yg), yg.stride(0), yg.stride(1), n, d,
        1 if same else 0, _ptr(out), n, B, _stream(),
    )
    check(rc, "gpk_kernel_diag")
    return out


def kernel_cross_bwd(flat, xsg, xg, *, W=None, r=None, u=None, v=None, gdiag=None, term_sum=None, grad_xsg=None,
                     grad_xg=None, param_sum=None):
    """Rectangular K1-backward (``gpk_kernel_cross_bwd``) of ``K = k(x*, x)`` ``[B, m, n]`` for the upstream gradient
    ``G_ij = r_i W_ij + u_i v_j`` (+ ``gdiag_i`` on ``k(x*_i, x*_i)``).  ``W``: ``[B, >= m, ldw]`` with a unit inner stride;
    ``r``, ``u``, ``gdiag``: ``[B, m]``; ``v``: ``[B, n]``.  The outputs ``term_sum [B, GPK_MAX_TERMS]``, ``grad_xsg`` (like
    ``xsg``), ``grad_xg`` (like ``xg``) and ``param_sum [B, GPK_MAX_FACTORS]`` (the gradient of every factor's shape
    parameter, RQ's alpha) are accumulated into; pass the ones wanted (None: not formed)."""
    _check_groups(xsg, flat)
    _check_groups(xg, flat)
    _require_cuda(xsg, xg, W, r, u, v, gdiag, term_sum, grad_xsg, grad_xg, param_sum)
    for t, like in ((grad_xsg, xsg), (grad_xg, xg)):
        if t is not None and (t.shape != like.shape or not t.is_contiguous()):
            raise ValueError("kernel_cross_bwd: gradient outputs must be contiguous and shaped like their inputs")
    xsg, xg = xsg.contiguous(), xg.contiguous()
    B, m, d = xsg.shape[1], xsg.shape[2], xsg.shape[3]
    n = xg.shape[2]
    if W is not None and W.stride(2) != 1:
        W = W.contiguous()
    r, u, v, gdiag = [None if t is None else t.contiguous() for t in (r, u, v, gdiag)]
    desc = flat.desc()
    rc = _fn("gpk_kernel_cross_bwd", xsg.dtype)(
        ctypes.byref(desc), _ptr(xsg), xsg.stride(0), xsg.stride(1), m, _ptr(xg), xg.stride(0), xg.stride(1), n, d,
        _ptr(W), (W.stride(1) if W is not None else 0), (W.stride(0) if W is not None else 0), _ptr(r), _ptr(u), _ptr(v),
        _ptr(gdiag), _ptr(term_sum), _ptr(grad_xsg), _ptr(grad_xg), _ptr(param_sum), B, _stream(),
    )
    check(rc, "gpk_kernel_cross_bwd")


def gemm_nt(A, Bm, C=None, *, alpha=1.0, beta=0.0, lower=False):
    """``C = beta * C + alpha * A @ Bm^T`` on padded ``[B, M, K]`` / ``[B, N, K]`` tensors (views with a unit inner
    stride are fine).  Returns ``C``."""
    _require_cuda(A, Bm, C)
    Bn, M, K = A.shape
    N = Bm.shape[1]
    if C is None:
        C = torch.empty(Bn, M, N, device=A.device, dtype=A.dtype)
        beta = 0.0
    for t in (A, Bm, C):
        if t.stride(2) != 1:
            raise ValueError("gemm_nt needs a unit inner stride")
    em = _emulation(A.dtype, A.device, lambda lib, s: lib.gpk_gemm_nt_oz_ws_bytes(M, N, K, s) if Bn == 1 else 0)
    rc = _fn("gpk_gemm_nt", A.dtype)(
        M, N, K, alpha, _ptr(A), A.stride(1), A.stride(0), _ptr(Bm), Bm.stride(1), Bm.stride(0), beta, _ptr(C),
        C.stride(1), C.stride(0), 1 if lower else 0, Bn, *em, _stream(),
    )
    check(rc, "gpk_gemm_nt")
    return C


def feature_eval(x, omega, b, amp, W, out=None, chunk=1 << 20):
    """``out[i, s] (+)= sum_j W[s, j] amp[j] cos(x_i . omega_j + b_j)`` (``gpk_feature_eval``): ``x [n, d]``, ``omega [F, d]``,
    ``b, amp [F]``, ``W [num, F]`` -> ``[n, num]``.  With ``out`` (a ``[n, num]`` tensor with a unit inner stride) the sum is
    added to it, else a new tensor is returned.  Rows are launched ``chunk`` at a time; the ``n x F`` features are never held."""
    _require_cuda(x, omega, b, amp, W, out)
    x, omega, b, amp, W = [t.contiguous() for t in (x, omega, b, amp, W)]
    n, d = x.shape
    F, num = omega.shape[0], W.shape[0]
    if omega.shape[1] != d or b.shape != (F,) or amp.shape != (F,) or W.shape[1] != F:
        raise ValueError("feature_eval: shapes do not match")
    if any(t.dtype != x.dtype for t in (omega, b, amp, W, out) if t is not None):
        raise TypeError("feature_eval: x, omega, b, amp, W and out must share one dtype")
    accumulate = out is not None
    if out is None:
        out = torch.empty(n, num, device=x.device, dtype=x.dtype)
    elif out.shape != (n, num) or out.stride(1) != 1:
        raise ValueError("feature_eval: out must be [n, num] with a unit inner stride")
    fn = _fn("gpk_feature_eval", x.dtype)
    for a in range(0, n, chunk):
        c = min(n, a + chunk) - a
        rc = fn(_ptr(x[a]), d, c, d, _ptr(omega), _ptr(b), _ptr(amp), F, _ptr(W), F, num, _ptr(out[a]), out.stride(0),
                1 if accumulate else 0, _stream())
        check(rc, "gpk_feature_eval")
    return out


def feature_eval_bwd(x, omega, b, amp, W, G, out=None, chunk=1 << 20):
    """The gradient in ``x`` of ``sum_is G[i, s] feature_eval(x, omega, b, amp, W)[i, s]`` (``gpk_feature_eval_bwd``):
    ``-sum_j c_ij sin(x_i . omega_j + b_j) omega_j`` with ``c_ij = amp_j sum_s G[i, s] W[s, j]``; ``G [n, num]`` -> ``[n, d]``.
    With ``out`` (a ``[n, d]`` tensor with a unit inner stride) the gradient is added to it, else a new tensor is returned.
    Rows are launched ``chunk`` at a time; neither the ``n x F`` features nor ``c`` are held."""
    _require_cuda(x, omega, b, amp, W, G, out)
    x, omega, b, amp, W, G = [t.contiguous() for t in (x, omega, b, amp, W, G)]
    n, d = x.shape
    F, num = omega.shape[0], W.shape[0]
    if omega.shape[1] != d or b.shape != (F,) or amp.shape != (F,) or W.shape[1] != F or G.shape != (n, num):
        raise ValueError("feature_eval_bwd: shapes do not match")
    if any(t.dtype != x.dtype for t in (omega, b, amp, W, G, out) if t is not None):
        raise TypeError("feature_eval_bwd: x, omega, b, amp, W, G and out must share one dtype")
    accumulate = out is not None
    if out is None:
        out = (torch.zeros if F == 0 else torch.empty)(n, d, device=x.device, dtype=x.dtype)
    elif out.shape != (n, d) or out.stride(1) != 1:
        raise ValueError("feature_eval_bwd: out must be [n, d] with a unit inner stride")
    if F == 0:
        return out
    fn = _fn("gpk_feature_eval_bwd", x.dtype)
    for a in range(0, n, chunk):
        c = min(n, a + chunk) - a
        rc = fn(_ptr(x[a]), d, c, d, _ptr(omega), _ptr(b), _ptr(amp), F, _ptr(W), F, num, _ptr(G[a]), num, _ptr(out[a]),
                out.stride(0), 1 if accumulate else 0, _stream())
        check(rc, "gpk_feature_eval_bwd")
    return out


def _pad_copy(src, dst, rows, cols, rows_pad, cols_pad, diag_add, pad_identity):
    if src.stride(2) != 1:
        src = src.contiguous()
    rc = _fn("gpk_pad_copy", dst.dtype)(
        _ptr(src), src.stride(1), src.stride(0), rows, cols, _ptr(dst), dst.stride(1), dst.stride(0), rows_pad,
        cols_pad, float(diag_add), 1 if pad_identity else 0, dst.shape[0], _stream(),
    )
    check(rc, "gpk_pad_copy")


def symmetrize_(A, n):
    """Mirror the lower triangle of the leading ``n x n`` block into the upper one, in place."""
    rc = _fn("gpk_symmetrize", A.dtype)(_ptr(A), A.stride(1), A.stride(0), n, A.shape[0], _stream())
    check(rc, "gpk_symmetrize")
    return A


def transpose(src, rows, cols, out=None):
    """``out[B, cols, rows] = src[B, rows, cols]^T`` (leading block of possibly padded tensors)."""
    if src.stride(2) != 1:  # a transposed VIEW (e.g. a reversed cross-kernel): the kernels take a unit inner stride
        src = src.contiguous()
    if out is None:
        out = torch.empty(src.shape[0], cols, rows, device=src.device, dtype=src.dtype)
    rc = _fn("gpk_transpose", src.dtype)(
        _ptr(src), src.stride(1), src.stride(0), rows, cols, _ptr(out), out.stride(1), out.stride(0), src.shape[0],
        _stream(),
    )
    check(rc, "gpk_transpose")
    return out


def row_dot_sq(V, rows, n_cols, b=None, want_dot=True, want_sq=True):
    """Per-row ``<V[r, :n_cols], b>`` and ``|V[r, :n_cols]|^2`` of ``V[B, *, *]`` -> two ``[B, rows]`` tensors."""
    if V.stride(2) != 1:
        V = V.contiguous()
    Bn = V.shape[0]
    dot = torch.empty(Bn, rows, device=V.device, dtype=V.dtype) if (want_dot and b is not None) else None
    sq = torch.empty(Bn, rows, device=V.device, dtype=V.dtype) if want_sq else None
    if rows == 0:
        return dot, sq
    b_bs = 0
    if b is not None:
        b = b.contiguous()
        if b.dim() > 1 and b.shape[0] != Bn:  # one vector for a batch of row sets (the test-point sets of one problem)
            if b.shape[0] != 1:
                raise ValueError(f"row_dot_sq: {b.shape[0]} vectors against {Bn} row sets")
        elif b.dim() > 1:
            b_bs = b.stride(0)
    rc = _fn("gpk_row_dot_sq", V.dtype)(
        _ptr(V), V.stride(1), V.stride(0), rows, n_cols, _ptr(b), b_bs, _ptr(dot),
        _ptr(sq), rows, Bn, _stream(),
    )
    check(rc, "gpk_row_dot_sq")
    return dot, sq


class Chol:
    """Lower Cholesky factor ``L`` of ``K + jitter I`` in padded workspace storage, with fused right-hand sides.

    Attributes: ``W [B, n_pad + extra, n_pad]``, ``n``, ``n_pad``, ``k`` (number of fused right-hand sides),
    ``logdet [B]`` (= ``2 sum log diag L``), ``info [B]`` (int32; first non-positive pivot, 0 = ok)."""

    def __init__(self, W, n, k, logdet, info):
        self.W, self.n, self.k, self.logdet, self.info = W, int(n), int(k), logdet, info
        self.n_pad = W.shape[2]
        self.batch = W.shape[0]

    @property
    def dtype(self):
        return self.W.dtype

    @property
    def device(self):
        return self.W.device

    def check(self):
        """Raise ``torch.linalg.LinAlgError`` if a pivot was non-positive (forces a host sync)."""
        bad = self.info.nonzero()
        if bad.numel():
            b = int(bad[0, 0])
            raise torch.linalg.LinAlgError(
                f"Cholesky: leading minor of order {int(self.info[b])} is not positive definite (batch {b})"
            )
        return self

    def L_padded(self):
        return self.W[:, : self.n_pad, :]

    def L(self):
        """Dense ``[B, n, n]`` lower-triangular factor (copy; strict upper triangle zeroed)."""
        return torch.tril(self.W[:, : self.n, : self.n])

    def L_lower_(self):
        """The padded factor ``[B, n_pad, n_pad]`` with its strict upper triangle zeroed IN PLACE (no copy; done once): the
        form products with ``L`` need (``L eps`` of sampling, ``L_z A L_z^T``).  Nothing else reads the upper triangle."""
        if not getattr(self, "_upper_zeroed", False):
            self.W[:, : self.n_pad, :].tril_()
            self._upper_zeroed = True
        return self.W[:, : self.n_pad, :]

    def rhs_half(self):
        """``(L^-1 rhs)^T`` for the fused right-hand sides: ``[B, k, n]`` (a view)."""
        return self.W[:, self.n_pad : self.n_pad + self.k, : self.n]

    def logpdf(self):
        """``-0.5 (logdet + n log 2 pi + |L^-1 rhs_c|^2)`` for every fused right-hand side -> ``[B, k]``."""
        if self.k == 0:
            raise ValueError("no right-hand side was fused into this factorisation")
        out = torch.empty(self.batch, self.k, device=self.device, dtype=self.dtype)
        rows = self.W[:, self.n_pad :, :]
        rc = _fn("gpk_logpdf_finish", self.dtype)(
            _ptr(rows), rows.stride(1), rows.stride(0), self.n, self.n_pad, self.k, _ptr(self.logdet), _ptr(out),
            self.batch, _stream(),
        )
        check(rc, "gpk_logpdf_finish")
        return out

    def new_rows(self, rows, zero=True):
        """A padded ``[B, round_up(rows), n_pad]`` buffer for :meth:`solve_rows_`."""
        f = torch.zeros if zero else torch.empty
        return f(self.batch, round_up(rows), self.n_pad, device=self.device, dtype=self.dtype)

    def solve_rows_(self, Bt):
        """In place ``Bt <- Bt L^-T`` on a padded ``[B, rows_pad, n_pad]`` buffer: row r becomes ``(L^-1 b_r)^T``."""
        _require_cuda(Bt)
        if Bt.shape[2] != self.n_pad or Bt.shape[1] % TILE or Bt.stride(2) != 1:
            raise ValueError("solve_rows_ needs a padded [B, rows_pad, n_pad] buffer")
        Lp = self.L_padded()
        rows, n_pad, batch = Bt.shape[1], self.n_pad, Bt.shape[0]
        em = _emulation(self.dtype, self.device, lambda lib, s: lib.gpk_trsm_right_oz_ws_bytes(n_pad, rows, s) if batch == 1 else 0)
        rc = _fn("gpk_trsm_right", self.dtype)(
            _ptr(Lp), Lp.stride(1), self._batch_stride(Bt), n_pad, _ptr(Bt), Bt.stride(1), Bt.stride(0), rows, batch, *em,
            _stream(),
        )
        check(rc, "gpk_trsm_right")
        return Bt

    def solve_rows_t_(self, Bt):
        """In place ``Bt <- Bt L^-1``: row r becomes ``(L^-T b_r)^T`` (backward substitution)."""
        _require_cuda(Bt)
        Lp = self.L_padded()
        rc = _fn("gpk_trsm_right_t", self.dtype)(
            _ptr(Lp), Lp.stride(1), self._batch_stride(Bt), self.n_pad, _ptr(Bt), Bt.stride(1), Bt.stride(0), Bt.shape[1],
            Bt.shape[0], _stream(),
        )
        check(rc, "gpk_trsm_right_t")
        return Bt

    def _batch_stride(self, Bt):
        """The batch stride of ``L`` for the row buffer ``Bt``: one factor solves every member of a batch of row sets (the
        test-point sets of one problem) through stride 0; otherwise ``Bt`` has one member per factor."""
        if Bt.shape[0] == self.batch:
            return self.L_padded().stride(0)
        if self.batch != 1:
            raise ValueError(f"row buffer batch {Bt.shape[0]} against {self.batch} factors")
        return 0

    def solve_many_rows_t_(self, Bt, leaf=1024, panel=1024):
        """:meth:`solve_rows_t_` for many rows (a chunk of test points).  ``gpk_trsm_right_t`` is a CUDA-core backward
        substitution that re-reads ``L`` for every row; here ``L`` is split recursively, the trailing block is solved first
        and its product with the off-diagonal block is subtracted on the tensor-core GEMM (through transposed copies of
        ``panel`` columns of that block), so only diagonal blocks of at most ``leaf`` columns go through the substitution."""
        _require_cuda(Bt)
        if Bt.shape[2] != self.n_pad or Bt.shape[1] % TILE or Bt.stride(2) != 1:
            raise ValueError("solve_many_rows_t_ needs a padded [B, rows_pad, n_pad] buffer")
        if Bt.shape[0] != self.batch:
            raise ValueError(f"solve_many_rows_t_: row buffer batch {Bt.shape[0]} against {self.batch} factors")
        self._solve_t_block(Bt, 0, self.n_pad, leaf, panel)
        return Bt

    def _solve_t_block(self, Bt, a, b, leaf, panel):
        Lp = self.L_padded()
        if b - a <= leaf:
            L, X = Lp[:, a:b, a:b], Bt[:, :, a:b]
            rc = _fn("gpk_trsm_right_t", self.dtype)(
                _ptr(L), L.stride(1), L.stride(0), b - a, _ptr(X), X.stride(1), X.stride(0), Bt.shape[1], self.batch,
                _stream(),
            )
            check(rc, "gpk_trsm_right_t")
            return
        m = a + round_up((b - a) // 2)
        self._solve_t_block(Bt, m, b, leaf, panel)  # X2 L22 = B2
        for p0 in range(a, m, panel):  # B1 -= X2 L21, `panel` columns of L21 at a time
            p1 = min(m, p0 + panel)
            L21t = transpose(Lp[:, m:b, p0:p1], b - m, p1 - p0)
            gemm_nt(Bt[:, :, m:b], L21t, Bt[:, :, p0:p1], alpha=-1.0, beta=1.0)
        self._solve_t_block(Bt, a, m, leaf, panel)  # X1 L11 = B1

    def inverse_diag(self, chunk=2048):
        """``diag (L L^T)^-1`` ``[B, n]``: the squared norms of the rows of ``L^-T``.  Row ``r`` of ``L^-T`` is
        ``(L^-1 e_r)^T``, zero before column ``r``, so a chunk of identity rows from a 128-aligned ``r0`` is solved against
        the trailing factor ``L[r0:, r0:]`` alone: ``n^3 / 3`` flops in all and one ``[B, chunk, n_pad]`` buffer, never the
        ``n_pad^2`` inverse."""
        _require_cuda(self.W)
        Lp, n, n_pad, batch = self.L_padded(), self.n, self.n_pad, self.batch
        chunk = min(round_up(chunk), n_pad)
        out = torch.empty(batch, n, device=self.device, dtype=self.dtype)
        buf = torch.empty(batch, chunk, n_pad, device=self.device, dtype=self.dtype)
        fn = _fn("gpk_trsm_right", self.dtype)
        for r0 in range(0, n, chunk):
            rows, m = min(chunk, n_pad - r0), n_pad - r0
            L, X = Lp[:, r0:, r0:], buf[:, :rows, :m]
            X.zero_()
            X.diagonal(dim1=1, dim2=2).fill_(1.0)
            em = _emulation(self.dtype, self.device, lambda lib, s: lib.gpk_trsm_right_oz_ws_bytes(m, rows, s) if batch == 1 else 0)
            rc = fn(_ptr(L), L.stride(1), L.stride(0), m, _ptr(X), X.stride(1), X.stride(0), rows, batch, *em, _stream())
            check(rc, "gpk_trsm_right")
            r1 = min(n, r0 + rows)
            out[:, r0:r1] = row_dot_sq(X, r1 - r0, m, want_dot=False)[1]
        return out

    def loo(self, r, want_mean=True):
        """Leave-one-out quantities of ``N(0, L L^T)`` at the fused right-hand sides ``r [B, k, n]`` (the rows this factor
        was built with): ``(mean [B, k, n] (the LOO mean minus the prior mean; None without want_mean), var [B, n],
        lp [B, k], alpha [B, k, n], c [B, n])`` with ``alpha = K^-1 r`` and ``c = diag K^-1`` (:func:`loo_finish`)."""
        k, n = self.k, self.n
        arows = self.new_rows(k)
        arows[:, :k, :n] = self.rhs_half()
        self.solve_rows_t_(arows)
        alpha = arows[:, :k, :n]
        c = self.inverse_diag()
        mean, var, lp = loo_finish(c, alpha, r, want_mean=want_mean)
        return mean, var, lp, alpha, c

    def cv(self, r, sizes, want_mean=True, chunk=2048):
        """Multi-fold cross-validation quantities of ``N(0, L L^T)`` at the fused right-hand sides ``r [B, k, n]``, the
        entries in fold order (fold ``f`` is the ``sizes[f]`` entries after the folds before it).  With ``C = (L L^T)^-1``
        and ``alpha = C r``: ``(mean [B, k, n] (the CV mean minus the prior mean; None without want_mean), var [B, n],
        lp [B, k], folds)`` where ``folds`` (:class:`CVFolds`) holds ``alpha``, the residuals ``e`` and the factors of
        the blocks ``C_II`` for the backward (:func:`cv_finish`)."""
        k, n = self.k, self.n
        arows = self.new_rows(k)
        arows[:, :k, :n] = self.rhs_half()
        self.solve_rows_t_(arows)
        alpha = arows[:, :k, :n]
        folds = CVFolds(self, sizes, alpha, chunk)
        mean, var, lp = cv_finish(folds.offsets, folds.e, folds.z, folds.v, folds.ldet, r, want_mean=want_mean)
        return mean, var, lp, folds

    def half_solve(self, bt):
        """``bt [B, m, n]`` (rows = right-hand sides) -> ``(L^-1 b)^T [B, m, n]``."""
        m = bt.shape[1]
        buf = self.new_rows(m)
        buf[:, :m, : self.n] = bt
        self.solve_rows_(buf)
        return buf[:, :m, : self.n]

    def full_solve(self, bt):
        """``bt [B, m, n]`` -> ``(K^-1 b)^T [B, m, n]``."""
        m = bt.shape[1]
        buf = self.new_rows(m)
        buf[:, :m, : self.n] = bt
        self.solve_rows_(buf)
        self.solve_rows_t_(buf)
        return buf[:, :m, : self.n]


def loo_finish(c, alpha, r=None, g=None, *, want_mean=True, want_var=True, want_lp=True):
    """``gpk_loo_finish`` on ``c [B, n]`` (``diag K^-1``), ``alpha [B, k, n]`` (``K^-1 r``, rows with a unit inner stride)
    and ``r [B, k, n]``.  Without ``g``: ``(mean [B, k, n], var [B, n], lp [B, k])`` with ``mean = r - alpha / c``,
    ``var = 1 / c`` and ``lp`` the summed leave-one-out log densities (None for those not wanted).  With the upstream
    gradient ``g [B, k]`` of ``lp``: the backward weights ``(P [B, n], q [B, k, n])``."""
    _require_cuda(c, alpha, r, g)
    Bn, k, n = alpha.shape
    if c.shape != (Bn, n) or (r is not None and r.shape != (Bn, k, n)) or (g is not None and g.shape != (Bn, k)):
        raise ValueError("loo_finish: shapes do not match")
    if c.stride(1) != 1:
        c = c.contiguous()
    if alpha.stride(2) != 1:
        alpha = alpha.contiguous()
    if r is not None and r.stride(2) != 1:
        r = r.contiguous()
    new = lambda *shape: torch.empty(*shape, device=c.device, dtype=c.dtype)  # noqa: E731
    if g is not None:
        outs = (None, None, None, new(Bn, n), new(Bn, k, n))
        g = g.contiguous()
    else:
        if want_mean and r is None:
            raise ValueError("loo_finish: the mean needs r")
        outs = (new(Bn, k, n) if want_mean else None, new(Bn, n) if want_var else None, new(Bn, k) if want_lp else None,
                None, None)
    ld = lambda t: t.stride(1) if k > 1 else n  # noqa: E731  (a contiguous single row may report any row stride)
    rc = _fn("gpk_loo_finish", c.dtype)(
        _ptr(c), c.stride(0), _ptr(alpha), ld(alpha), alpha.stride(0), _ptr(r), ld(r) if r is not None else 0,
        r.stride(0) if r is not None else 0, n, k, _ptr(g), *[_ptr(t) for t in outs], Bn, _stream(),
    )
    check(rc, "gpk_loo_finish")
    return outs[3:] if g is not None else outs[:3]


#: the batched factorisation launches one grid row per matrix: at most this many fold blocks per call
_MAX_FOLD_BATCH = 32768


class CVFolds:
    """The diagonal blocks ``C_II`` of ``C = (L L^T)^-1`` for consecutive folds of ``sizes`` entries, factorised, with
    ``alpha [B, k, n]`` (``C r``) as their right-hand sides.

    Rows of ``V = L^-T`` (``C = V V^T``) from a 128-aligned ``a`` need only the trailing factor ``L[a:, a:]``: identity rows
    are solved in chunks whose boundaries fall on fold boundaries (at least as tall as the largest fold they hold; one
    ``[B, rows, n_pad]`` buffer), and each fold's block ``V_I V_I^T`` is formed by the lower-tile GEMM straight into a
    workspace padded with the identity to ``p = round_up(n_f)``, ``alpha_I`` in its right-hand-side rows -- consecutive
    folds of one size in one batched GEMM.  Folds of one padded size are factorised as one batch: ``log det C_II``,
    ``z_I = L_I^-1 alpha_I``, the residuals ``e_I = C_II^-1 alpha_I`` and ``diag C_II^-1``.  Attributes (fold order):
    ``offsets`` (device int64 ``[F + 1]``), ``alpha``, ``e``, ``z`` ``[B, k, n]``, ``v [B, n]``, ``ldet [B, F]``; ``groups``:
    ``{p: (folds, [Chol of <= _MAX_FOLD_BATCH slots], idx)}`` with slot ``i * B + b`` = fold ``folds[i]``, problem ``b``, and
    ``idx [len(folds), p]`` the entry of each padded row (-1: padding)."""

    def __init__(self, ch, sizes, alpha, chunk=2048):
        self.sizes = [int(s) for s in sizes]
        off = [0]
        for s in self.sizes:
            off.append(off[-1] + s)
        if off[-1] != ch.n or min(self.sizes) < 1:
            raise ValueError("CVFolds: the fold sizes must be positive and add up to n")
        self.off, self.alpha, self.batch, self.n = off, alpha, ch.batch, ch.n
        self.offsets = torch.tensor(off, dtype=torch.int64, device=ch.device)
        self.pads = [round_up(s) for s in self.sizes]
        self.members = {}  # padded size -> its folds, in fold order
        for f, p in enumerate(self.pads):
            self.members.setdefault(p, []).append(f)
        self.factor(self.blocks(ch, chunk))

    def blocks(self, ch, chunk=2048):
        """The fold-block product: ``{p: W [G B, p + round_up(k), p]}``, the blocks ``C_II`` on the lower tiles of each slot
        (the padding not yet the identity) and ``alpha_I`` in its right-hand-side rows."""
        Bn, n_pad, off, sizes, pads = ch.batch, ch.n_pad, self.off, self.sizes, self.pads
        alpha = self.alpha
        k = alpha.shape[1]
        dev, dt = ch.device, ch.dtype
        F = len(sizes)
        slot, Ws, self.idxs = {}, {}, {}
        a_ext = torch.cat([alpha, torch.zeros(Bn, k, 1, dtype=dt, device=dev)], dim=2)  # entry -1 (padding) reads 0
        for p, fs in self.members.items():
            for i, f in enumerate(fs):
                slot[f] = i
            ar = torch.arange(p)
            nf = torch.tensor([sizes[f] for f in fs])
            idx = torch.where(ar[None, :] < nf[:, None], torch.tensor([off[f] for f in fs])[:, None] + ar[None, :], -1)
            self.idxs[p] = idx = idx.to(dev)
            W = torch.zeros(len(fs) * Bn, p + round_up(k), p, dtype=dt, device=dev)
            W[:, p : p + k, :] = a_ext[:, :, idx].permute(2, 0, 1, 3).reshape(len(fs) * Bn, k, p)
            Ws[p] = W
        plan, f = [], 0
        while f < F:
            a = off[f] // TILE * TILE
            g = f + 1
            while g < F and round_up(off[g + 1] - a) <= chunk:
                g += 1
            plan.append((a, f, g))
            f = g
        rows_max = max(round_up(off[g] - a) for a, _, g in plan) + TILE  # a fold's p rows from its start stay inside
        buf = torch.empty(Bn, rows_max, n_pad, dtype=dt, device=dev)
        fn = _fn("gpk_trsm_right", dt)
        Lp = ch.L_padded()
        for a, f0, f1 in plan:
            rows, m = round_up(off[f1] - a), n_pad - a
            X = buf[:, :, :m]
            X.zero_()
            X[:, :rows].diagonal(dim1=1, dim2=2).fill_(1.0)
            L = Lp[:, a:, a:]
            em = _emulation(dt, dev, lambda lib, s: lib.gpk_trsm_right_oz_ws_bytes(m, rows, s) if Bn == 1 else 0)
            rc = fn(_ptr(L), L.stride(1), L.stride(0), m, _ptr(X), X.stride(1), X.stride(0), rows, Bn, *em, _stream())
            check(rc, "gpk_trsm_right")
            i = f0
            while i < f1:  # runs of consecutive folds of one size: consecutive slots of one group
                j = i + 1
                while j < f1 and sizes[j] == sizes[i]:
                    j += 1
                nf, p, s0 = sizes[i], pads[i], slot[i]
                W = Ws[p]
                for b in range(Bn):  # fold t of the run: rows [off[i] + t nf - a, + p) of the chunk, slot (s0 + t) B + b
                    A = buf.as_strided((j - i, p, m), (nf * buf.stride(1), buf.stride(1), 1),
                                       b * buf.stride(0) + (off[i] - a) * buf.stride(1))
                    C = W.as_strided((j - i, p, p), (Bn * W.stride(0), W.stride(1), 1), (s0 * Bn + b) * W.stride(0))
                    gemm_nt(A, A, C, alpha=1.0, beta=0.0, lower=True)
                i = j
        return Ws

    def factor(self, Ws):
        """The fold factorisations, in place on the workspaces of :meth:`blocks`: the padding of each block back to the
        identity, then one batched factorisation per padded size and its solves; sets ``e``, ``z``, ``v``, ``ldet``,
        ``groups``."""
        Bn, n, k = self.batch, self.n, self.alpha.shape[1]
        dev, dt = self.alpha.device, self.alpha.dtype
        self.e = torch.zeros(Bn, k, n, dtype=dt, device=dev)
        self.z = torch.zeros(Bn, k, n, dtype=dt, device=dev)
        self.v = torch.empty(Bn, n, dtype=dt, device=dev)
        self.ldet = torch.empty(Bn, len(self.sizes), dtype=dt, device=dev)
        self.groups = {}
        for p, fs in self.members.items():
            W, idx = Ws.pop(p), self.idxs[p]
            G = len(fs)
            if any(self.sizes[f] < p for f in fs):
                nf = torch.tensor([self.sizes[f] for f in fs], device=dev).repeat_interleave(Bn)
                inside = torch.arange(p, device=dev)[None, :] < nf[:, None]
                W[:, :p, :].masked_fill_(~(inside[:, :, None] & inside[:, None, :]), 0.0)
                W[:, :p, :].diagonal(dim1=1, dim2=2).masked_fill_(~inside, 1.0)
            chols, es, zs, vs, lds = [], [], [], [], []
            for s0 in range(0, G * Bn, _MAX_FOLD_BATCH):
                cg = _potrf(W[s0 : s0 + _MAX_FOLD_BATCH], p, p, W.shape[1] - p, k)
                er = cg.new_rows(k)
                er[:, :k] = cg.rhs_half()
                cg.solve_rows_t_(er)
                chols.append(cg)
                es.append(er[:, :k])
                zs.append(cg.rhs_half())
                vs.append(cg.inverse_diag())
                lds.append(cg.logdet)
            self.groups[p] = (fs, chols, idx)
            pos = idx.reshape(-1)
            inside = pos >= 0
            pos = pos[inside]
            for dst, parts in ((self.e, es), (self.z, zs)):
                t = torch.cat(parts).reshape(G, Bn, k, p).permute(1, 2, 0, 3).reshape(Bn, k, G * p)
                dst[:, :, pos] = t[:, :, inside]
            t = torch.cat(vs).reshape(G, Bn, p).permute(1, 0, 2).reshape(Bn, G * p)
            self.v[:, pos] = t[:, inside]
            self.ldet[:, fs] = torch.cat(lds).reshape(G, Bn).t()

    def to_slots(self, t, p):
        """Entries ``t [B, c, n]`` (fold order) -> the padded rows of group ``p``'s slots ``[G B, p, c]`` (padding 0)."""
        fs, _, idx = self.groups[p]
        Bn, c = t.shape[0], t.shape[1]
        t_ext = torch.cat([t, torch.zeros(Bn, c, 1, dtype=t.dtype, device=t.device)], dim=2)
        return t_ext[:, :, idx].permute(2, 0, 3, 1).reshape(len(fs) * Bn, idx.shape[1], c)


def cv_finish(offsets, e, z=None, v=None, ldet=None, r=None, g=None, *, want_mean=True, want_var=True, want_lp=True):
    """``gpk_cv_finish`` on entries in fold order (fold ``f`` = ``[offsets[f], offsets[f + 1])``, ``offsets`` a device
    int64 ``[F + 1]``): the residuals ``e [B, k, n]`` (``C_II^-1 alpha_I``), ``z [B, k, n]`` (``L_I^-1 alpha_I``), ``v [B, n]``
    (``diag C_II^-1``), ``ldet [B, F]`` (``log det C_II``) and ``r [B, k, n]``.  Without ``g``: ``(mean [B, k, n], var [B, n],
    lp [B, k])`` with ``mean = r - e``, ``var = v`` and ``lp`` the summed fold log densities (None for those not wanted).
    With the upstream gradient ``g [B, k]`` of ``lp``: the backward weights ``(q [B, k, n], s [B, F])``, ``q = g e``,
    ``s = 1/2 sum_c g_c``."""
    _require_cuda(offsets, e, z, v, ldet, r, g)
    Bn, k, n = e.shape
    F = offsets.shape[0] - 1
    for t, shape in ((z, (Bn, k, n)), (r, (Bn, k, n)), (v, (Bn, n)), (ldet, (Bn, F)), (g, (Bn, k))):
        if t is not None and tuple(t.shape) != shape:
            raise ValueError("cv_finish: shapes do not match")
    e, z, v, ldet, r = [None if t is None else (t if t.stride(-1) == 1 else t.contiguous()) for t in (e, z, v, ldet, r)]
    new = lambda *shape: torch.empty(*shape, device=e.device, dtype=e.dtype)  # noqa: E731
    if g is not None:
        outs = (None, None, None, new(Bn, k, n), new(Bn, F))
        g = g.contiguous()
    else:
        if want_mean and r is None:
            raise ValueError("cv_finish: the mean needs r")
        outs = (new(Bn, k, n) if want_mean else None, new(Bn, n) if want_var else None, new(Bn, k) if want_lp else None,
                None, None)
    ld = lambda t: (t.stride(1) if k > 1 else n) if t is not None else 0  # noqa: E731
    bs = lambda t: t.stride(0) if t is not None else 0  # noqa: E731
    rc = _fn("gpk_cv_finish", e.dtype)(
        _ptr(offsets), F, _ptr(e), ld(e), bs(e), _ptr(z), ld(z), bs(z), _ptr(v), bs(v), _ptr(ldet), bs(ldet), _ptr(r), ld(r),
        bs(r), n, k, _ptr(g), *[_ptr(t) for t in outs], Bn, _stream(),
    )
    check(rc, "gpk_cv_finish")
    return outs[3:] if g is not None else outs[:3]


def _new_workspace(B, n, k, device, dtype, rhs_t):
    n_pad = round_up(max(n, 1))
    extra = round_up(k) if k > 0 else 0
    W = torch.empty(B, n_pad + extra, n_pad, device=device, dtype=dtype)
    if extra:
        W[:, n_pad:, :].zero_()
        W[:, n_pad : n_pad + k, :n] = rhs_t
    return W, n_pad, extra


def _potrf(W, n, n_pad, extra, k, well_conditioned=False):
    B = W.shape[0]
    logdet = torch.zeros(B, device=W.device, dtype=W.dtype)
    info = torch.zeros(B, device=W.device, dtype=torch.int32)
    from . import B as _Bns

    if W.dtype == torch.float64 and B == 1 and getattr(_Bns, "precision", "fp64") == "tf32x3" and n_pad > 512:
        # opt-in mixed precision: trailing updates on the wgmma tensor cores (3xTF32) from an fp32 panel copy
        ws = torch.empty((n_pad + extra) * 512, device=W.device, dtype=torch.float32)
        rc = _lib.load().gpk_potrf_f64_tf32x3(_ptr(W), W.stride(1), W.stride(0), n_pad, extra, _ptr(logdet), _ptr(info),
                                              B, _ptr(ws), ws.numel(), _stream())
        check(rc, "gpk_potrf_f64_tf32x3")
        return Chol(W, n, k, logdet, info)
    em = _emulation(W.dtype, W.device, lambda lib, s: lib.gpk_potrf_oz_ws_bytes(n_pad, extra, s) if B == 1 else 0,
                    well_conditioned)
    rc = _fn("gpk_potrf", W.dtype)(_ptr(W), W.stride(1), W.stride(0), n_pad, extra, _ptr(logdet), _ptr(info), B, *em,
                                   _stream())
    check(rc, "gpk_potrf")
    return Chol(W, n, k, logdet, info)


#: the slice count of ``product_slices`` for the calling host thread (8 outside a ``with`` block)
_PRODUCT_SLICES = threading.local()


class product_slices:
    """``with ops.product_slices(7): ...`` -- inside the block, ``B.precision = "auto"`` emulates the large products and solves
    with that many int8 slices instead of 8.  Used by the analytic log-pdf backward, which forms ``K^-1`` from one big
    solve and one big product, 1.3x faster with 7 slices.  Measured against torch fp64 autograd
    (``tests/test_logpdf_grad_paths.py``), 7-slice solves and products on an 8-slice factor keep the gradients within a
    small factor of native fp64's error from noise 1e-2 to 1e-6 of the variance; a 7-slice FACTOR does not (up to 45x
    at 1e-2), so a factorisation whose gradient is taken is asked for with ``full_precision``.  The setting belongs to the
    host thread that enters the block: calls made meanwhile on other threads keep their own."""

    def __init__(self, slices):
        self.slices = int(slices)

    def __enter__(self):
        self.prev = getattr(_PRODUCT_SLICES, "auto", 8)
        _PRODUCT_SLICES.auto = self.slices

    def __exit__(self, *exc):
        _PRODUCT_SLICES.auto = self.prev


def _oz_slices(well_conditioned=False):
    """``B.precision`` -> number of int8 slices of the emulated large fp64 updates (0: native fp64 tensor cores only).

    "auto" uses 8 slices (56-bit operands >= fp64's 53: the accuracy of the fp64 tensor-core kernel itself) everywhere EXCEPT
    the one place where 7 slices (49-bit operands, product error ~3e-14) are measured to stay three orders inside the 1e-10
    parity bar: the factorisation inside a stand-alone ``logpdf`` of a matrix that is well conditioned BY CONSTRUCTION (a known
    scalar noise of at least 1e-3 of the kernel's variance on the diagonal) -- the log-pdf is a well-conditioned functional of
    the factor (log-det and one quadratic form).  Measured (round 2, ``profiles/r02_conditioning_sweep.txt`` and the full-size
    oracle tests): at n = 16384, noise 0.1 the 7-slice log-pdf is 3e-14 from the CPU oracle, but the ELEMENTS of a posterior
    mean computed from a 7-slice factor and 7-slice solves are up to 2e-10 off (1.2e-10 of the largest element) -- so
    factorisations that serve a posterior (``Observations.K_x``) and every triangular solve / product use 8 slices; and the
    7-slice log-pdf error grows like 1.5e-14 / (noise / variance), reaching 1e-10 near 1e-4 -- hence the 1e-3 threshold."""
    from . import B as _Bns

    mode = getattr(_Bns, "precision", "auto")
    if mode == "auto":
        return 7 if well_conditioned else getattr(_PRODUCT_SLICES, "auto", 8)
    return {"int8x5": 5, "int8x6": 6, "int8x7": 7, "int8x8": 8}.get(mode, 0)


def _well_conditioned(flat, noise_scalar, noise_vec, jitter):
    """True when ``k(x, x) + noise`` is well conditioned by construction: scalar diagonal term >= 1e-3 of the kernel's
    variance scale (sum of |coefficients| of the bounded stationary terms; anything with a Linear factor is unbounded)."""
    if noise_vec is not None:
        return False
    scale = 0.0
    for coef, fs in flat.terms:
        if any(f[0] == "linear" for f in fs):
            return False
        if all(f[0] == "delta" for f in fs):
            continue  # a Delta term only adds to the diagonal
        scale += abs(coef)
    diag = float(noise_scalar) + float(jitter) + sum(c for c, fs in flat.terms if fs and all(f[0] == "delta" for f in fs) and c > 0)
    return diag >= 1e-3 * max(scale, 1e-300)


#: scratch of the int8-slice emulation per (device, stream): the calls on one stream are ordered by it, calls on two streams
#: may run at the same time, so each stream has its own
_OZ_SCRATCH = {}
_OZ_SCRATCH_MAX_BYTES = 8 << 30


def _emulation(dtype, device, need, well_conditioned=False):
    """The trailing ``(slices, ws, ws_bytes)`` arguments of an fp64 entry point (none for fp32): ``B.precision``'s slice count
    (:func:`_oz_slices`) and the scratch of the current stream, grown on demand to ``need(lib, slices)`` bytes -- the library's
    size query for the call -- and capped (larger requests stay on the fp64 tensor cores).  ``(0, NULL, 0)`` when the slice
    count or the need is 0: the call runs on the fp64 tensor cores.  The scratch is allocated on the stream that uses it, so
    the buffer a growth replaces returns to that stream's pool, reused only by work ordered after the calls that read it."""
    if dtype != torch.float64:
        return ()
    slices = _oz_slices(well_conditioned)
    need_bytes = min(int(need(_lib.load(), slices)), _OZ_SCRATCH_MAX_BYTES) if slices else 0
    if not need_bytes:
        return 0, None, 0
    stream = torch.cuda.current_stream(device)
    key = (stream.device_index, stream.cuda_stream)
    buf = _OZ_SCRATCH.get(key)
    if buf is None or buf.numel() < need_bytes:
        buf = _OZ_SCRATCH[key] = _aligned_bytes(max(need_bytes, 64 << 20), stream.device)
    return slices, _ptr(buf), buf.numel()


def release_scratch(stream=None):
    """Drop the emulation scratch of ``stream`` (a ``torch.cuda.Stream``; every stream's when None), for a stream that will not
    run emulated calls again.  Safe while work that uses it is still queued: the buffer goes back to the pool of the stream it
    was allocated on and is reused only by work ordered after that; ``torch.cuda.empty_cache()`` then returns it to the
    device."""
    if stream is None:
        _OZ_SCRATCH.clear()
    else:
        _OZ_SCRATCH.pop((stream.device_index, stream.cuda_stream), None)


def _aligned_bytes(nbytes, device, align=1024):
    buf = torch.empty(int(nbytes) + align, device=device, dtype=torch.uint8)
    off = (-buf.data_ptr()) % align
    return buf[off : off + int(nbytes)]


def gemm_nt_oz(A, Bm, C=None, *, alpha=1.0, beta=0.0, lower=False, slices=6):
    """``C = beta C + alpha A B^T`` for fp64 row-major 2-D tensors through the int8 tensor-core emulation
    (``gpk_gemm_nt_f64_oz``).  ``A: [M, K]``, ``Bm: [N, K]``; M % 128 == 0, N % 64 == 0, K % 128 == 0."""
    _require_cuda(A, Bm, C)
    M, K = A.shape
    N = Bm.shape[0]
    if C is None:
        C = torch.zeros(M, N, device=A.device, dtype=A.dtype)
    for t in (A, Bm, C):
        if t.dim() != 2 or t.stride(1) != 1 or t.dtype != torch.float64:
            raise ValueError("gemm_nt_oz takes fp64 matrices with a unit inner stride")
    if Bm.shape[1] != K or C.shape != (M, N):
        raise ValueError("gemm_nt_oz: shapes do not match")
    lib = _lib.load()
    need = ((lib.gpk_oz_ws_bytes(M, K, slices) + 1023) // 1024) * 1024 + lib.gpk_oz_ws_bytes(N, K, slices)
    ws = _aligned_bytes(need, A.device)
    rc = lib.gpk_gemm_nt_f64_oz(M, N, K, float(alpha), _ptr(A), A.stride(0), _ptr(Bm), Bm.stride(0), float(beta), _ptr(C),
                                C.stride(0), int(lower), int(slices), _ptr(ws), ws.numel(), _stream())
    check(rc, "gpk_gemm_nt_f64_oz")
    return C


def chol_from_kernel(flat, xg, *, noise_scalar=0.0, noise_vec=None, jitter=0.0, rhs_t=None, full_precision=False):
    """Build ``k(x, x) + noise + jitter I`` straight into the padded lower workspace (K1), factorise it in place
    (K2) and carry ``rhs_t [B, k, n]`` through the factorisation (fused K3).  Returns a :class:`Chol`.
    ``full_precision``: the factor will serve element-wise quantities (posterior means / variances, the ``alpha`` and
    ``K^-1`` of a log-pdf backward): never the 7-slice emulation (see :func:`_oz_slices`)."""
    _check_groups(xg, flat)
    _require_cuda(xg, noise_vec, rhs_t)
    B, n, d = xg.shape[1], xg.shape[2], xg.shape[3]
    k = 0 if rhs_t is None else rhs_t.shape[1]
    W, n_pad, extra = _new_workspace(B, n, k, xg.device, xg.dtype, rhs_t)
    _km_launch(flat, xg, xg, n, n, d, KM_LOWER | KM_SAME | KM_PAD_IDENTITY, noise_scalar, noise_vec, jitter, W,
               W.stride(1), W.stride(0), B)
    return _potrf(W, n, n_pad, extra, k, (not full_precision) and _well_conditioned(flat, noise_scalar, noise_vec, jitter))


def chol_from_dense(K, *, jitter=0.0, rhs_t=None):
    """Factorise a given dense SPD ``K [B, n, n]`` (+ ``jitter I``); only its lower triangle is used."""
    _require_cuda(K, rhs_t)
    if K.stride(2) != 1:
        K = K.contiguous()
    B, n = K.shape[0], K.shape[1]
    k = 0 if rhs_t is None else rhs_t.shape[1]
    W, n_pad, extra = _new_workspace(B, n, k, K.device, K.dtype, rhs_t)
    _pad_copy(K, W, n, n, n_pad, n_pad, jitter, True)
    return _potrf(W, n, n_pad, extra, k)


def kernel_rows_padded(flat, xsg, xg, chol):
    """``k(x*, x)`` as a zero-padded ``[B, m_pad, n_pad]`` buffer (rows = test points) ready for ``solve_rows_``."""
    _check_groups(xg, flat)
    B, m, d = xsg.shape[1], xsg.shape[2], xsg.shape[3]
    n = xg.shape[2]
    if xg.shape[1] != B:  # one problem, a batch of test-point sets: every set reads the same data points
        if xg.shape[1] != 1:
            raise ValueError(f"kernel_rows_padded: data batch {xg.shape[1]} against test-point batch {B}")
        xg = xg.expand(-1, B, -1, -1)
    out = torch.empty(B, round_up(max(m, 1)), chol.n_pad, device=xg.device, dtype=xg.dtype)
    _km_launch(flat, xsg, xg, m, n, d, KM_PAD_ZERO, 0.0, None, 0.0, out, out.stride(1), out.stride(0), B)
    return out


def posterior_marginals(flat, xsg, xg, chol, half_y=None, want_sq=True, chunk=4096):
    """K3 in one call (``gpk_posterior_marginals``): ``(dot [m], sq [m])`` with ``V^T = k(x*, x) L^-T``, ``dot = V^T half_y``,
    ``sq = |v_i|^2``; one problem (no batch), test points streamed in chunks of ``chunk`` rows."""
    _check_groups(xg, flat)
    _require_cuda(xsg, xg, half_y)
    if chol.batch != 1 or xsg.shape[1] != 1 or xg.shape[1] != 1:
        raise ValueError("posterior_marginals handles a single problem")
    xsg, xg = xsg.contiguous(), xg.contiguous()
    m, d = xsg.shape[2], xsg.shape[3]
    dt, dev = chol.dtype, chol.device
    dot = torch.empty(m, dtype=dt, device=dev) if half_y is not None else None
    sq = torch.empty(m, dtype=dt, device=dev) if want_sq else None
    if m == 0:
        return dot, sq
    chunk = min(round_up(chunk), round_up(m))
    ws = torch.empty(chunk * chol.n_pad, dtype=dt, device=dev)
    em = _emulation(dt, dev, lambda lib, s: lib.gpk_trsm_right_oz_ws_bytes(chol.n_pad, chunk, s))
    Lp = chol.L_padded()
    hy = None if half_y is None else half_y.contiguous()
    desc = flat.desc()
    rc = _fn("gpk_posterior_marginals", dt)(
        ctypes.byref(desc), _ptr(xsg), xsg.stride(0), m, _ptr(xg), xg.stride(0), xg.shape[2], d, _ptr(Lp), Lp.stride(1),
        chol.n_pad, _ptr(hy), _ptr(dot), _ptr(sq), chunk, _ptr(ws), ws.numel(), *em, _stream(),
    )
    check(rc, "gpk_posterior_marginals")
    return dot, sq


def sparse_posterior_marginals(flat, xsg, zg, ch_z, ch_s, half_y, want_dot=True, chunk=4096):
    """The marginals of a sparse posterior in one call (``gpk_sparse_posterior_marginals``): ``(dot [n*] or None, sq_z [n*],
    sq_s [n*])`` with ``V^T = k(x*, z) L_z^-T``, ``U^T = k(x*, z) L_S^-T``, ``dot = V^T half_y``, ``sq_z = |v_i|^2``,
    ``sq_s = |u_i|^2``.  ``ch_z``: factor of ``K_z``; ``ch_s``: factor of the stored ``A`` (``L_z A L_z^T``) + eps I.  One
    problem (no batch); test points streamed in chunks of ``chunk`` rows through two ``chunk x m_pad`` buffers."""
    _check_groups(zg, flat)
    _require_cuda(xsg, zg, half_y)
    if ch_z.batch != 1 or ch_s.batch != 1 or xsg.shape[1] != 1 or zg.shape[1] != 1:
        raise ValueError("sparse_posterior_marginals handles a single problem")
    if ch_s.n_pad != ch_z.n_pad or zg.shape[2] != ch_z.n:
        raise ValueError("sparse_posterior_marginals: the factors and the inducing points do not match")
    xsg, zg = xsg.contiguous(), zg.contiguous()
    ns, d = xsg.shape[2], xsg.shape[3]
    dt, dev, m_pad = ch_z.dtype, ch_z.device, ch_z.n_pad
    dot = torch.empty(ns, dtype=dt, device=dev) if want_dot else None
    sq_z = torch.empty(ns, dtype=dt, device=dev)
    sq_s = torch.empty(ns, dtype=dt, device=dev)
    if ns == 0:
        return dot, sq_z, sq_s
    chunk = min(round_up(chunk), round_up(ns))
    lib = _lib.load()
    ws = torch.empty(int(lib.gpk_sparse_posterior_ws_elems(chunk, m_pad)), dtype=dt, device=dev)
    em = _emulation(dt, dev, lambda lib, s: lib.gpk_trsm_right_oz_ws_bytes(m_pad, chunk, s))
    Lz, Ls = ch_z.L_padded(), ch_s.L_padded()
    hy = half_y.contiguous() if want_dot else None
    desc = flat.desc()
    rc = _fn("gpk_sparse_posterior_marginals", dt)(
        ctypes.byref(desc), _ptr(xsg), xsg.stride(0), ns, _ptr(zg), zg.stride(0), ch_z.n, d, _ptr(Lz), Lz.stride(1), _ptr(Ls),
        Ls.stride(1), m_pad, _ptr(hy), _ptr(dot), _ptr(sq_z), _ptr(sq_s), chunk, _ptr(ws), ws.numel(), *em, _stream(),
    )
    check(rc, "gpk_sparse_posterior_marginals")
    return dot, sq_z, sq_s


def sparse_posterior_marginals_bwd(flat, xsg, zg, ch_z, ch_s, half_y, a, b, chunk=4096):
    """Gradient w.r.t. ``xsg`` of :func:`sparse_posterior_marginals` for the upstream gradients ``a [n*]`` of the mean (``dot``)
    and ``b [n*]`` of the variance ``(k - sq_z) + sq_s`` (either may be None).  The factors are constants: with
    ``r_i = k(x*_i, z)``, ``dL/dr_i = L_z^-T (a_i h - 2 b_i v_i) + L_S^-T (2 b_i u_i)``.  Per chunk of test points, as the forward
    walks them: K1 rows into ``V``, copied to ``U``, the right solves against ``L_z`` and ``L_S``, ``gpk_sparse_posterior_rows_bwd``,
    the transposed solves, ``V += U`` and the rectangular K1-backward.  Returns ``grad_xsg`` (like ``xsg``).  Device memory: two
    ``chunk x m_pad`` buffers and the copies the transposed solves make, whatever ``n*`` is."""
    _check_groups(zg, flat)
    _require_cuda(xsg, zg, half_y, a, b)
    if ch_z.batch != 1 or ch_s.batch != 1 or xsg.shape[1] != 1 or zg.shape[1] != 1:
        raise ValueError("sparse_posterior_marginals_bwd handles a single problem")
    if ch_s.n_pad != ch_z.n_pad or zg.shape[2] != ch_z.n:
        raise ValueError("sparse_posterior_marginals_bwd: the factors and the inducing points do not match")
    if a is None and b is None:
        raise ValueError("sparse_posterior_marginals_bwd needs an upstream gradient")
    xsg, zg = xsg.contiguous(), zg.contiguous()
    ns, d = xsg.shape[2], xsg.shape[3]
    dt, dev, m, m_pad = ch_z.dtype, ch_z.device, ch_z.n, ch_z.n_pad
    grad = torch.zeros_like(xsg)
    if ns == 0:
        return grad
    a, b = [None if t is None else t.reshape(-1).contiguous() for t in (a, b)]
    hy = half_y.contiguous() if a is not None else None
    chunk = min(round_up(chunk), round_up(ns))
    Vb = torch.empty(1, chunk, m_pad, dtype=dt, device=dev)
    Ub = torch.empty(1, chunk, m_pad, dtype=dt, device=dev)
    fn = _fn("gpk_sparse_posterior_rows_bwd", dt)
    for c0 in range(0, ns, chunk):
        c1 = min(ns, c0 + chunk)
        c, cp = c1 - c0, round_up(c1 - c0)
        xs_c = xsg[:, :, c0:c1].contiguous()
        V, U = Vb[:, :cp], Ub[:, :cp]
        if b is not None:  # without a variance upstream the rows kernel reads neither buffer
            _km_launch(flat, xs_c, zg, c, m, d, KM_PAD_ZERO, 0.0, None, 0.0, V, V.stride(1), V.stride(0), 1)
            U.copy_(V)
            ch_z.solve_rows_(V)
            ch_s.solve_rows_(U)
        rc = fn(c, m_pad, _ptr(V), _ptr(U), V.stride(1), _ptr(hy), _ptr(None if a is None else a[c0:c1]),
                _ptr(None if b is None else b[c0:c1]), _stream())
        check(rc, "gpk_sparse_posterior_rows_bwd")
        ch_z.solve_many_rows_t_(V)
        if b is not None:  # else U is zero
            ch_s.solve_many_rows_t_(U)
            V += U
        gx = torch.zeros_like(xs_c)
        kernel_cross_bwd(flat, xs_c, zg, W=V, grad_xsg=gx)
        grad[:, :, c0:c1] = gx
    return grad


SPARSE_METHOD = {"vfe": 0, "fitc": 1, "dtc": 2}


class SparseAccumulator:
    """Streamed ``AbstractPseudoObservations._compute`` (``stheno/model/observations.py:279-336``) for ONE problem (no batch
    dimension): the data are walked in chunks of ``chunk`` points through ``gpk_sparse_accumulate``; ``K_zx`` is never held.

    ``A [1, m_pad, m_pad]`` starts at the identity and receives ``W K_n^-1 W^T`` on its lower tiles, ``prod [m_pad]`` receives
    ``W K_n^-1 ybar``, ``scalars`` = (sum log(2 pi K_n), sum ybar^2 / K_n, trace part).  Device memory: two
    ``chunk x m_pad`` buffers + ``A``."""

    def __init__(self, flat, zg, ch_z, method, chunk=16384):
        _require_cuda(zg, ch_z.W)
        if ch_z.batch != 1 or zg.shape[1] != 1:
            raise ValueError("SparseAccumulator handles a single problem (batched sparse problems use the materialised path)")
        self.flat, self.zg, self.ch, self.method = flat, zg.contiguous(), ch_z, SPARSE_METHOD[method]
        self.m, self.m_pad, self.d = ch_z.n, ch_z.n_pad, zg.shape[3]
        self.chunk = int(chunk)
        dt, dev = ch_z.dtype, ch_z.device
        self.A = torch.zeros(1, self.m_pad, self.m_pad, dtype=dt, device=dev)
        self.A.diagonal(dim1=1, dim2=2).fill_(1.0)
        self.prod = torch.zeros(self.m_pad, dtype=dt, device=dev)
        self.scalars = torch.zeros(3, dtype=dt, device=dev)
        self.lib = _lib.load()
        self.ws = None

    def _workspace(self, c):
        need = int(self.lib.gpk_sparse_ws_elems(c, self.m_pad))
        if self.ws is None or self.ws.numel() < need:
            self.ws = torch.empty(need, dtype=self.ch.dtype, device=self.ch.device)
        return self.ws

    def add(self, xg_chunk, kdiag, kn, ybar):
        """One chunk: ``xg_chunk [G, 1, c, d]`` pre-stretched points, ``kdiag / kn / ybar [c]`` (``kdiag`` None for DTC)."""
        _require_cuda(xg_chunk, kdiag, kn, ybar)
        xg_chunk = xg_chunk.contiguous()
        c = xg_chunk.shape[2]
        if c == 0:
            return
        ws = self._workspace(c)
        m_pad, c_pad = self.m_pad, round_up(c)
        # the emulation scratch holds the larger of the solve's products and the K = c accumulation
        em = _emulation(self.ch.dtype, self.ch.device, lambda lib, s: max(lib.gpk_trsm_right_oz_ws_bytes(m_pad, c_pad, s),
                                                                          lib.gpk_gemm_nt_oz_ws_bytes(m_pad, m_pad, c_pad, s)))
        kd = None if kdiag is None else kdiag.contiguous()
        kn, ybar = kn.contiguous(), ybar.contiguous()
        Lp = self.ch.L_padded()
        desc = self.flat.desc()
        rc = _fn("gpk_sparse_accumulate", self.ch.dtype)(
            ctypes.byref(desc), _ptr(xg_chunk), xg_chunk.stride(0), c, _ptr(self.zg), self.zg.stride(0), self.m, self.d,
            _ptr(Lp), Lp.stride(1), self.m_pad, _ptr(kd), _ptr(kn), _ptr(ybar), self.method, _ptr(self.A), self.A.stride(1),
            _ptr(self.prod), _ptr(self.scalars), _ptr(ws), ws.numel(), *em, _stream(),
        )
        check(rc, "gpk_sparse_accumulate")


class CrossBlock:
    """One nonzero block ``k(f_p, u_q)`` of a sparse problem, for :func:`sparse_elbo_bwd`: its flat kernel, the
    pre-stretched points ``xg [G, 1, n_p, d]`` of ``f_p`` and ``zg [G, 1, m_q, d]`` of ``u_q``, the first column ``col`` of
    ``u_q`` in ``K_z``, and the optional outputs ``term_sum``, ``grad_xg`` (like ``xg``), ``grad_zg`` (like ``zg``) and
    ``param_sum`` the rectangular K1-backward accumulates into (None: not formed)."""

    def __init__(self, flat, xg, zg, col, term_sum=None, grad_xg=None, grad_zg=None, param_sum=None):
        self.flat, self.xg, self.zg, self.col = flat, xg, zg.contiguous(), int(col)
        self.term_sum, self.grad_xg, self.grad_zg, self.param_sum = term_sum, grad_xg, grad_zg, param_sum


def sparse_elbo_bwd(procs, ch_z, ch_A, s, kdiag, kn, ybar, method, chunk, want_H=True, want_cross=True):
    """Backward of the sparse ELBO over chunks of data points.  ``procs``: one entry per observed process ``f_p``, in data
    order, ``(n_p, [CrossBlock, ...])`` (the nonzero blocks ``k(f_p, u_q)``; one process with one block for a problem over
    one inducing and one observed process); ``ch_z``: factor of ``K_z``; ``ch_A``: factor of ``A = I + W K_n^-1 W^T``;
    ``s = A^-1 prod [m]``; ``kdiag`` (None for DTC), ``kn`` and ``ybar``: ``[n]`` over all processes.

    The data are walked in chunks of at most ``chunk`` points that never straddle two processes.  A chunk's rows
    ``k(x_c, z)`` are one ``c_pad x m_pad`` buffer: one K1 launch per block writes exactly ``c x m_q`` entries at the block's
    column offset (no padding flag: a padded launch would write past ``m_q`` into the next block), and the columns of zero
    blocks and the ragged rows are zeroed.  The solve against ``L_z`` gives ``W_c`` (the forward's launches),
    ``U_c = W_c A^-1``, and ``gpk_sparse_rows_bwd`` turns ``U_c`` into ``G_c`` (rows ``dE/dw_i``) and writes the per-point
    gradients.  With ``want_H``, ``H += G_c^T W_c`` on the lower tiles (mirrored after the last chunk;
    ``dE/dK_z = -1/2 L^-T H L^-1``).  With ``want_cross``, the transposed solve turns ``G_c`` into rows ``dE/dk(x_i, z)`` and
    the rectangular K1-backward runs once per block on its column slice, accumulating into the block's outputs.  Returns
    ``(g_kn [n], g_kd [n] or None, g_ybar [n], H [1, m_pad, m_pad] or None)``.  Device memory: four ``chunk x m_pad`` buffers
    and three ``m_pad x m_pad`` ones."""
    _require_cuda(kdiag, kn, ybar)
    meth = SPARSE_METHOD[method]
    m, m_pad, dt, dev = ch_z.n, ch_z.n_pad, ch_z.dtype, ch_z.device
    n = sum(n_p for n_p, _ in procs)
    V = torch.zeros(1, m_pad, m_pad, dtype=dt, device=dev)
    V.diagonal(dim1=1, dim2=2).fill_(1.0)
    ch_A.solve_rows_(V)  # V = L_A^-T, A^-1 = V V^T (the identity on the padding)
    Ainv = gemm_nt(V, V)
    del V
    sp = torch.zeros(m_pad, dtype=dt, device=dev)
    sp[:m] = s
    g_kn = torch.empty(n, dtype=dt, device=dev)
    g_ybar = torch.empty(n, dtype=dt, device=dev)
    g_kd = torch.empty(n, dtype=dt, device=dev) if meth != 2 else None
    kdiag, kn, ybar = [None if t is None else t.contiguous() for t in (kdiag, kn, ybar)]
    H = torch.zeros(1, m_pad, m_pad, dtype=dt, device=dev) if want_H else None
    rows = round_up(min(int(chunk), max([n_p for n_p, _ in procs] + [1])))
    Wb = torch.zeros(1, rows, m_pad, dtype=dt, device=dev)  # the padding columns stay zero through the solve
    Ub = torch.empty(1, rows, m_pad, dtype=dt, device=dev)
    if want_H:
        WTb = torch.empty(1, m_pad, rows, dtype=dt, device=dev)
        GTb = torch.empty(1, m_pad, rows, dtype=dt, device=dev)
    fn = _fn("gpk_sparse_rows_bwd", dt)
    a0 = 0
    for n_p, blocks in procs:
        gaps, pos = [], 0  # column ranges of zero blocks: the solve of the previous chunk left numbers there
        for j0, j1 in sorted((blk.col, blk.col + blk.zg.shape[2]) for blk in blocks) + [(m, m)]:
            if j0 > pos:
                gaps.append((pos, j0))
            pos = max(pos, j1)
        for a in range(0, n_p, int(chunk)):
            b = min(n_p, a + int(chunk))
            c, cp = b - a, round_up(b - a)
            ga, gb = a0 + a, a0 + b
            Wc, Uc = Wb[:, :cp], Ub[:, :cp]
            Wc[:, c:].zero_()
            for j0, j1 in gaps:
                Wc[:, :c, j0:j1].zero_()
            for blk in blocks:
                xc = blk.xg[:, :, a:b].contiguous()
                Wq = Wc[:, :, blk.col :]
                _km_launch(blk.flat, xc, blk.zg, c, blk.zg.shape[2], blk.zg.shape[3], 0, 0.0, None, 0.0, Wq, Wq.stride(1),
                           Wq.stride(0), 1)
            ch_z.solve_rows_(Wc)
            q = row_dot_sq(Wc, c, m_pad, None)[1] if meth != 2 else None
            gemm_nt(Wc, Ainv, Uc)
            rc = fn(c, m_pad, _ptr(Wc), Wc.stride(1), _ptr(Uc), Uc.stride(1), _ptr(sp), _ptr(q),
                    _ptr(None if kdiag is None else kdiag[ga:gb]), _ptr(kn[ga:gb]), _ptr(ybar[ga:gb]), meth, _ptr(g_kn[ga:gb]),
                    _ptr(None if g_kd is None else g_kd[ga:gb]), _ptr(g_ybar[ga:gb]), _stream())
            check(rc, "gpk_sparse_rows_bwd")
            if want_H:
                WT, GT = WTb[:, :, :cp], GTb[:, :, :cp]
                transpose(Wc, cp, m_pad, out=WT)
                transpose(Uc, cp, m_pad, out=GT)
                gemm_nt(GT, WT, H, beta=1.0, lower=True)
            if want_cross and blocks:
                ch_z.solve_many_rows_t_(Uc)
                for blk in blocks:
                    xc = blk.xg[:, :, a:b].contiguous()
                    mq = blk.zg.shape[2]
                    gx = torch.zeros_like(xc) if blk.grad_xg is not None else None
                    kernel_cross_bwd(blk.flat, xc, blk.zg, W=Uc[:, :, blk.col : blk.col + mq], term_sum=blk.term_sum,
                                     grad_xsg=gx, grad_xg=blk.grad_zg, param_sum=blk.param_sum)
                    if gx is not None:
                        blk.grad_xg[:, :, a:b] += gx
        a0 += n_p
    if want_H:
        symmetrize_(H, m_pad)
    return g_kn, g_kd, g_ybar, H


def gemm_profile(enable):
    """Switch the in-situ event timing of the fp64 GEMM kernel on / off (clears the record)."""
    _lib.load().gpk_gemm_profile_enable(1 if enable else 0)


def gemm_profile_read(kind=0):
    """``(total_ms, algorithmic_flops, launches)`` of the profiled GEMM launches since ``gemm_profile(True)``; synchronises.
    ``kind``: 0 = fp64 DMMA trailing-update kernel, 1 = int8-slice emulation kernel (fp64-equivalent flops), -1 = both."""
    torch.cuda.synchronize()
    ms, fl, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
    check(_lib.load().gpk_gemm_profile_read_kind(int(kind), ctypes.byref(ms), ctypes.byref(fl), ctypes.byref(n)),
          "gpk_gemm_profile_read_kind")
    return ms.value, fl.value, n.value


def probe_dmma_tflops():
    return float(_lib.load().gpk_probe_dmma_tflops())


LOG_2_PI = math.log(2 * math.pi)
