"""Differentiable log-marginal likelihood: ``torch.autograd.Function`` around the fused K1 -> K2 -> K4 path with an
ANALYTIC backward (SURVEY.md section 7 step 8, section 8 row a16):

    d logpdf / dK = 1/2 (alpha alpha^T - K^-1),   alpha = K^-1 (y - mu)

``K^-1 = L^-T L^-1`` comes from one tensor-core TRSM on the identity and one SYRK; the contraction with ``dK/dtheta``
(kernel scales, length scales through the pre-stretched inputs, inputs, noise, RQ's alpha) happens inside the K1-backward kernel
(``csrc/kernel_matrix_bwd.cu``) so no ``n x n`` gradient tensor per hyper-parameter is ever formed.  The reference gets
these gradients from torch autograd through ``exp`` / ``cholesky`` / ``triangular_solve``
(``readme_example13_optimisation_torch.py:46-53``).

Cross-covariances ``k(x, y)``, ``k.elwise(x)`` and exact posterior predictions get analytic backwards the same way: the
rectangular K1-backward (``gpk_kernel_cross_bwd``) contracts ``d loss / d k(x*, x)`` in factored form."""
import ctypes

import torch

from . import _lib, ops

__all__ = ["kernel_logpdf", "dense_logpdf", "kernel_matrix_grad", "kernel_cross_grad", "kernel_diag_grad", "exact_posterior",
           "sparse_posterior_marginals", "subspace_cov", "no_gradient"]


def _bwd_kernel(flat, xg, G, n, param_sum=None):
    """``(term_sum [B, T], grad_xg like xg, diag [B, n])`` from the K1-backward kernel; with ``param_sum``
    (``[B, GPK_MAX_FACTORS]``, zeroed by the caller) the same launch also adds the gradient of every factor's shape
    parameter into it."""
    Bn, d = xg.shape[1], xg.shape[3]
    term_sum = torch.zeros(Bn, _lib.GPK_MAX_TERMS, dtype=xg.dtype, device=xg.device)
    grad_xg = torch.zeros_like(xg)
    diag = torch.zeros(Bn, n, dtype=xg.dtype, device=xg.device)
    desc = flat.desc()
    rc = ops._fn("gpk_kernel_matrix_bwd", xg.dtype)(
        ctypes.byref(desc), ops._ptr(xg), xg.stride(0), xg.stride(1), n, d, ops._ptr(G), G.stride(1), G.stride(0),
        ops._ptr(term_sum), ops._ptr(grad_xg), ops._ptr(diag), ops._ptr(param_sum), Bn, ops._stream(),
    )
    _lib.check(rc, "gpk_kernel_matrix_bwd")
    return term_sum, grad_xg, diag


def _param_buf(want, B, like):
    """A zeroed ``[B, GPK_MAX_FACTORS]`` parameter-gradient output when ``want``, else None."""
    return torch.zeros(B, _lib.GPK_MAX_FACTORS, dtype=like.dtype, device=like.device) if want else None


def _param_grad(flat, param_sum):
    """The ``[F]`` gradient of :func:`param_tensor` from a ``[B, GPK_MAX_FACTORS]`` parameter sum (None stays None)."""
    return None if param_sum is None else param_sum[:, : _n_factors(flat)].sum(0)


def _n_factors(flat):
    return sum(len(fs) for _, fs in flat.terms)


class _KernelLogpdf(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flat, coefs, xg, noise_scalar, noise_vec, rhs_t, jitter, params):
        # flat: the caller's descriptor, which the launches read (as in the three functions below); coefs [T] and params [F]
        # (coef_tensor, param_tensor) only route the gradients of its hyper-parameters to those given as tensors
        # xg [G, B, n, d], noise_scalar [] , noise_vec [B, n] or None, rhs_t [B, k, n]
        # the backward reads alpha and K^-1 element by element off this factor: never the 7-slice factorisation
        ch = ops.chol_from_kernel(flat, xg.detach().contiguous(), noise_scalar=float(noise_scalar),
                                  noise_vec=None if noise_vec is None else noise_vec.detach(), jitter=jitter,
                                  rhs_t=rhs_t.detach(), full_precision=True)
        ctx.ch, ctx.flat = ch, flat
        ctx.xg = xg.detach().contiguous()
        ctx.has_nv = noise_vec is not None
        return ch.logpdf()

    @staticmethod
    def backward(ctx, g):
        ch, flat, xg = ctx.ch, ctx.flat, ctx.xg
        alpha, Gm = _alpha_and_G(ch, g)
        ps = _param_buf(ctx.needs_input_grad[7], xg.shape[1], xg)
        term_sum, grad_xg, diag = _bwd_kernel(flat, xg, Gm, ch.n, ps)
        T = len(flat.terms)
        grad_coefs = term_sum[:, :T].sum(0)
        grad_noise_scalar = diag.sum()
        grad_noise_vec = diag if ctx.has_nv else None
        grad_rhs = -g.unsqueeze(-1) * alpha
        return None, grad_coefs, grad_xg, grad_noise_scalar, grad_noise_vec, grad_rhs, None, _param_grad(flat, ps)


def _alpha_and_G(ch, g):
    """``alpha = K^-1 ybar`` (rows) and ``G = d(sum_c g_c logpdf_c)/dK = 1/2 (sum_c g_c alpha_c alpha_c^T - (sum g) K^-1)``
    as a full symmetric padded ``[B, n_pad, n_pad]`` tensor, from the factor ``ch`` with fused right-hand sides."""
    # 7-slice solve and products: against torch fp64 autograd they lose no more than native fp64 does, from noise 1e-2 to
    # 1e-6 of the variance, as long as the factor ch has 8 slices (tests/test_logpdf_grad_paths.py)
    with ops.product_slices(7):
        return _alpha_and_G_impl(ch, g)


def _alpha_and_G_impl(ch, g):
    Bn, n, n_pad, k = ch.batch, ch.n, ch.n_pad, ch.k
    dtype, dev = ch.dtype, ch.device
    arows = ch.new_rows(k)
    arows[:, :k, :n] = ch.rhs_half()
    ch.solve_rows_t_(arows)
    alpha = arows[:, :k, :n]
    V = torch.zeros(Bn, n_pad, n_pad, dtype=dtype, device=dev)
    V.diagonal(dim1=1, dim2=2).fill_(1.0)
    ch.solve_rows_(V)  # rows (L^-1 e_r)^T, i.e. V = L^-T ; K^-1 = V V^T
    Gm = torch.empty(Bn, n_pad, n_pad, dtype=dtype, device=dev)
    kp = ops.round_up(k, 16)
    for b in range(Bn):
        # the weight sum(g_c) scales the product on the device: reading it on the host would make the backward wait for
        # everything enqueued before it on the stream
        ops.gemm_nt(V[b : b + 1], V[b : b + 1], Gm[b : b + 1], alpha=-0.5, beta=0.0, lower=True)
        Gm[b].mul_(g[b].sum())
        A = torch.zeros(1, n_pad, kp, dtype=dtype, device=dev)
        Bm = torch.zeros(1, n_pad, kp, dtype=dtype, device=dev)
        A[0, :n, :k] = (alpha[b] * (0.5 * g[b]).unsqueeze(-1)).t()
        Bm[0, :n, :k] = alpha[b].t()
        ops.gemm_nt(A, Bm, Gm[b : b + 1], alpha=1.0, beta=1.0, lower=True)
    del V
    ops.symmetrize_(Gm, n_pad)
    return alpha, Gm


class _DenseLogpdf(torch.autograd.Function):
    """``logpdf`` of ``N(0, K + jitter I)`` for an explicit dense ``K [B, n, n]`` with a gradient w.r.t. ``K`` itself --
    the route for covariances assembled from several kernel matrices (multi-output joints, ``stheno/mo``)."""

    @staticmethod
    def forward(ctx, K, rhs_t, jitter):
        ch = ops.chol_from_dense(K.detach(), jitter=jitter, rhs_t=rhs_t.detach())
        ctx.ch = ch
        return ch.logpdf()

    @staticmethod
    def backward(ctx, g):
        ch = ctx.ch
        alpha, Gm = _alpha_and_G(ch, g)
        n = ch.n
        return Gm[:, :n, :n].contiguous(), -g.unsqueeze(-1) * alpha, None


def dense_logpdf(K, rhs_t, jitter):
    return _DenseLogpdf.apply(K, rhs_t, jitter)


class _KernelMatrix(torch.autograd.Function):
    """Differentiable ``k(x, x)`` (same points) built by K1; backward = K1-backward on the symmetrised upstream gradient."""

    @staticmethod
    def forward(ctx, flat, coefs, xg, params):
        ctx.flat, ctx.xg = flat, xg.detach().contiguous()
        return ops.kernel_matrix(flat, ctx.xg)

    @staticmethod
    def backward(ctx, G):
        flat, xg = ctx.flat, ctx.xg
        n = xg.shape[2]
        Gs = (0.5 * (G + G.transpose(1, 2))).contiguous()  # K is symmetric: only the symmetric part of G matters
        ps = _param_buf(ctx.needs_input_grad[3], xg.shape[1], xg)
        term_sum, grad_xg, _ = _bwd_kernel(flat, xg, Gs, n, ps)
        return None, term_sum[:, : len(flat.terms)].sum(0), grad_xg, _param_grad(flat, ps)


def _scalar(v, like):
    """``v`` as a 0-d tensor of ``like``'s dtype and device, with its graph when it is a tensor."""
    if isinstance(v, torch.Tensor):
        return v.to(device=like.device, dtype=like.dtype).reshape(())
    return torch.tensor(float(v), device=like.device, dtype=like.dtype)


def coef_tensor(flat, like):
    """The coefficients of ``flat`` as one ``[T]`` tensor on ``like``'s device, with the graph of those given as tensors."""
    raw = getattr(flat, "coef_raw", None) or [c for c, _ in flat.terms]
    return torch.stack([_scalar(c, like) for c in raw])


def param_tensor(flat, like):
    """The shape parameters of ``flat``'s factors, in descriptor order (RQ's alpha; 0 for kinds without one), as one ``[F]``
    tensor on ``like``'s device, with the graph of those given as tensors."""
    vals = [fac[2] if len(fac) > 2 else 0.0 for _, fs in flat.terms for fac in fs]
    raw = getattr(flat, "param_raw", None) or vals
    if not vals:
        return torch.zeros(0, dtype=like.dtype, device=like.device)
    return torch.stack([_scalar(v if r is None else r, like) for r, v in zip(raw, vals)])


def kernel_matrix_grad(flat, xg):
    """``k(x, x) [B, n, n]`` with an autograd graph to the kernel's tensor hyper-parameters and to ``xg``."""
    return _KernelMatrix.apply(flat, coef_tensor(flat, xg), xg, param_tensor(flat, xg))


def kernel_logpdf(flat, xg, noise_scalar, noise_vec, rhs_t, jitter):
    """Differentiable ``logpdf`` ``[B, k]`` of ``N(0, k(x, x) + noise + jitter I)`` at ``rhs_t`` for the flat kernel ``flat``
    on ``xg``, with an autograd graph to the kernel's tensor hyper-parameters, ``xg``, the noise (``noise_scalar``: a float
    or a tensor; ``noise_vec [B, n]`` or None) and ``rhs_t``."""
    return _KernelLogpdf.apply(flat, coef_tensor(flat, xg), xg, _scalar(noise_scalar, xg), noise_vec, rhs_t, jitter,
                               param_tensor(flat, xg))


class _KernelCross(torch.autograd.Function):
    """Differentiable ``k(x, y)`` for two different point sets, built by K1; backward = the rectangular K1-backward."""

    @staticmethod
    def forward(ctx, flat, coefs, xsg, xg, params):
        ctx.flat, ctx.xsg, ctx.xg = flat, xsg.detach().contiguous(), xg.detach().contiguous()
        return ops.kernel_matrix(flat, ctx.xsg, ctx.xg, same=False)

    @staticmethod
    def backward(ctx, G):
        flat, xsg, xg = ctx.flat, ctx.xsg, ctx.xg
        nig = ctx.needs_input_grad
        ts = torch.zeros(xsg.shape[1], _lib.GPK_MAX_TERMS, dtype=xsg.dtype, device=xsg.device) if nig[1] else None
        gxs = torch.zeros_like(xsg) if nig[2] else None
        gx = torch.zeros_like(xg) if nig[3] else None
        ps = _param_buf(nig[4], xsg.shape[1], xsg)
        ops.kernel_cross_bwd(flat, xsg, xg, W=G.contiguous(), term_sum=ts, grad_xsg=gxs, grad_xg=gx, param_sum=ps)
        return None, None if ts is None else ts[:, : len(flat.terms)].sum(0), gxs, gx, _param_grad(flat, ps)


def kernel_cross_grad(flat, xsg, xg):
    """``k(x, y) [B, m, n]`` (``x is not y``) with an autograd graph to the kernel's tensor hyper-parameters, ``xsg`` and
    ``xg``."""
    return _KernelCross.apply(flat, coef_tensor(flat, xsg), xsg, xg, param_tensor(flat, xsg))


class _KernelDiag(torch.autograd.Function):
    """Differentiable ``k.elwise(x)`` (same points); the backward is the prior-variance term of the rectangular K1-backward."""

    @staticmethod
    def forward(ctx, flat, coefs, xg, params):
        ctx.flat, ctx.xg = flat, xg.detach().contiguous()
        return ops.kernel_diag(flat, ctx.xg)

    @staticmethod
    def backward(ctx, g):
        flat, xg = ctx.flat, ctx.xg
        nig = ctx.needs_input_grad
        ts = torch.zeros(xg.shape[1], _lib.GPK_MAX_TERMS, dtype=xg.dtype, device=xg.device) if nig[1] else None
        gx = torch.zeros_like(xg) if nig[2] else None
        ps = _param_buf(nig[3], xg.shape[1], xg)
        ops.kernel_cross_bwd(flat, xg, xg, gdiag=g.contiguous(), term_sum=ts, grad_xsg=gx, param_sum=ps)
        return None, None if ts is None else ts[:, : len(flat.terms)].sum(0), gx, _param_grad(flat, ps)


def kernel_diag_grad(flat, xg):
    """``k.elwise(x) [B, n]`` with an autograd graph to the kernel's tensor hyper-parameters and to ``xg``."""
    return _KernelDiag.apply(flat, coef_tensor(flat, xg), xg, param_tensor(flat, xg))


class _NoGradient(torch.autograd.Function):
    @staticmethod
    def forward(ctx, route, value, *inputs):
        ctx.route = route
        return value.detach().clone()

    @staticmethod
    def backward(ctx, *grads):
        raise NotImplementedError(f"gradients through {ctx.route} are not implemented")


def no_gradient(route, value, inputs):
    """``value`` unchanged, attached to ``inputs`` (the tensors that require grad and feed it) by a node whose backward raises
    ``NotImplementedError`` naming ``route``: reading the value works, a ``backward()`` that would return wrong gradients
    through a raw-pointer kernel does not."""
    return _NoGradient.apply(route, value, *inputs)


# ---- the sparse ELBO (PseudoObs VFE / FITC / DTC) -----------------------------------------------------------------------
#
# L = chol(K_z + eps I), W = L^-1 K_zx (columns w_i), kappa_i = K_n' (:311-313), A = I + W diag(1/kappa) W^T, s = A^-1 prod.
# gpk_sparse_rows_bwd gives the per-point gradients and g_i = dE/dw_i; E depends on W only through W^T W, so H = sum_i g_i w_i^T
# is symmetric and   dE/dK_zx[:, i] = L^-T g_i,   dE/dK_z = -1/2 L^-T H L^-1.
# K_z = [k(u_q, u_q')], K_zx = [k(u_q, f_p)] and diag K_x = [diag k(f_p)] are assembled from blocks, one per pair of
# processes (one of each over one inducing and one observed process): only forming the rows and contracting the gradients
# go block by block.  The forward factors K_z with the lower blocks only, so a block below the diagonal receives
# dE/dK_z[q, q'] + dE/dK_z[q', q]^T = 2 GK[q, q'] (GK = dE/dK_z is symmetric).
class SparseElboSpec:
    """What one sparse ELBO needs beyond its tensor inputs: the method, ``z_sizes`` (``m_q``) and ``x_sizes`` (``n_p``);
    the nonzero blocks as flat kernels: ``kz`` ``[(q, q', flat)]`` with ``q' <= q``, ``cross`` ``[(p, q, flat)]``
    (``k(f_p, u_q)``) and ``kx`` ``[(p, flat)]`` (``k(f_p)``, empty for DTC); the chunk; and ``fwd()``, which runs the
    launches of the no-grad path and returns ``(ch_z, ch_A, s, kdiag, elbo)`` (``kdiag``: the ``diag K_x`` that path
    streamed, else None: the backward then forms it from the ``kx`` blocks)."""

    def __init__(self, method, z_sizes, x_sizes, kz, cross, kx, chunk, fwd):
        self.method, self.z_sizes, self.x_sizes, self.chunk, self.fwd = method, list(z_sizes), list(x_sizes), chunk, fwd
        self.kz, self.cross, self.kx = kz, cross, kx
        self.z_off = [sum(self.z_sizes[:q]) for q in range(len(self.z_sizes))]
        self.x_off = [sum(self.x_sizes[:p]) for p in range(len(self.x_sizes))]


class _SparseElbo(torch.autograd.Function):
    """Inputs after ``spec``: per ``kz`` block ``(coefs, zg_q, zg_q' or None on the diagonal, params)``, the inducing noise
    ``nz [m]`` or None, per ``cross`` block ``(coefs, xg_p, zg_q, params)``, per ``kx`` block ``(coefs, xg_p, params)``, then
    ``kn [n]`` and ``ybar [n]``."""

    @staticmethod
    def forward(ctx, spec, *ts):
        ch_z, ch_A, s, kdiag, elbo = spec.fwd()
        ctx.spec, ctx.ch_z, ctx.ch_A, ctx.s, ctx.kdiag = spec, ch_z, ch_A, s, kdiag
        ctx.ts = [None if t is None else t.detach() for t in ts]
        return elbo

    @staticmethod
    def backward(ctx, g):
        spec, ch_z, ts = ctx.spec, ctx.ch_z, ctx.ts
        nig = ctx.needs_input_grad[1:]
        dt, dev, m_pad = ch_z.dtype, ch_z.device, ch_z.n_pad
        nkz, ncr = len(spec.kz), len(spec.cross)
        i_nz, i_cr = 4 * nkz, 4 * nkz + 1
        i_kx = i_cr + 4 * ncr
        i_kn = i_kx + 3 * len(spec.kx)
        grads = [None] * len(ts)
        want_K = any(nig[:i_cr])
        want_cross = any(nig[i_cr:i_kx])

        def term_buf(i):
            return torch.zeros(1, _lib.GPK_MAX_TERMS, dtype=dt, device=dev) if nig[i] else None

        # kdiag = diag K_x over all processes (VFE / FITC): what the forward's rows read
        kdiag = ctx.kdiag
        if kdiag is None and spec.method != "dtc":
            kdiag = torch.zeros(sum(spec.x_sizes), dtype=dt, device=dev)
            for b, (p, flat) in enumerate(spec.kx):
                a = spec.x_off[p]
                kdiag[a : a + spec.x_sizes[p]] = ops.kernel_diag(flat, ts[i_kx + 3 * b + 1])[0]

        procs = [(n_p, []) for n_p in spec.x_sizes]
        outs = []
        for b, (p, q, flat) in enumerate(spec.cross):
            k = i_cr + 4 * b
            xg, zg = ts[k + 1], ts[k + 2]
            blk = ops.CrossBlock(flat, xg, zg, spec.z_off[q], term_sum=term_buf(k),
                                 grad_xg=torch.zeros_like(xg) if nig[k + 1] else None,
                                 grad_zg=torch.zeros_like(zg) if nig[k + 2] else None,
                                 param_sum=_param_buf(nig[k + 3], 1, xg))
            procs[p][1].append(blk)
            outs.append((k, flat, blk))
        g_kn, g_kd, g_y, H = ops.sparse_elbo_bwd(procs, ch_z, ctx.ch_A, ctx.s, kdiag, ts[i_kn], ts[i_kn + 1], spec.method,
                                                 spec.chunk, want_H=want_K, want_cross=want_cross)
        grads[i_kn], grads[i_kn + 1] = g_kn, g_y
        for k, flat, blk in outs:
            grads[k] = None if blk.term_sum is None else blk.term_sum[0, : len(flat.terms)]
            grads[k + 1], grads[k + 2], grads[k + 3] = blk.grad_xg, blk.grad_zg, _param_grad(flat, blk.param_sum)

        if want_K:
            # dE/dK_z = -1/2 L^-T H L^-1: two transposed solves with a transpose between them
            ch_z.solve_many_rows_t_(H)
            GK = ops.transpose(H, m_pad, m_pad)
            del H
            ch_z.solve_many_rows_t_(GK)
            GK.mul_(-0.5)
            ops.symmetrize_(GK, m_pad)
            for b, (q, q2, flat) in enumerate(spec.kz):
                k = 4 * b
                if not any(nig[k : k + 4]):
                    continue
                o, o2, mq, mq2 = spec.z_off[q], spec.z_off[q2], spec.z_sizes[q], spec.z_sizes[q2]
                zg, zg2 = ts[k + 1], ts[k + 2]
                ps = _param_buf(nig[k + 3], 1, zg)
                if q == q2:
                    term_sum, g_z, _ = _bwd_kernel(flat, zg, GK[:, o : o + mq, o : o + mq], mq, ps)
                    grads[k + 1] = g_z if nig[k + 1] else None
                    scale = 1.0
                else:
                    term_sum = torch.zeros(1, _lib.GPK_MAX_TERMS, dtype=dt, device=dev)
                    g_z = torch.zeros_like(zg) if nig[k + 1] else None
                    g_z2 = torch.zeros_like(zg2) if nig[k + 2] else None
                    ops.kernel_cross_bwd(flat, zg, zg2, W=GK[:, o : o + mq, o2 : o2 + mq2], term_sum=term_sum, grad_xsg=g_z,
                                         grad_xg=g_z2, param_sum=ps)
                    grads[k + 1], grads[k + 2] = (None if t is None else 2.0 * t for t in (g_z, g_z2))
                    scale = 2.0
                grads[k] = scale * term_sum[0, : len(flat.terms)] if nig[k] else None
                pg = _param_grad(flat, ps)
                grads[k + 3] = None if pg is None else scale * pg
            if nig[i_nz]:
                grads[i_nz] = GK.diagonal(dim1=1, dim2=2)[0, : ch_z.n].clone()
            del GK

        for b, (p, flat) in enumerate(spec.kx):
            k = i_kx + 3 * b
            if not any(nig[k : k + 3]):
                continue
            xg = ts[k + 1]
            ts_x = term_buf(k)
            g_x = torch.zeros_like(xg) if nig[k + 1] else None
            ps_x = _param_buf(nig[k + 2], 1, xg)
            a = spec.x_off[p]
            ops.kernel_cross_bwd(flat, xg, xg, gdiag=g_kd[a : a + spec.x_sizes[p]].unsqueeze(0), term_sum=ts_x, grad_xsg=g_x,
                                 param_sum=ps_x)
            grads[k] = None if ts_x is None else ts_x[0, : len(flat.terms)]
            grads[k + 1], grads[k + 2] = g_x, _param_grad(flat, ps_x)
        return (None,) + tuple(None if (gr is None or not w) else g * gr for gr, w in zip(grads, nig))


def sparse_elbo(spec, kz, nz, cross, kx, kn, ybar):
    """The ELBO ``spec.fwd()`` computes, differentiable w.r.t. every block's coefficients, pre-stretched inputs and shape
    parameters (``kz``, ``cross``, ``kx``: one tuple of tensors per block of ``spec``, in :class:`_SparseElbo`'s order), the
    inducing noise ``nz [m]`` (None: none), the observation noise ``kn [n]`` and ``ybar [n]``."""
    flat_ts = [t for blk in kz for t in blk] + [nz] + [t for blk in cross for t in blk] + [t for blk in kx for t in blk]
    return _SparseElbo.apply(spec, *flat_ts, kn, ybar)


# ---- sparse posterior predictions in the test inputs ------------------------------------------------------------------------
#
# PseudoObs* posteriors: r_i = k(x*_i, z), v_i = L_z^-1 r_i, u_i = L_S^-1 r_i (L_S: the factor of the stored A + eps I),
# mean_i = m(x*_i) + <v_i, h>, var_i = k(x*_i, x*_i) - |v_i|^2 + |u_i|^2, C = P - V V^T + U U^T.  With K_z, A and mu constant
# (nothing that feeds the approximation requires grad) the gradient in x* needs only the factors the forward holds:
#   dL/dr_i = L_z^-T (a_i h - 2 b_i v_i) + L_S^-T (2 b_i u_i)          (marginals; a, b: upstream of mean, var)
#   dL/dR   = (2 Hs U) L_S^-1 for the U U^T term of C, Hs = (gC + gC^T) / 2 (the P - V V^T term is exact_posterior's)
# The derivative of what the forward computes, eps included; the prior terms m(x*), k(x*, x*) and P keep their own graphs.
class SparsePosteriorSpec:
    """What the sparse marginals need beyond the test points: the cross kernel ``flat`` and the pre-stretched inducing points
    ``zg``, the factors ``ch_z`` of ``K_z`` and ``ch_s`` of the stored ``A`` (+ eps I), ``half_y = L_z^-1 (mu - m_z(z))``
    (``[m_pad]``; None: variances only) and the chunk of test points."""

    def __init__(self, flat, zg, ch_z, ch_s, half_y, chunk=4096):
        self.flat, self.zg, self.ch_z, self.ch_s, self.half_y, self.chunk = flat, zg, ch_z, ch_s, half_y, chunk


class _SparsePosteriorMarginals(torch.autograd.Function):
    @staticmethod
    def forward(ctx, spec, xsg, prior_m, prior_v):
        ctx.set_materialize_grads(False)
        ctx.spec, ctx.xsg = spec, xsg.detach()
        ctx.shapes = (None if prior_m is None else prior_m.shape, prior_v.shape)
        dot, sq_z, sq_s = ops.sparse_posterior_marginals(spec.flat, ctx.xsg, spec.zg, spec.ch_z, spec.ch_s, spec.half_y,
                                                         want_dot=spec.half_y is not None, chunk=spec.chunk)
        n = xsg.shape[2]
        var = (prior_v - sq_z.reshape(n, 1)) + sq_s.reshape(n, 1)
        if prior_m is None:
            mean = xsg.new_empty(0)
            ctx.mark_non_differentiable(mean)
        else:
            mean = prior_m + dot.reshape(n, 1)
        return mean, var

    @staticmethod
    def backward(ctx, g_mean, g_var):
        spec, xsg = ctx.spec, ctx.xsg
        _, want_xs, want_pm, want_pv = ctx.needs_input_grad
        grad_xs = None
        if want_xs and (g_mean is not None or g_var is not None):
            grad_xs = ops.sparse_posterior_marginals_bwd(spec.flat, xsg, spec.zg, spec.ch_z, spec.ch_s, spec.half_y, g_mean,
                                                         g_var, chunk=spec.chunk)
        shape_m, shape_v = ctx.shapes
        grad_pm = g_mean.sum_to_size(shape_m) if (want_pm and g_mean is not None) else None
        grad_pv = g_var.sum_to_size(shape_v) if (want_pv and g_var is not None) else None
        return None, grad_xs, grad_pm, grad_pv


def sparse_posterior_marginals(spec, xsg, prior_m, prior_v):
    """``(mean, var)`` of a sparse posterior at the pre-stretched test points ``xsg [G, 1, n*, d]``: ``prior_m + dot`` (an empty
    tensor when ``prior_m`` is None) and ``(prior_v - sq_z) + sq_s``, each ``[n*, 1]``, from ``ops.sparse_posterior_marginals``.
    Differentiable w.r.t. ``xsg`` (the factors are constants) and, unchanged, w.r.t. the prior terms ``prior_m`` and
    ``prior_v [n*, 1]``."""
    return _SparsePosteriorMarginals.apply(spec, xsg, prior_m, prior_v)


class _SubspaceCov(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ch, flat, zg, xsg, fwd):
        C, U = fwd()
        ctx.ch, ctx.flat, ctx.zg, ctx.xsg, ctx.U = ch, flat, zg, xsg.detach(), U
        return C

    @staticmethod
    def backward(ctx, gC):
        U, xsg = ctx.U, ctx.xsg
        m, mp, m_pad = xsg.shape[2], U.shape[1], U.shape[2]
        g = gC.reshape(1, m, m)
        D2 = torch.zeros(1, mp, mp, dtype=U.dtype, device=U.device)
        D2[:, :m, :m] = g + g.transpose(1, 2)  # 2 Hs
        Y = ops.gemm_nt(D2, ops.transpose(U, mp, m_pad))  # 2 Hs U
        del D2
        ctx.ch.solve_many_rows_t_(Y)
        grad_xs = torch.zeros_like(xsg)
        ops.kernel_cross_bwd(ctx.flat, xsg, ctx.zg, W=Y, grad_xsg=grad_xs)
        return None, None, None, grad_xs, None


def subspace_cov(ch, flat, zg, xsg, fwd):
    """``U U^T`` as ``fwd()`` computes it -- ``fwd`` returns ``(C, U)`` with ``U = k(x*, z) L_S^-T`` the padded solved rows
    ``[1, m_pad*, m_pad]`` and ``ch`` the factor ``L_S`` -- differentiable w.r.t. the pre-stretched test points ``xsg`` of the
    cross kernel ``flat`` (``zg``: its pre-stretched inducing points; the factor is a constant)."""
    return _SubspaceCov.apply(ch, flat, zg, xsg, fwd)


# ---- exact posterior predictions --------------------------------------------------------------------------------------
#
# K = k(x, x) + noise + eps I = L L^T,  alpha = K^-1 ybar,  K* = k(x*, x),  V = K* L^-T,  W = V L^-1 = K* K^-1.
# Outputs (per problem): dot = K* alpha,  sq = rowsum(V o V),  C = P - V V^T (P = k(x*, x*), lower triangle mirrored).
# With upstream gradients a (dot), s (sq), gC (C), H = -(gC + gC^T) / 2 and D = diag(s) + H:
#   d/dK*  = a alpha^T + 2 D W                         (rectangular K1-backward, factored: no m x n buffer for D = 0)
#   d/dK   = -(beta alpha^T + alpha beta^T) / 2 - W^T D W,   beta = W^T a = K^-1 K*^T a   (square K1-backward)
#   d/dybar = beta,   d/dP = the lower-mirrored gC
class PosteriorSpec:
    """What one exact-posterior evaluation needs beyond its tensor inputs: the factor ``ch`` of ``K_x``, ``K_x``'s flat
    kernel, the cross kernel ``flat_c``, ``half_y = L^-1 ybar`` padded ``[B, n_pad]`` (None without a mean output), and
    ``fwd()``, which runs the launches of the no-grad path and returns ``(dot, sq, cov)`` (None for outputs not formed)."""

    def __init__(self, ch, flat_x, flat_c, half_y, fwd, chunk=4096):
        self.ch, self.flat_x, self.flat_c, self.half_y, self.fwd, self.chunk = ch, flat_x, flat_c, half_y, fwd, chunk


class _ExactPosterior(torch.autograd.Function):
    @staticmethod
    def forward(ctx, spec, coefs_x, xg_x, noise_s, noise_v, ybar, coefs_c, xsg, zg, P, params_x, params_c):
        ctx.set_materialize_grads(False)
        ctx.spec = spec
        ctx.xg_x, ctx.xsg, ctx.zg = xg_x.detach().contiguous(), xsg.detach().contiguous(), zg.detach().contiguous()
        ctx.ybar_shape = None if ybar is None else ybar.shape
        ctx.P_shape = None if P is None else P.shape
        outs = []
        for t in spec.fwd():
            if t is None:
                t = xsg.new_empty(0)
                ctx.mark_non_differentiable(t)
            outs.append(t)
        return tuple(outs)

    @staticmethod
    def backward(ctx, g_dot, g_sq, g_cov):
        return (None,) + _posterior_backward(ctx, g_dot, g_sq, g_cov)


def exact_posterior(spec, coefs_x, xg_x, noise_s, noise_v, ybar, coefs_c, xsg, zg, P=None, params_x=None, params_c=None):
    """``(dot, sq, cov)`` of the exact posterior as ``spec.fwd()`` computes them (an empty tensor for those not formed),
    differentiable w.r.t. ``K_x``'s coefficients, inputs ``xg_x`` and noise (``noise_s``: a float or a tensor; ``noise_v``
    ``[B, n]`` or None), ``ybar [B, n]``, the cross kernel's coefficients, the test points ``xsg``, the data points ``zg``
    (both stretched by the cross kernel's length scales), the prior covariance ``P`` of ``cov`` and the shape parameters of
    ``K_x``'s and the cross kernel (``params_x``, ``params_c``: :func:`param_tensor`)."""
    return _ExactPosterior.apply(spec, coefs_x, xg_x, _scalar(noise_s, xg_x), noise_v, ybar, coefs_c, xsg, zg, P, params_x,
                                 params_c)


def _posterior_backward(ctx, a, s, gc):
    spec, ch = ctx.spec, ctx.spec.ch
    flat_c, flat_x = spec.flat_c, spec.flat_x
    xsg, zg, xg_x = ctx.xsg, ctx.zg, ctx.xg_x
    (_, want_coefs_x, want_xg_x, want_ns, want_nv, want_y, want_coefs_c, want_xs, want_z, want_P, want_params_x,
     want_params_c) = ctx.needs_input_grad
    Bn, n, n_pad, m = ch.batch, ch.n, ch.n_pad, xsg.shape[2]
    dt, dev = ch.dtype, ch.device
    want_K = want_coefs_x or want_xg_x or want_ns or want_nv or want_params_x
    want_cross = want_coefs_c or want_xs or want_z or want_params_c
    a = None if a is None else a.reshape(Bn, m)
    s = None if s is None else s.reshape(Bn, m)
    need_W = (s is not None or gc is not None) and (want_cross or want_K)
    need_beta = a is not None and (want_K or want_y)

    # alpha = K^-1 ybar and beta = K^-1 K*^T a: one-row solves in one 128-row buffer
    alpha = beta = None
    if a is not None and (want_cross or want_K or want_y):
        buf = ch.new_rows(2)
        if need_beta:
            buf[:, 1, :n] = _kt_dot(flat_c, zg, xsg, a)
            ch.solve_rows_(buf)
        buf[:, 0, :] = spec.half_y
        ch.solve_rows_t_(buf)
        alpha, beta = buf[:, 0, :n], buf[:, 1, :n]

    ts_c = torch.zeros(Bn, _lib.GPK_MAX_TERMS, dtype=dt, device=dev) if want_coefs_c else None
    g_xs = torch.zeros_like(xsg) if want_xs else None
    g_z = torch.zeros_like(zg) if want_z else None
    GK = torch.zeros(Bn, n_pad, n_pad, dtype=dt, device=dev) if want_K else None
    ps_c = _param_buf(want_params_c, Bn, xsg)
    cross_out = dict(term_sum=ts_c, grad_xg=g_z, param_sum=ps_c)
    fac = dict(u=a, v=alpha) if a is not None else {}

    if not need_W:
        if want_cross and a is not None:
            ops.kernel_cross_bwd(flat_c, xsg, zg, grad_xsg=g_xs, **fac, **cross_out)
    elif gc is None:
        # marginals: walk the test points in chunks, as the forward does; D = diag(s)
        for c0 in range(0, m, spec.chunk):
            c1 = min(m, c0 + spec.chunk)
            xs_c = xsg[:, :, c0:c1].contiguous()
            Wc = _solved_rows(ch, flat_c, xs_c, zg)
            s_c = s[:, c0:c1]
            if want_cross:
                gxs_c = torch.zeros_like(xs_c) if want_xs else None
                fac_c = dict(u=a[:, c0:c1], v=alpha) if a is not None else {}
                ops.kernel_cross_bwd(flat_c, xs_c, zg, W=Wc, r=2.0 * s_c, grad_xsg=gxs_c, **fac_c, **cross_out)
                if want_xs:
                    g_xs[:, :, c0:c1] = gxs_c
            if want_K:  # GK -= W_c^T diag(s_c) W_c
                cp = Wc.shape[1]
                Wt = ops.transpose(Wc, cp, n_pad)
                del Wc
                sp = torch.zeros(Bn, 1, cp, dtype=dt, device=dev)
                sp[:, 0, : c1 - c0] = s_c
                ops.gemm_nt(Wt * sp, Wt, GK, alpha=-1.0, beta=1.0, lower=True)
    else:
        # full covariance: every test point at once (the forward holds them all too); D = diag(s) + H
        W = _solved_rows(ch, flat_c, xsg, zg)
        mp = W.shape[1]
        D2 = torch.zeros(Bn, mp, mp, dtype=dt, device=dev)
        D2[:, :m, :m] = -(gc.reshape(Bn, m, m) + gc.reshape(Bn, m, m).transpose(1, 2))
        if s is not None:
            D2.diagonal(dim1=1, dim2=2)[:, :m] += 2.0 * s
        Wt = ops.transpose(W, mp, n_pad)
        Y = ops.gemm_nt(D2, Wt)  # 2 D W
        del D2
        if want_cross:
            ops.kernel_cross_bwd(flat_c, xsg, zg, W=Y, grad_xsg=g_xs, **fac, **cross_out)
        if want_K:
            Yt = ops.transpose(Y, mp, n_pad)
            ops.gemm_nt(Wt, Yt, GK, alpha=-0.5, beta=1.0, lower=True)

    grad_coefs_x = grad_xg_x = grad_ns = grad_nv = grad_params_x = None
    if want_K:
        if a is not None:  # GK -= (beta alpha^T + alpha beta^T) / 2
            A2 = torch.zeros(Bn, n_pad, 16, dtype=dt, device=dev)
            B2 = torch.zeros(Bn, n_pad, 16, dtype=dt, device=dev)
            A2[:, :n, 0], A2[:, :n, 1] = beta, alpha
            B2[:, :n, 0], B2[:, :n, 1] = alpha, beta
            ops.gemm_nt(A2, B2, GK, alpha=-0.5, beta=1.0, lower=True)
        ops.symmetrize_(GK, n_pad)
        ps_x = _param_buf(want_params_x, Bn, xg_x)
        term_sum, grad_xg_x, diag = _bwd_kernel(flat_x, xg_x, GK, n, ps_x)
        del GK
        grad_params_x = _param_grad(flat_x, ps_x)
        grad_coefs_x = term_sum[:, : len(flat_x.terms)].sum(0) if want_coefs_x else None
        grad_xg_x = grad_xg_x if want_xg_x else None
        grad_ns = diag.sum() if want_ns else None
        grad_nv = diag if want_nv else None
    grad_y = beta.reshape(ctx.ybar_shape) if (want_y and beta is not None) else None
    grad_coefs_c = ts_c[:, : len(flat_c.terms)].sum(0) if want_coefs_c else None
    grad_P = None
    if want_P:
        g = gc.reshape(-1, m, m)
        grad_P = (torch.tril(g + g.transpose(1, 2), -1) + torch.diag_embed(torch.diagonal(g, dim1=1, dim2=2)))
        grad_P = grad_P.reshape(ctx.P_shape)
    return (grad_coefs_x, grad_xg_x, grad_ns, grad_nv, grad_y, grad_coefs_c, g_xs, g_z, grad_P, grad_params_x,
            _param_grad(flat_c, ps_c))


def _solved_rows(ch, flat_c, xs_c, zg):
    """``W_c = k(x*_c, x) K^-1`` as padded rows ``[B, c_pad, n_pad]``: K1 rows, then both triangular solves in place."""
    Wc = ops.kernel_rows_padded(flat_c, xs_c, zg, ch)
    ch.solve_rows_(Wc)
    ch.solve_many_rows_t_(Wc)
    return Wc


def _kt_dot(flat_c, zg, xsg, a, max_bytes=32 << 20):
    """``u = k(x*, x)^T a`` ``[B, n]``: K1 builds ``k(x, x*_c)`` for chunks of test points small enough that a chunk takes
    at most ``max_bytes``, and one row reduction per chunk contracts it with ``a_c``."""
    Bn, n, m = zg.shape[1], zg.shape[2], xsg.shape[2]
    c = max(128, (max_bytes // (n * zg.element_size())) // 128 * 128)
    u = torch.zeros(Bn, n, dtype=zg.dtype, device=zg.device)
    for c0 in range(0, m, c):
        c1 = min(m, c0 + c)
        Kt = ops.kernel_matrix(flat_c, zg, xsg[:, :, c0:c1].contiguous(), same=False)  # [B, n, c]
        dot, _ = ops.row_dot_sq(Kt, n, c1 - c0, a[:, c0:c1], want_sq=False)
        u += dot
        del Kt
    return u
