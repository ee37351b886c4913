"""``Normal``: a Gaussian with lazily resolved mean / variance -- the hot-path entry point
(``stheno/random.py:48-393``).  ``logpdf`` = ``-(logdet + n log 2 pi + iqf_diag) / 2`` (``:272-279``), with the
kernel-matrix build, Cholesky, triangular solve and log-det fused on the device (``matrix.KernelDense``)."""
from types import FunctionType

import numpy as np
import torch

from . import B
from . import matrix as M
from . import ops
from ._util import NUMPY, batch_flatten, from_dev, origin_of, to_dev, uprank
from .kernels import _grad_tensors

__all__ = ["Random", "RandomProcess", "RandomVector", "Normal"]


class Random:
    def __radd__(self, other):
        return self + other

    def __rmul__(self, other):
        return self * other

    def __neg__(self):
        return -1 * self

    def __sub__(self, other):
        return self + (-other)

    def __rsub__(self, other):
        return (-self) + other

    def __truediv__(self, other):
        return self * (1 / other)


class RandomProcess(Random):
    pass


class RandomVector(Random):
    pass


def _is_zero_scalar(m):
    return isinstance(m, (int, float)) and m == 0


_allow_missing = True
_flag_bufs = {}


class _NanFlag:
    """``isnan(y).any()`` evaluated on the device, its result travelling to pinned host memory behind the caller's back;
    :meth:`read` waits for THAT copy only (an event recorded right after it), not for the stream to drain."""

    def __init__(self, xd):
        key = (xd.device.index or 0, torch.cuda.current_stream(xd.device).cuda_stream)
        slot = _flag_bufs.get(key)
        if slot is None:
            slot = _flag_bufs[key] = [torch.zeros(16, dtype=torch.uint8).pin_memory(), 0]
        buf, i = slot
        slot[1] = (i + 1) % 16  # ring: the host runs at most one evaluation ahead, 16 slots are plenty
        self.cell = buf[i : i + 1]
        self.cell.copy_(torch.isnan(xd).any().to(torch.uint8).reshape(1), non_blocking=True)
        self.event = torch.cuda.Event()
        self.event.record()

    def read(self):
        self.event.synchronize()
        return bool(self.cell.item())


def _loo_structured(var, rhs_t):
    """``(c [B, n], alpha [B, k, n])`` of a Diagonal (``c = 1 / d``) or Woodbury (``D + U U^T``: inversion lemma, ``O(n r^2)``)
    covariance in differentiable torch ops, with the Schur complement regularised by ``B.epsilon`` as in the Woodbury log-pdf."""
    n = rhs_t.shape[-1]
    if isinstance(var, M.Diagonal):
        d = var.diag.reshape(-1, n)
        return 1.0 / d, rhs_t / d.unsqueeze(1)
    d3, H, alpha = _woodbury_inverse(var, rhs_t)
    return 1.0 / d3 - (H * H).sum(1), alpha


def _woodbury_inverse(var, rhs_t):
    """``(d [B, n], H [B, r, n], alpha [B, k, n])`` of a Woodbury covariance ``D + U U^T``: ``Sigma^-1 = D^-1 - H^T H`` with
    ``H = L^-1 U^T D^-1`` (``L L^T`` the Schur complement, regularised by ``B.epsilon``) and ``alpha = Sigma^-1 r``."""
    n = rhs_t.shape[-1]
    U, d = var.lr.left, var.diag_m.diag
    U3 = U.reshape((-1,) + tuple(U.shape[-2:]))
    r = U3.shape[-1]
    d3 = d.reshape(-1, n)
    Ud = U3 / d3.unsqueeze(-1)  # D^-1 U
    S = torch.eye(r, dtype=U.dtype, device=U.device) + U3.transpose(1, 2) @ Ud
    L = torch.linalg.cholesky(S + B.epsilon * torch.eye(r, dtype=U.dtype, device=U.device))
    H = torch.linalg.solve_triangular(L, Ud.transpose(1, 2), upper=False)  # [B, r, n]: L^-1 U^T D^-1
    h = H @ rhs_t.transpose(1, 2)  # [B, r, k]
    alpha = rhs_t / d3.unsqueeze(1) - (H.transpose(1, 2) @ h).transpose(1, 2)
    return d3, H, alpha


def _fold_order(folds, n):
    """``(perm [n] int64, sizes)`` of fold labels: the stable sort of the labels and the sizes of the folds in label order.
    Raises ``ValueError`` unless ``folds`` is a 1-D array or tensor of ``n`` finite integer labels."""
    lab = folds.detach().cpu().numpy() if isinstance(folds, torch.Tensor) else np.asarray(folds)
    if lab.ndim != 1 or lab.shape[0] != n:
        raise ValueError(f"folds must be a 1-D array of {n} labels, got shape {lab.shape}")
    if lab.dtype.kind == "f":
        if not np.isfinite(lab).all() or (lab != np.round(lab)).any():
            raise ValueError("fold labels must be finite integers")
        lab = lab.astype(np.int64)
    elif lab.dtype.kind not in "iu":
        raise ValueError(f"fold labels must be integers, got dtype {lab.dtype}")
    perm = np.argsort(lab, kind="stable")
    sizes = np.unique(lab[perm], return_counts=True)[1]
    return perm, [int(s) for s in sizes]


def _cv_woodbury(var, rhs_t, sizes):
    """``(mean [B, k, n], var [B, n], lp [B, k])`` of a Woodbury covariance whose entries are in fold order, in differentiable
    torch ops: the fold blocks of ``Sigma^-1`` by the inversion lemma, ``D_I^-1 - H_I^T H_I`` (``O(sum n_f^2 r)``), factorised
    in one batch per fold size."""
    d3, H, alpha = _woodbury_inverse(var, rhs_t)
    Bn, k, n = rhs_t.shape
    off = np.concatenate([[0], np.cumsum(sizes)])
    pos, means, vs, lp = [], [], [], 0.0
    for s in sorted(set(sizes)):
        starts = off[:-1][np.asarray(sizes) == s]
        idx = torch.as_tensor(starts[:, None] + np.arange(s)[None, :], device=rhs_t.device)  # [G, s]
        HI = H[:, :, idx].permute(0, 2, 1, 3)  # [B, G, r, s]
        C = torch.diag_embed(1.0 / d3[:, idx]) - HI.transpose(-1, -2) @ HI
        Lc = torch.linalg.cholesky(C)
        aI = alpha[:, :, idx].permute(0, 2, 3, 1)  # [B, G, s, k]
        z = torch.linalg.solve_triangular(Lc, aI, upper=False)
        e = torch.linalg.solve_triangular(Lc.transpose(-1, -2), z, upper=True)
        ldet = 2 * torch.log(torch.diagonal(Lc, dim1=-2, dim2=-1)).sum(-1)  # [B, G]
        lp = lp + 0.5 * ((ldet.sum(1) - len(starts) * s * B.log_2_pi).unsqueeze(-1) - (z * z).sum((1, 2)))
        pos.append(idx.reshape(-1))
        means.append((rhs_t[:, :, idx] - e.permute(0, 3, 1, 2)).reshape(Bn, k, -1))
        vs.append(torch.diagonal(torch.cholesky_inverse(Lc), dim1=-2, dim2=-1).reshape(Bn, -1))
    order = torch.argsort(torch.cat(pos))
    return torch.cat(means, -1)[:, :, order], torch.cat(vs, -1)[:, order], lp


def _loo_torch(c, alpha, r):
    """``gpk_loo_finish``'s forward in differentiable torch ops: ``(mean [B, k, n], var [B, n], lp [B, k])``."""
    s = alpha / c.unsqueeze(1)
    lp = 0.5 * ((torch.log(c).unsqueeze(1) - alpha * s).sum(-1) - c.shape[-1] * B.log_2_pi)
    return r - s, 1.0 / c, lp


class Normal(RandomVector):
    """``Normal(mean, var)``, ``Normal(var)`` or the lazy form ``Normal(mean_fn, var_fn, var_diag=..., mean_var=...,
    mean_var_diag=...)`` whose constructors return DEVICE tensors / matrices (``stheno/random.py:56-94``)."""

    def __init__(self, *args, var_diag=None, mean_var=None, mean_var_diag=None, origin=None):
        if len(args) == 1:
            mean, var = (lambda: 0) if isinstance(args[0], FunctionType) else 0, args[0]
        elif len(args) == 2:
            mean, var = args
        else:
            raise TypeError("Normal(mean, var) or Normal(var)")
        self._origin = origin
        self._var_diag = None
        self._mean_is_zero = None
        if isinstance(var, FunctionType):
            self._mean, self._var = None, None
            self._construct_mean = mean
            self._construct_var = var
            self._construct_var_diag = var_diag
            self._construct_mean_var = mean_var
            self._construct_mean_var_diag = mean_var_diag
        else:
            if self._origin is None:
                self._origin = var.origin if isinstance(var, M.AbstractMatrix) and var.origin is not None else origin_of(var)
            self._var = var if isinstance(var, M.AbstractMatrix) else M.Dense(uprank(to_dev(var)), self._origin)
            if isinstance(mean, M.AbstractMatrix):
                mean = M.dense(mean)
            self._mean = mean if _is_zero_scalar(mean) else uprank(to_dev(mean, self._var.dtype))
            self._construct_var_diag = None
            self._construct_mean_var = None
            self._construct_mean_var_diag = None

    # ---- lazy resolution (stheno/random.py:96-117) -----------------------------------------------------------------
    def _resolve_mean(self, construct_zeros):
        if self._mean is None:
            self._mean = self._construct_mean()
        if self._mean_is_zero is None:
            self._mean_is_zero = _is_zero_scalar(self._mean) or isinstance(self._mean, M.Zero)
        if _is_zero_scalar(self._mean) and construct_zeros:
            v = self._var_dev()
            self._mean = torch.zeros(v.shape[:-2] + (v.shape[-1], 1), dtype=v.dtype, device=v.device)

    def _resolve_var(self):
        if self._var is None:
            self._var = self._construct_var()
        self._var = M.as_matrix(self._var, self._origin)
        if self._var.origin is None:
            self._var.origin = self._origin

    def _resolve_var_diag(self):
        if self._var_diag is None:
            if self._construct_var_diag is not None:
                self._var_diag = self._construct_var_diag()
            else:
                self._var_diag = M.diag(self._var_dev())

    def _var_dev(self):
        self._resolve_var()
        return self._var

    def _mean_dev(self):
        self._resolve_mean(construct_zeros=True)
        return self._mean

    def _out(self, t):
        return from_dev(t, self._origin if self._origin is not None else NUMPY)

    # ---- public properties -----------------------------------------------------------------------------------------
    @property
    def mean(self):
        """Mean as a column ``(n, 1)``."""
        return self._out(self._mean_dev())

    @property
    def mean_is_zero(self):
        self._resolve_mean(construct_zeros=False)
        return self._mean_is_zero

    @property
    def var(self):
        """Variance as a structured matrix (``.mat`` / ``B.dense`` give the plain array)."""
        return self._var_dev()

    @property
    def var_diag(self):
        self._resolve_var_diag()
        return self._out(self._var_diag)

    def _mean_var_dev(self):
        if self._mean is not None and self._var is not None:
            pass
        elif self._mean is None and self._var is None and self._construct_mean_var is not None:
            self._mean, self._var = self._construct_mean_var()
        return self._mean_dev(), self._var_dev()

    @property
    def mean_var(self):
        """``(mean, var)`` computed together when that shares work (``stheno/random.py:173-187``)."""
        m, v = self._mean_var_dev()
        return self._out(m), v

    @property
    def dtype(self):
        return self._var_dev().dtype

    @property
    def dim(self):
        return self._var_dev().shape[-1]

    @property
    def m2(self):
        m = self._mean_dev()
        return self._out(M.dense(self._var_dev()) + m @ m.transpose(-1, -2))

    def _marginals_dev(self):
        if self._mean is not None and self._var_diag is not None:
            pass
        elif self._mean is None and self._var_diag is None and self._construct_mean_var_diag is not None:
            self._mean, self._var_diag = self._construct_mean_var_diag()
        mean = self._mean_dev()
        self._resolve_var_diag()
        vd = self._var_diag
        return mean.squeeze(-1), torch.clamp_min(vd, 0.0)

    def marginals(self):
        """Marginal means and variances, the latter clamped at zero (``stheno/random.py:204-227``)."""
        m, v = self._marginals_dev()
        return self._out(m), self._out(v)

    def marginal_credible_bounds(self):
        """Mean and central 95% bounds ``mean -+ 1.96 sd`` (``stheno/random.py:229-238``)."""
        m, v = self._marginals_dev()
        err = 1.96 * torch.sqrt(v)
        return self._out(m), self._out(m - err), self._out(m + err)

    def diagonalise(self):
        self._resolve_var_diag()
        return Normal(self._mean_dev(), M.Diagonal(self._var_diag, self._origin), origin=self._origin)

    # ---- the hot path ----------------------------------------------------------------------------------------------
    def logpdf(self, x):
        """Log-density of ``x``: ``(n,)``/``(n, 1)`` -> scalar, ``(n, k)`` -> ``(k,)``, batched ``(B, n, 1)`` -> ``(B,)``
        (``stheno/random.py:248-280``).  NaN entries of a single column are treated as missing (``:261-270``)."""
        out_origin = origin_of(x) if self._origin is None else self._origin
        xd = uprank(to_dev(x, None))
        var = self._var_dev()
        xd = xd.to(var.dtype)
        pending = None
        if xd.dim() == 2 and xd.shape[1] == 1:
            # Missing data (``random.py:261-270``).  Host-resident observations are checked on the host.  Device-resident
            # ones: one tiny device reduction whose flag is copied to pinned host memory ASYNCHRONOUSLY and only read
            # after the whole log-pdf has been enqueued (SURVEY H4) -- the host never waits for the device to drain
            # between two evaluations, so the launches of step k + 1 are enqueued while step k still runs.  If the flag
            # does say "NaN" (rare), the enqueued result is discarded and the gather path below runs.
            if isinstance(x, torch.Tensor) and x.is_cuda:
                nan, has_nan = None, False
                if _allow_missing:
                    pending = _NanFlag(xd)
            else:
                host = x.detach().numpy() if isinstance(x, torch.Tensor) else np.asarray(x, dtype=float)
                has_nan = bool(np.isnan(host).any())
                nan = torch.isnan(xd[:, 0]) if has_nan else None
            if has_nan:
                return self._logpdf_missing(xd, nan, var, out_origin)
        n = var.shape[-1]
        diff = xd if self.mean_is_zero else xd - self._mean_dev()
        if isinstance(var, M.Woodbury) and _grad_tensors(var, diff):
            from .generic_grad import woodbury_terms_torch

            ld, q = woodbury_terms_torch(var.lr.left, var.diag_m.diag, diff, B.epsilon)
            lp = -(ld.unsqueeze(-1) + n * B.log_2_pi + q) / 2
        elif isinstance(var, (M.Diagonal, M.Woodbury)):
            ld = M.logdet(var)
            q = M.iqf_diag(var, diff)
            lp = -(ld.unsqueeze(-1) + n * B.log_2_pi + q) / 2
        else:
            if isinstance(var, M.LowRank):
                var = M.Dense(var.dev, var.origin)
            d3, bs = batch_flatten(diff, 2)
            rhs_t = d3.transpose(1, 2).contiguous()  # [B, k, n]: right-hand sides as rows
            if isinstance(var, M.KernelDense) and _grad_tensors(var, rhs_t):
                lp = var.logpdf_grad(rhs_t)  # analytic backward (autograd.py)
            elif not isinstance(var, M.KernelDense) and torch.is_grad_enabled() and _grad_tensors(var.dev, rhs_t):
                # grad mode first: ``dev`` materialises a BlockDense grid, which the fused factorisation below never does
                from .autograd import dense_logpdf

                K3, _ = batch_flatten(var.dev, 2)
                lp = dense_logpdf(K3, rhs_t, B.epsilon)  # gradient w.r.t. the assembled covariance itself
            elif var._chol is None:
                key = ("logpdf", id(xd))
                var.attach_rhs(key, rhs_t)
                ch = var.chol()
                a, b = var._rhs_slices[key]
                lp = ch.logpdf()[:, a:b]
            else:
                ch = var.chol()
                half = ch.half_solve(rhs_t)
                lp = -(ch.logdet.unsqueeze(-1) + n * B.log_2_pi + (half * half).sum(-1)) / 2
            lp = lp.reshape(bs + (lp.shape[-1],))
        lp = lp[..., 0] if lp.shape[-1] == 1 else lp
        if pending is not None and pending.read():
            return self._logpdf_missing(xd, torch.isnan(xd[:, 0]), var, out_origin)
        return from_dev(lp, out_origin)

    def _logpdf_missing(self, xd, nan, var, out_origin):
        avail = ~nan
        sub = Normal(self._mean_dev()[avail], M.submatrix(var, avail), origin=self._origin)
        return sub.logpdf(from_dev(xd[avail], out_origin))

    # ---- leave-one-out predictive distributions (model checking, LOO cross-validation) --------------------------------
    def loo_marginals(self, x):
        """Mean and variance of every ``x_i`` given all the other entries of its column: ``(n,)``/``(n, 1)`` -> ``(n,)``
        and ``(n,)``, ``(n, k)`` -> ``(n, k)`` and ``(n,)`` (the variance does not depend on ``x``), batched ``(B, n, 1)``
        -> ``(B, n)`` and ``(B, n)``.  NaN entries of a single column are missing: the others are predicted from the
        observed ones, and missing positions get NaN.  With ``Sigma = var + B.epsilon I``, ``c = diag Sigma^-1`` and
        ``alpha = Sigma^-1 (x - mean)``: mean ``x_i - alpha_i / c_i``, variance ``1 / c_i``.  Gradients flow through
        diagonal and Woodbury covariances only; elsewhere a backward through these values raises."""
        return self._loo(x, marginals=True)

    def loo_logpdf(self, x):
        """``sum_i log p(x_i | x_-i)``, the leave-one-out log predictive density, with the output shapes of
        :meth:`logpdf` and its missing-data rule.  Differentiable like :meth:`logpdf`: every route has a gradient, the
        kernel-matrix one an analytic one on the GPU."""
        return self._loo(x, marginals=False)

    def _loo(self, x, marginals):
        out_origin = origin_of(x) if self._origin is None else self._origin
        var = self._var_dev()
        xd = uprank(to_dev(x, None)).to(var.dtype)
        pending = None
        if xd.dim() == 2 and xd.shape[1] == 1:  # missing data, detected as in logpdf
            if isinstance(x, torch.Tensor) and x.is_cuda:
                if _allow_missing:
                    pending = _NanFlag(xd)
            else:
                host = x.detach().numpy() if isinstance(x, torch.Tensor) else np.asarray(x, dtype=float)
                if np.isnan(host).any():
                    return self._loo_missing(xd, marginals, out_origin)
        n = var.shape[-1]
        diff = xd if self.mean_is_zero else xd - self._mean_dev()
        d3, bs = batch_flatten(diff, 2)
        rhs_t = d3.transpose(1, 2).contiguous()  # [B, k, n]
        if isinstance(var, (M.Diagonal, M.Woodbury)):
            c, alpha = _loo_structured(var, rhs_t)
            mean_r, v, lp = _loo_torch(c, alpha, rhs_t)
        else:
            if isinstance(var, M.LowRank):
                var = M.Dense(var.dev, var.origin)
            ts = _grad_tensors(var, rhs_t)  # walks the blocks of a BlockDense: never materialises it
            mean_r = v = None
            if ts and not marginals and isinstance(var, M.KernelDense):
                lp = var.loo_grad(rhs_t)
            elif ts and not marginals:
                from .autograd import dense_loo

                K3, _ = batch_flatten(var.dev, 2)
                lp = dense_loo(K3, rhs_t, B.epsilon)  # gradient w.r.t. the assembled covariance itself
            else:
                ch = var.loo_chol(rhs_t.detach()) if isinstance(var, M.KernelDense) else var._factorize(rhs_t.detach())
                mean_r, v, lp, _, _ = ch.loo(rhs_t.detach(), want_mean=marginals)
                if ts:  # raw-pointer values: a gradient through them would be silently wrong
                    from .autograd import no_gradient

                    mean_r, v = no_gradient("loo_marginals", mean_r, ts), no_gradient("loo_marginals", v, ts)
        if pending is not None and pending.read():
            return self._loo_missing(xd, marginals, out_origin)
        if not marginals:
            lp = lp.reshape(bs + (lp.shape[-1],))
            return from_dev(lp[..., 0] if lp.shape[-1] == 1 else lp, out_origin)
        mean = mean_r.transpose(1, 2).reshape(bs + (n, rhs_t.shape[1]))
        if not self.mean_is_zero:
            mean = mean + self._mean_dev()
        mean = mean[..., 0] if mean.shape[-1] == 1 else mean
        return from_dev(mean, out_origin), from_dev(v.reshape(bs + (n,)), out_origin)

    def _loo_missing(self, xd, marginals, out_origin):
        avail = ~torch.isnan(xd[:, 0])
        sub = Normal(self._mean_dev()[avail], M.submatrix(self._var_dev(), avail), origin=self._origin)
        res = sub._loo(from_dev(xd[avail], out_origin), marginals)
        if not marginals:
            return res
        out = []
        for t in res:
            t = to_dev(t, xd.dtype)
            full = torch.full((xd.shape[0],), float("nan"), dtype=xd.dtype, device=t.device)
            out.append(from_dev(full.masked_scatter(avail.to(t.device), t), out_origin))
        return tuple(out)

    # ---- multi-fold cross-validation (blocked / grouped / K-fold) ----------------------------------------------------------
    def cv_marginals(self, x, folds):
        """Mean and variance of every ``x_i`` given all the entries outside its fold, with the shapes of
        :meth:`loo_marginals`.  ``folds``: ``n`` integer labels (array or tensor; any values, in any order); entries with
        one label form a fold, and one ``folds`` serves every batch member and column.  NaN entries of a single column are
        missing: dropped before folding, with NaN marginals.  With ``Sigma = var + B.epsilon I``, ``C = Sigma^-1``,
        ``alpha = C (x - mean)`` and ``C_II`` the block of fold ``I``: mean ``x_I - C_II^-1 alpha_I``, variance
        ``diag C_II^-1``.  Singleton folds give :meth:`loo_marginals`, a single fold the prior marginals.  Gradients flow
        through diagonal and Woodbury covariances only; elsewhere a backward through these values raises."""
        return self._cv(x, folds, marginals=True)

    def cv_logpdf(self, x, folds):
        """``sum_I log p(x_I | x_-I)`` over the folds of ``folds`` (as in :meth:`cv_marginals`), with the output shapes of
        :meth:`logpdf` and its missing-data rule; a fold whose entries are all missing contributes nothing.  Singleton
        folds give :meth:`loo_logpdf`, a single fold :meth:`logpdf`.  Differentiable on every route, the kernel-matrix
        one with an analytic gradient on the GPU."""
        return self._cv(x, folds, marginals=False)

    def _cv(self, x, folds, marginals):
        out_origin = origin_of(x) if self._origin is None else self._origin
        var = self._var_dev()
        xd = uprank(to_dev(x, None)).to(var.dtype)
        n = var.shape[-1]
        perm, sizes = _fold_order(folds, n)
        if max(sizes, default=1) == 1:  # singleton folds are leave-one-out, without a 128-padded workspace per entry
            return self._loo(x, marginals)
        pending = None
        if xd.dim() == 2 and xd.shape[1] == 1:  # missing data, detected as in logpdf
            if isinstance(x, torch.Tensor) and x.is_cuda:
                if _allow_missing:
                    pending = _NanFlag(xd)
            else:
                host = x.detach().numpy() if isinstance(x, torch.Tensor) else np.asarray(x, dtype=float)
                if np.isnan(host).any():
                    return self._cv_missing(xd, folds, marginals, out_origin)
        diff = xd if self.mean_is_zero else xd - self._mean_dev()
        d3, bs = batch_flatten(diff, 2)
        rhs_t = d3.transpose(1, 2).contiguous()  # [B, k, n]
        p = torch.as_tensor(perm, device=rhs_t.device)
        rhs_p = rhs_t[:, :, p]  # fold order: fold f is one contiguous range of entries
        if isinstance(var, M.Diagonal):  # the folds decouple into single entries: leave-one-out
            c, alpha = _loo_structured(var, rhs_t)
            mean_r, v, lp = _loo_torch(c, alpha, rhs_t)
            p = None
        elif isinstance(var, M.Woodbury):
            vp = M.Woodbury(M.Diagonal(var.diag_m.diag[..., p], var.origin), M.LowRank(var.lr.left[..., p, :], var.origin))
            mean_r, v, lp = _cv_woodbury(vp, rhs_p, sizes)
        else:
            if isinstance(var, M.LowRank):
                var = M.Dense(var.dev, var.origin)
            ts = _grad_tensors(var, rhs_t)
            mean_r = v = None
            if isinstance(var, M.KernelDense):
                vp = var.permuted(p)
                if ts and not marginals:
                    lp = vp.cv_grad(rhs_p, sizes)
                else:
                    ch = vp.loo_chol(rhs_p.detach())
            elif ts and not marginals:
                from .autograd import dense_cv

                K3, _ = batch_flatten(var.dev, 2)
                lp = dense_cv(K3[:, p][:, :, p], rhs_p, B.epsilon, sizes)  # gradient w.r.t. the assembled covariance
            else:
                K3, _ = batch_flatten(var.dev, 2)
                ch = ops.chol_from_dense(K3.detach()[:, p][:, :, p], jitter=B.epsilon, rhs_t=rhs_p.detach())
            if marginals or not ts:
                mean_r, v, lp, _ = ch.cv(rhs_p.detach(), sizes, want_mean=marginals)
                del ch
                if ts:  # raw-pointer values: a gradient through them would be silently wrong
                    from .autograd import no_gradient

                    mean_r, v = no_gradient("cv_marginals", mean_r, ts), no_gradient("cv_marginals", v, ts)
        if pending is not None and pending.read():
            return self._cv_missing(xd, folds, marginals, out_origin)
        if not marginals:
            lp = lp.reshape(bs + (lp.shape[-1],))
            return from_dev(lp[..., 0] if lp.shape[-1] == 1 else lp, out_origin)
        if p is not None:  # back to the caller's order
            inv = torch.empty_like(p)
            inv[p] = torch.arange(n, device=p.device)
            mean_r, v = mean_r[:, :, inv], v[:, inv]
        mean = mean_r.transpose(1, 2).reshape(bs + (n, rhs_t.shape[1]))
        if not self.mean_is_zero:
            mean = mean + self._mean_dev()
        mean = mean[..., 0] if mean.shape[-1] == 1 else mean
        return from_dev(mean, out_origin), from_dev(v.reshape(bs + (n,)), out_origin)

    def _cv_missing(self, xd, folds, marginals, out_origin):
        avail = ~torch.isnan(xd[:, 0])
        lab = folds.detach().cpu() if isinstance(folds, torch.Tensor) else torch.as_tensor(np.asarray(folds))
        sub = Normal(self._mean_dev()[avail], M.submatrix(self._var_dev(), avail), origin=self._origin)
        res = sub._cv(from_dev(xd[avail], out_origin), lab[avail.cpu()], marginals)
        if not marginals:
            return res
        out = []
        for t in res:
            t = to_dev(t, xd.dtype)
            full = torch.full((xd.shape[0],), float("nan"), dtype=xd.dtype, device=t.device)
            out.append(from_dev(full.masked_scatter(avail.to(t.device), t), out_origin))
        return tuple(out)

    def entropy(self):
        return self._out((M.logdet(self._var_dev()) + self.dim * (B.log_2_pi + 1)) / 2)

    def kl(self, other):
        """KL(self || other) (``stheno/random.py:293-309``)."""
        d = other._mean_dev() - self._mean_dev()
        out = (
            M.iqf_diag(other._var_dev(), d)[..., 0]
            + M.ratio(self._var_dev(), other._var_dev())
            + M.logdet(other._var_dev())
            - M.logdet(self._var_dev())
            - self.dim
        ) / 2
        return self._out(out)

    def w2(self, other):
        """2-Wasserstein distance to another normal (``stheno/random.py:311-329``).  ``B.root`` (the symmetric PSD square
        root) comes from a library symmetric eigensolver (``torch.linalg.eigh`` = cuSOLVER): this is off the hot path."""

        def root(a):
            lam, v = torch.linalg.eigh((a + a.transpose(-1, -2)) / 2)
            return (v * lam.clamp_min(0).sqrt().unsqueeze(-2)) @ v.transpose(-1, -2)

        a, b = M.dense(self._var_dev()), M.dense(other._var_dev())
        ra = root(a)
        r = root(ra @ b @ ra)
        tr = lambda t: torch.diagonal(t, dim1=-2, dim2=-1).sum(-1)
        var_part = tr(a) + tr(b) - 2 * tr(r)
        mean_part = ((self._mean_dev() - other._mean_dev()) ** 2).sum((-1, -2))
        return self._out(torch.sqrt(torch.clamp(mean_part + var_part, min=0)))

    # ---- sampling (SURVEY 8f rank 1) -----------------------------------------------------------------------------
    def sample(self, *args, num=1, noise=None):
        """``sample([state,] num=1, noise=None)`` -> ``(n, num)`` samples ``mean + L eps``
        (``stheno/random.py:331-363``).  ``state`` is a ``torch.Generator``; returns ``(state, sample)`` then."""
        state = None
        if args and isinstance(args[0], torch.Generator):
            state, args = args[0], args[1:]
        if args:
            num = int(args[0])
        var = self._var_dev()
        if noise is not None:
            n = var.shape[-1]
            var = M.add(var, M.fill_diag(float(noise), n, var.dtype, var.device, self._origin))
        n = var.shape[-1]
        bs = tuple(var.shape[:-2])
        if isinstance(var, M.Diagonal):
            eps = torch.randn(bs + (n, num), dtype=var.dtype, device=var.device, generator=state)
            s = torch.sqrt(var.diag).unsqueeze(-1) * eps
        elif isinstance(var, M.Zero):
            s = torch.zeros(bs + (n, num), dtype=var.dtype, device=var.device)
        else:
            # mean + L eps with L read straight from the factorisation workspace by the in-tree tensor-core GEMM:
            # (L eps)^T = eps^T L^T is an "NT" product with both operands K-contiguous (no tril copy, no library GEMM)
            ch = M.cholesky(var)
            eps = torch.randn((ch.batch, n, num), dtype=var.dtype, device=var.device, generator=state)
            E = torch.zeros(ch.batch, ops.round_up(max(num, 1)), ch.n_pad, dtype=var.dtype, device=var.device)
            E[:, :num, :n] = eps.transpose(1, 2)
            St = ops.gemm_nt(E, ch.L_lower_())
            s = St[:, :num, :n].transpose(1, 2).reshape(bs + (n, num))
            ts = _grad_tensors(var)
            if ts:  # L eps comes from the raw-pointer factorisation: a gradient through it would be silently wrong
                from .autograd import no_gradient

                s = no_gradient("sampling", s, ts)
        if not self.mean_is_zero:
            s = s + self._mean_dev()
        s = self._out(s)
        return (state, s) if state is not None else s

    # ---- arithmetic ------------------------------------------------------------------------------------------------
    def __add__(self, other):
        if isinstance(other, Normal):
            return Normal(self._mean_dev() + other._mean_dev(), M.add(self._var_dev(), other._var_dev()),
                          origin=self._origin)
        return Normal(self._mean_dev() + other, self._var_dev(), origin=self._origin)

    def __mul__(self, other):
        return Normal(self._mean_dev() * other, M.Dense(M.dense(self._var_dev()) * other**2, self._origin),
                      origin=self._origin)

    def lmatmul(self, other):
        a = to_dev(other, self.dtype)
        return Normal(a @ self._mean_dev(), M.Dense(a @ M.dense(self._var_dev()) @ a.transpose(-1, -2), self._origin),
                      origin=self._origin)

    def rmatmul(self, other):
        a = to_dev(other, self.dtype)
        return Normal(a.transpose(-1, -2) @ self._mean_dev(),
                      M.Dense(a.transpose(-1, -2) @ M.dense(self._var_dev()) @ a, self._origin), origin=self._origin)

    def __str__(self):
        m = "unresolved" if self._mean is None else str(self._mean)
        v = "unresolved" if self._var is None else str(self._var)
        return f"<Normal:\n    mean={m},\n    var={v}>"

    __repr__ = __str__
