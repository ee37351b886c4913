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
