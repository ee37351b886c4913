"""Pathwise function samples (Wilson et al. 2020, "Efficiently sampling functions from Gaussian process posteriors"):
a sample drawn once and evaluated at any points, in any number of calls.  Device memory beyond the factor: the ``[n, num]``
output, the (mapped) points and one ``chunk x n_pad`` block of K1 rows of the update; never an ``n x F`` feature matrix.

    prior:      f~(x) = m(x) + sum_t sqrt(2 c_t / F_t) sum_j w_j cos(omega_j . x / l_t + b_j) + sum_lin sqrt(c) x . w / l
    posterior:  f(x)  = f~(x) + k(x, X) V^T,   V = K^-1 (y - f~(X) - eps),   K = k(X, X) + Sigma_noise + B.epsilon I

The cosine features run in ``gpk_feature_eval`` (``csrc/sample_fn.cu``), which never holds the n x F feature matrix; the
update reuses the factor of ``K`` that ``Observations.K_x`` keeps, the K1 rows and the tensor-core GEMM.

Spectral measures of the unit-length-scale factors of ``include/gpk.h``:
    EQ ``exp(-r^2 / 2)``:                 omega ~ N(0, I)
    Matern-nu (nu = 1/2, 3/2, 5/2):       omega = z / sqrt(u),  z ~ N(0, I),  u ~ Gamma(nu, rate nu)  (multivariate t, 2 nu dof)
    RQ ``(1 + r^2 / (2 alpha))^-alpha``:  omega = sqrt(tau) z,  tau ~ Gamma(alpha, rate alpha)  (a Gamma mixture of EQs)
    One ``1``:                            omega = 0
"""
import math

import numpy as np
import torch

from . import _util, ops
from . import matrix as M
from ._util import from_dev
from .kernels import (DerivativeKernel, FunctionScaledKernel, MappedKernel, PosteriorKernel, PosteriorMean, SubspaceKernel,
                      _children, _grad_tensors, _is_multi, _same_map, as_input, k1_block)

__all__ = ["FunctionSample"]

_MATERN_NU = {"matern12": 0.5, "matern32": 1.5, "matern52": 2.5}
_STATIONARY = ("eq", "rq", "one") + tuple(_MATERN_NU)


def _contains(k, cls):
    return isinstance(k, cls) or any(_contains(c, cls) for c in _children(k))


def _terms(kernel):
    """``(stationary, linear, scales)`` of a covered kernel: ``stationary`` = ``[(coef, kind, group, param)]``, ``linear`` =
    ``[(coef, group)]``, ``scales`` the length scales per group (:meth:`Kernel._flat`).  Raises ``ValueError`` naming what is
    not covered."""
    if hasattr(kernel, "_elwise_multi"):
        raise ValueError("function sampling covers single-output processes, not multi-output kernels")
    k = kernel
    while isinstance(k, MappedKernel):
        if not _same_map(k.m1, k.m2):
            raise ValueError("function sampling needs a kernel whose input maps act on both arguments alike")
        k = k.k
    if _contains(k, DerivativeKernel):
        raise ValueError("function sampling does not cover derivative kernels")
    if _contains(k, FunctionScaledKernel):
        raise ValueError("function sampling does not cover function-scaled kernels")
    if isinstance(k, (PosteriorKernel, SubspaceKernel)) or _contains(k, PosteriorKernel):
        raise ValueError("function sampling conditions a prior once: the kernel is already a posterior kernel")
    flat, scales = k._flat()
    if flat is None:
        raise ValueError(f"function sampling needs a kernel that flattens to one sum of scaled terms, not {k.render()}")
    stationary, linear = [], []
    for coef, fs in flat.terms:
        kinds = [f[0] for f in fs]
        if "delta" in kinds:
            raise ValueError("function sampling does not cover Delta terms: white noise is not a function")
        fs = [f for f in fs if f[0] != "one"] or fs[:1]  # a constant factor 1 changes nothing
        if len(fs) > 1:
            raise ValueError("function sampling does not cover products of kernel factors: their spectral measure is a "
                             "convolution")
        if coef < 0:
            raise ValueError("function sampling needs non-negative term coefficients")
        kind, g = fs[0][0], fs[0][1]
        if kind == "linear":
            linear.append((coef, g))
        elif kind in _STATIONARY:
            stationary.append((coef, kind, g, fs[0][2] if len(fs[0]) > 2 else None))
        else:
            raise ValueError(f"function sampling does not cover {kind} factors")
    return stationary, linear, scales


def _posterior_parts(mean, kernel):
    """``(prior mean, prior kernel, PosteriorMean or None)`` of a GP; raises ``ValueError`` for the posteriors not covered."""
    if isinstance(kernel, SubspaceKernel) or _contains(kernel, SubspaceKernel):
        raise ValueError("function sampling does not cover sparse (PseudoObs) posteriors")
    if not isinstance(kernel, PosteriorKernel) and not isinstance(mean, PosteriorMean):
        return mean, kernel, None
    if not (isinstance(mean, PosteriorMean) and isinstance(kernel, PosteriorKernel)):
        raise ValueError("function sampling needs the mean and kernel of one exact posterior")
    if _is_multi(kernel.z) or isinstance(kernel.K_z, M.BlockDense):
        raise ValueError("function sampling does not cover posteriors of several observed processes")
    if not (kernel.k_zi is kernel.k_ij and kernel.k_zj is kernel.k_ij and mean.m_i is mean.m_z and mean.K_z is kernel.K_z):
        raise ValueError("function sampling covers the observed process itself, not the prediction of another process")
    if not isinstance(kernel.K_z, M.KernelDense):
        raise ValueError("function sampling needs observations whose covariance is a kernel matrix plus scalar or diagonal "
                         "noise")
    if kernel.K_z.chol().batch != 1:
        raise ValueError("function sampling does not cover batched observations")
    return mean.m_i, kernel.k_ij, mean


def _scale_tensor(s, d, device):
    """A length scale (None, number, array or tensor) as a ``[d]`` fp64 tensor on ``device``, without a graph."""
    if s is None:
        return torch.ones(d, dtype=torch.float64, device=device)
    t = s.detach() if isinstance(s, torch.Tensor) else torch.as_tensor(np.asarray(s, np.float64))
    return t.to(device=device, dtype=torch.float64).reshape(-1).expand(d).clone()


def _gamma(shape, size, gen, device):
    """``size`` draws of Gamma(shape, rate 1) from ``gen`` (Marsaglia and Tsang; shape < 1 boosted by ``U^(1/shape)``)."""
    a = float(shape)
    a1 = a + 1.0 if a < 1.0 else a
    dd = a1 - 1.0 / 3.0
    c = 1.0 / math.sqrt(9.0 * dd)
    out = torch.empty(size, dtype=torch.float64, device=device)
    todo = torch.arange(size, device=device)
    while todo.numel():
        z = torch.randn(todo.numel(), dtype=torch.float64, device=device, generator=gen)
        u = torch.rand(todo.numel(), dtype=torch.float64, device=device, generator=gen)
        v = (1.0 + c * z) ** 3
        ok = (v > 0) & (torch.log(u) < 0.5 * z * z + dd - dd * v + dd * torch.log(v.clamp_min(1e-300)))
        out[todo[ok]] = dd * v[ok]
        todo = todo[~ok]
    if a < 1.0:
        out *= torch.rand(size, dtype=torch.float64, device=device, generator=gen) ** (1.0 / a)
    return out


def spectral_draw(kind, param, count, d, gen, device):
    """``count`` frequencies ``[count, d]`` (fp64) of the unit-length-scale factor ``kind`` (module docstring)."""
    z = torch.randn(count, d, dtype=torch.float64, device=device, generator=gen)
    if kind == "eq":
        return z
    if kind == "one":
        return torch.zeros_like(z)
    if kind in _MATERN_NU:
        dof = int(2 * _MATERN_NU[kind])  # Gamma(nu, rate nu) = chi^2_(2 nu) / (2 nu)
        chi2 = (torch.randn(count, dof, dtype=torch.float64, device=device, generator=gen) ** 2).sum(1)
        return z / torch.sqrt(chi2 / dof).unsqueeze(1)
    if kind == "rq":
        tau = _gamma(param, count, gen, device) / float(param)
        return z * torch.sqrt(tau).unsqueeze(1)
    raise ValueError(kind)


class FunctionSample:
    """``num`` functions drawn from a GP (prior or exact posterior, :meth:`GP.sample_function`); ``sample(x)`` is ``(n, num)``.

    The draws come from a generator of the compute device seeded once from ``state`` (a ``torch.Generator``; the global one
    when None), so equal states give equal functions.  A prior's frequencies are drawn at its first evaluation, when the input
    dimension is known; later evaluations must have that dimension.  After drawing, ``omega [F, d]`` (divided by the length
    scales), ``b [F]``, ``amp [F]``, ``W [num, F]``, ``linear [d, num]`` (or None) and, for a posterior, ``eps [n, num]`` and
    ``V [1, num_pad, n_pad]`` (rows ``K^-1 (y - f~(X) - eps)``) hold them, fp64 except ``V``."""

    def __init__(self, gp, num=1, features=4096, state=None, chunk=2048):
        self.num, self.features, self.chunk = int(num), int(features), int(chunk)
        if self.num < 1 or self.features < 1:
            raise ValueError("function sampling needs num >= 1 and features >= 1")
        self._gp_mean, self._gp_kernel = gp.mean, gp.kernel
        self.mean, self.kernel, self._post = _posterior_parts(gp.mean, gp.kernel)
        self._stationary, self._linear, self._scales = _terms(self.kernel)
        if self.features < len(self._stationary):
            raise ValueError(f"{len(self._stationary)} stationary terms need at least as many features")
        self.device = _util._device_fn()
        seed = int(torch.randint(0, 2**62, (1,), generator=state,
                                 device=state.device if state is not None else "cpu").item())
        self._gen = torch.Generator(device=self.device).manual_seed(seed)
        self.omega = None
        self.eps = self.V = None
        if self._post is not None:
            with torch.no_grad():
                self._condition()

    # ---- the prior sample f~ -----------------------------------------------------------------------------------------
    def _draw(self, d):
        """Frequencies, phases and weights for mapped inputs of dimension ``d``."""
        gen, dev, num, scales = self._gen, self.device, self.num, self._scales
        T = len(self._stationary)
        omegas, amps = [], []
        for t, (coef, kind, g, param) in enumerate(self._stationary):
            F_t = self.features // T + (1 if t < self.features % T else 0)
            omegas.append(spectral_draw(kind, param, F_t, d, gen, dev) / _scale_tensor(scales[g], d, dev))
            amps.append(torch.full((F_t,), math.sqrt(2.0 * coef / F_t), dtype=torch.float64, device=dev))
        F = sum(o.shape[0] for o in omegas)
        self.omega = torch.cat(omegas) if omegas else torch.zeros(0, d, dtype=torch.float64, device=dev)
        self.amp = torch.cat(amps) if amps else torch.zeros(0, dtype=torch.float64, device=dev)
        self.b = 2 * math.pi * torch.rand(F, dtype=torch.float64, device=dev, generator=gen)
        self.W = torch.randn(num, F, dtype=torch.float64, device=dev, generator=gen)
        self.linear = None
        for coef, g in self._linear:
            w = torch.randn(d, num, dtype=torch.float64, device=dev, generator=gen)
            part = math.sqrt(coef) * w / _scale_tensor(scales[g], d, dev).unsqueeze(1)
            self.linear = part if self.linear is None else self.linear + part
        self._cast = {}

    def _params(self, dtype):
        if dtype not in self._cast:
            self._cast[dtype] = [None if t is None else t.to(dtype) for t in (self.omega, self.b, self.amp, self.W,
                                                                              self.linear)]
        return self._cast[dtype]

    def _prior(self, xi):
        """``f~`` at the points of the :class:`Input` ``xi``: ``[n, num]``."""
        _, _, xm, _ = k1_block(self.kernel, xi, through_maps=True, zero=True)
        t = xm.t
        if self.omega is None:
            self._draw(t.shape[-1])
        elif t.shape[-1] != self.omega.shape[1]:
            raise ValueError(f"this function sample was drawn for inputs of dimension {self.omega.shape[1]} (after the "
                             f"kernel's input maps), not {t.shape[-1]}")
        omega, b, amp, W, lin = self._params(t.dtype)
        out = self.mean.dev(xi).reshape(-1, 1).expand(-1, self.num).contiguous()
        if omega.shape[0]:
            ops.feature_eval(t, omega, b, amp, W, out=out)
        if lin is not None:
            out += t @ lin
        return out

    # ---- the update ----------------------------------------------------------------------------------------------------
    def _condition(self):
        post = self._post
        K = post.K_z
        ch = K.chol()
        X = post.z
        n, dtype = ch.n, ch.dtype
        fX = self._prior(X)
        var = torch.full((n,), K.noise_scalar, dtype=torch.float64, device=self.device)
        if K.noise_vec is not None:
            var = var + K.noise_vec.detach().reshape(-1).to(torch.float64)
        self.eps = torch.sqrt(var.clamp_min(0)).unsqueeze(1) * torch.randn(n, self.num, dtype=torch.float64,
                                                                            device=self.device, generator=self._gen)
        rhs = post.y.detach().reshape(n, 1).to(dtype) - fX - self.eps.to(dtype)
        V = ch.new_rows(self.num)
        V[0, : self.num, :n] = rhs.transpose(0, 1)
        ch.solve_rows_(V)
        ch.solve_rows_t_(V)
        self.V = V
        self._zg = None

    def _update(self, xi):
        """``k(x, X) V^T`` at the points of ``xi``: ``[n, num]``."""
        post = self._post
        ch = post.K_z.chol()
        flat, scales, zm, xm = k1_block(post.k_zi, post.z, xi, through_maps=True)
        if self._zg is None:
            self._zg = zm.scaled(scales)
        rows = ops.kernel_rows_padded(flat, xm.scaled(scales), self._zg, ch)
        # rows V^T has one 128-column tile for up to 128 samples: split the n_pad-long reduction into `s` batched partial
        # products so that s times as many CTAs share it (each part a multiple of 32 long, as the fp32 tensor-core GEMM needs)
        s = 8 if ch.n_pad % 256 == 0 else 4
        k, c_pad = ch.n_pad // s, rows.shape[1]
        A = rows[0].view(c_pad, s, k).transpose(0, 1)
        Bm = self.V[0].view(self.V.shape[1], s, k).transpose(0, 1)
        return ops.gemm_nt(A, Bm).sum(0)[: xi.n, : self.num]

    # ---- evaluation ----------------------------------------------------------------------------------------------------
    def __call__(self, x):
        """The ``num`` functions at ``x`` (``(n,)`` or ``(n, d)``): ``(n, num)``, numpy for numpy input, else a tensor on the
        input's device."""
        if _is_multi(x):
            raise ValueError("function sampling covers single-output inputs, not multi-output ones")
        xi = as_input(x)
        if xi.batch_shape:
            raise ValueError("function sampling does not cover batched inputs")
        dtype = self.V.dtype if self.V is not None else xi.t.dtype
        ts = _grad_tensors(self._gp_mean, self._gp_kernel, xi)
        with torch.no_grad():
            xd = as_input(xi.t.detach().to(dtype))
            out = self._prior(xd)  # one feature launch over every point: the kernel holds no n x F buffer
            if self._post is not None:  # the update holds a chunk x n_pad block of K1 rows: chunked
                for a in range(0, xd.n, self.chunk):
                    out[a : a + self.chunk] += self._update(as_input(xd.t[a : a + self.chunk]))
        if ts:
            from .autograd import no_gradient

            out = no_gradient("function sampling", out, ts)
        return from_dev(out, xi.origin)
