"""Kernels and means: the slice of ``mlkernels`` on the GP hot path (SURVEY.md 2.2 E1), re-designed so that a
whole kernel *expression* (scale / sum / product / stretch of EQ, Matern12/32/52, Linear, Delta) is flattened to
one descriptor and evaluated by ONE fused CUDA kernel (``csrc/kernel_matrix.cu``) instead of one pass per node.

Reference call sites: ``p.kernel(x)`` ``stheno/model/fdd.py:79``; ``k.elwise(x)`` ``fdd.py:66``;
``measure.kernels[...](z, x)`` ``stheno/model/observations.py:139,285,286,304``; ``PosteriorKernel`` /
``PosteriorMean`` / ``SubspaceKernel`` ``observations.py:148-168,255-277``.
Formulas [UPSTREAM-RECALLED] as restated in ``oracle/gp_oracle.py``.
"""
import itertools
from types import FunctionType

import numpy as np
import torch

from . import matrix as M
from . import ops
from ._lib import GpkError as _GpkError
from ._util import batch_flatten, from_dev, origin_of, to_dev, uprank

__all__ = [
    "Kernel", "EQ", "RQ", "Exp", "Matern12", "Matern32", "Matern52", "Linear", "Delta", "OneKernel", "ZeroKernel",
    "ScaledKernel", "SumKernel", "ProductKernel", "StretchedKernel", "ReversedKernel", "PosteriorKernel",
    "SubspaceKernel", "Mean", "ZeroMean", "OneMean", "ScaledMean", "SumMean", "ProductMean", "StretchedMean",
    "FunctionMean", "DerivativeMean", "DerivativeKernel", "PosteriorMean", "mean_var", "mean_var_diag", "num_elements", "pairwise", "elwise",
]


# ------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------
class Input:
    """A numeric input on the device, ``[..., n, d]`` (vectors are up-ranked to columns like ``B.uprank``)."""

    __slots__ = ("t", "origin", "_groups", "src")

    def __init__(self, x):
        self.origin = origin_of(x)
        self.t = uprank(to_dev(x))
        self._groups = {}
        self.src = x  # the caller's object: "x is y" semantics of the reference survive the move to the device

    @property
    def n(self):
        return self.t.shape[-2]

    @property
    def d(self):
        return self.t.shape[-1]

    @property
    def batch_shape(self):
        return tuple(self.t.shape[:-2])

    def scaled(self, scales):
        """``[G, B, n, d]``: one pre-stretched copy of the points per distinct length scale (``x / scale``)."""
        key = tuple(_scale_key(s) for s in scales)
        if key not in self._groups:
            t3, _ = batch_flatten(self.t, 2)
            parts = []
            for s in scales:
                if s is None:
                    parts.append(t3)
                elif isinstance(s, torch.Tensor):
                    parts.append(t3 / s.to(device=t3.device, dtype=t3.dtype))
                else:
                    a = np.asarray(s, np.float64)
                    parts.append(t3 / (float(a) if a.ndim == 0 else torch.as_tensor(a, dtype=t3.dtype, device=t3.device)))
            self._groups[key] = torch.stack(parts).contiguous()
        return self._groups[key]


def as_input(x):
    return x if isinstance(x, Input) else Input(x)


def num_elements(x):
    """``mlkernels.num_elements`` (+ the tuple / FDD extensions of ``stheno/mo/infer.py:16-19``,
    ``stheno/model/fdd.py:120-122``)."""
    from .model.fdd import FDD

    if isinstance(x, FDD):
        return num_elements(x.x)
    if isinstance(x, tuple):
        return sum(num_elements(xi) for xi in x)
    if isinstance(x, Input):
        return x.n
    x = np.asarray(x) if not isinstance(x, torch.Tensor) else x
    if x.ndim == 0:
        return 1
    return x.shape[0] if x.ndim == 1 else x.shape[-2]


def _is_multi(x):
    from .model.fdd import FDD

    return isinstance(x, (tuple, FDD))


# ------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------
def _scale_key(s):
    if s is None:
        return None
    if isinstance(s, torch.Tensor):
        return ("t", id(s))
    a = np.asarray(s, dtype=np.float64)
    return ("v", a.shape, a.tobytes())


def _mul_scale(a, b):
    if a is None:
        return b
    if b is None:
        return a
    if not isinstance(a, torch.Tensor) and not isinstance(b, torch.Tensor):
        return np.asarray(a, np.float64) * np.asarray(b, np.float64)
    return _scale_tensor(a) * _scale_tensor(b)


def _scale_tensor(s):
    return s if isinstance(s, torch.Tensor) else torch.as_tensor(np.asarray(s, np.float64))


class Kernel:
    """Base class.  ``k(x, y)`` returns a structured matrix, ``k.elwise(x, y)`` a column."""

    # -- public API -------------------------------------------------------------------------------------------
    def __call__(self, x, y=None):
        return pairwise(self, x, y)

    def elwise(self, x, y=None):
        return elwise(self, x, y)

    def stretch(self, *stretches):
        """``k.stretch(l)``: inputs divided by ``l`` (scalar or per-dimension vector).  Two arguments stretch the
        two inputs separately (``k.stretch(l, 1)`` in ``stheno/model/measure.py:305``)."""
        if len(stretches) == 1:
            return _simplify_stretch(self, stretches[0], stretches[0])
        return _simplify_stretch(self, stretches[0], stretches[1])

    def shift(self, *shifts):
        """``k.shift(c)``: ``k(x - c, y - c)``; ``k.shift(c1, c2)`` shifts the inputs separately (``measure.py:286``)."""
        return _map_kernel(self, "shift", shifts)

    def select(self, *dims):
        """``k.select(dims)``: ``k(x[:, dims], y[:, dims])``; ``k.select(dims1, dims2)`` per input, ``None`` = all
        (``measure.py:324``).  ``dims``: a tuple / list of column indices."""
        dims = tuple(None if d is None else tuple(np.atleast_1d(d).tolist()) for d in dims)
        return _map_kernel(self, "select", dims)

    def periodic(self, period=1.0):
        """``k.periodic(p)``: ``k(u(x), u(y))`` with ``u(x) = [sin(2 pi x / p), cos(2 pi x / p)]`` (mlkernels
        ``PeriodicKernel``; ``README.md`` decomposition example).  An input map like the others: the inner kernel is unchanged."""
        m = InputMap("periodic", period)
        return self if isinstance(self, ZeroKernel) else MappedKernel(self, m, m)

    def transform(self, *fs):
        """``k.transform(f)``: ``k(f(x), f(y))``; ``k.transform(f1, f2)`` per input, ``None`` = identity (``measure.py:343``).
        ``f`` receives the points as a device tensor ``[..., n, d]`` and returns a tensor (or anything array-like)."""
        return _map_kernel(self, "transform", fs)

    def diff(self, *dims):
        """``k.diff(dim)``: ``d^2 k / dx_dim dy_dim``; ``k.diff(d1, d2)`` differentiates the arguments separately, ``None`` =
        not at all (the cross-kernels of ``stheno/model/measure.py:343-360``; mlkernels ``DerivativeKernel``)."""
        d1, d2 = (dims[0], dims[0]) if len(dims) == 1 else dims
        if isinstance(self, ZeroKernel) or (d1 is None and d2 is None):
            return self
        return DerivativeKernel(self, d1, d2)

    def __add__(self, other):
        other = _as_kernel(other)
        if isinstance(other, ZeroKernel):
            return self
        if isinstance(self, ZeroKernel):
            return other
        return SumKernel(self, other)

    def __radd__(self, other):
        return _as_kernel(other) + self

    def __mul__(self, other):
        if isinstance(other, Kernel):
            if isinstance(self, ZeroKernel) or isinstance(other, ZeroKernel):
                return ZeroKernel()
            if isinstance(other, OneKernel):
                return self
            if isinstance(self, OneKernel):
                return other
            return ProductKernel(self, other)
        if isinstance(other, FunctionType):
            # ``f * k``: ``f(x) k(x, y) f(y)`` (mlkernels ``TensorProductKernel(f) * k``, ``stheno/model/measure.py:249``)
            return self if isinstance(self, ZeroKernel) else FunctionScaledKernel(self, other, other)
        if isinstance(self, ZeroKernel):
            return self
        if not isinstance(other, torch.Tensor) and float(other) == 0.0:
            return ZeroKernel()
        if not isinstance(other, torch.Tensor) and float(other) == 1.0:
            return self
        if isinstance(self, ScaledKernel):
            return ScaledKernel(self.k, self.scale * other)
        return ScaledKernel(self, other)

    __rmul__ = __mul__

    def __neg__(self):
        return self * -1.0

    def __sub__(self, other):
        return self + (-_as_kernel(other))

    def __reversed__(self):
        return self.reversed()

    def reversed(self):
        return self if self.symmetric else ReversedKernel(self)

    symmetric = True  # k(x, y) == k(y, x)^T  (all elementary kernels and their sums/products/stretches)

    # -- internals --------------------------------------------------------------------------------------------
    def flat_terms(self):
        """Sum-of-products form ``[(coef, [(kind, scale), ...]), ...]`` or None if the kernel is not an elementwise
        expression of elementary kernels."""
        return None

    def _flat(self):
        terms = self.flat_terms()
        if terms is None:
            return None, None
        scales, keys = [], {}
        out, raw, praw = [], [], []
        for coef, fs in terms:
            nf = []
            for fac in fs:  # (kind, scale) or (kind, scale, shape parameter)
                kind, s = fac[0], fac[1]
                k = _scale_key(s)
                if k not in keys:
                    keys[k] = len(scales)
                    scales.append(s)
                nf.append((kind, keys[k]) + tuple(_value(v) for v in fac[2:3]))
                praw.append(fac[2] if len(fac) > 2 else None)
            out.append((_value(coef), nf))
            raw.append(coef)
        if not scales:
            scales = [None]
        try:
            flat = ops.FlatKernel(out, len(scales))
        except _GpkError:
            # more product terms / factors / length scales than one K1 descriptor holds: not flattenable as a whole; the
            # callers fall back to evaluating the children separately (each child gets its own descriptor) and combining
            return None, None
        # hyper-parameters given as torch tensors that require grad: remember them for the differentiable path (coef_raw
        # per term, param_raw per factor: the shape parameters, RQ's alpha)
        flat.coef_raw = raw if any(_requires_grad(c) for c in raw) else None
        flat.param_raw = praw if any(_requires_grad(v) for v in praw) else None
        return flat, scales

    def _flattenable(self):
        """True when the whole expression fits ONE K1 descriptor (``ops.FlatKernel`` limits)."""
        return self._flat()[0] is not None

    def _pairwise_dev(self, x, y, same):
        """Device tensor ``[..., n, m]`` for numeric inputs ``x, y`` (:class:`Input`)."""
        flat, scales = self._flat()
        if flat is None:
            raise NotImplementedError(f"pairwise not implemented for {type(self).__name__}")
        if not flat.terms:
            return torch.zeros(x.batch_shape + (x.n, y.n), dtype=x.t.dtype, device=x.t.device)
        xg = x.scaled(scales)
        yg = xg if same else y.scaled(scales)
        if _grad_tensors(flat, xg, yg):
            from .autograd import kernel_cross_grad, kernel_matrix_grad

            K = kernel_matrix_grad(flat, xg) if same else kernel_cross_grad(flat, xg, yg)
        else:
            K = ops.kernel_matrix(flat, xg, None if same else yg, same=same)
        return K.reshape(x.batch_shape + (x.n, y.n))

    def _elwise_dev(self, x, y, same):
        flat, scales = self._flat()
        if flat is None:
            raise NotImplementedError(f"elwise not implemented for {type(self).__name__}")
        if not flat.terms:
            return torch.zeros(x.batch_shape + (x.n, 1), dtype=x.t.dtype, device=x.t.device)
        xg = x.scaled(scales)
        yg = xg if same else y.scaled(scales)
        if _grad_tensors(flat, xg, yg):
            from .autograd import kernel_diag_grad, no_gradient

            if same:
                k = kernel_diag_grad(flat, xg)
            else:
                k = no_gradient("k.elwise(x, y) with x is not y", ops.kernel_diag(flat, xg, yg, same=False),
                                _grad_tensors(self, x, y))
        else:
            k = ops.kernel_diag(flat, xg, None if same else yg, same=same)
        return k.reshape(x.batch_shape + (x.n, 1))

    def _matrix(self, x, y, same):
        """Structured result of ``k(x, y)`` for numeric inputs: symbolic :class:`KernelDense` when square & same."""
        flat, scales = self._flat()
        if flat is not None and same and flat.terms:
            return M.KernelDense(flat, x.scaled(scales), x.batch_shape, origin=x.origin)
        return M.Dense(self._pairwise_dev(x, y, same), x.origin)

    def __str__(self):
        return self.render()

    __repr__ = __str__

    def render(self):
        return type(self).__name__ + "()"

    def display(self, formatter=lambda v: v):
        return self.render()

    @property
    def stationary(self):
        return False


def _value(v):
    """A hyper-parameter as a float for the K1 descriptor (a tensor is detached first: no graph, no warning)."""
    return float(v.detach()) if isinstance(v, torch.Tensor) else float(v)


def _requires_grad(v):
    return isinstance(v, torch.Tensor) and v.requires_grad


def _as_kernel(k):
    if isinstance(k, Kernel):
        return k
    if isinstance(k, (int, float)) and k == 0:
        return ZeroKernel()
    return k * OneKernel()


class _Elementary(Kernel):
    kind = None

    def flat_terms(self):
        return [(1.0, [(self.kind, None)])]

    @property
    def stationary(self):
        return self.kind not in ("linear",)


class EQ(_Elementary):
    """Exponentiated quadratic ``exp(-r^2 / 2)`` (literal form at ``tests/model/test_model.py:345``)."""

    kind = "eq"


class Matern12(_Elementary):
    kind = "matern12"


Exp = Matern12


class Matern32(_Elementary):
    kind = "matern32"


class Matern52(_Elementary):
    kind = "matern52"


class RQ(_Elementary):
    """Rational quadratic ``(1 + r^2 / (2 alpha))^-alpha`` (mlkernels ``RQ(alpha)``; ``README.md:1076-1088``).  ``alpha``: a
    number, a NumPy scalar or a one-element torch tensor; a tensor that requires grad receives its gradient on every route
    with an analytic backward."""

    kind = "rq"

    def __init__(self, alpha):
        if isinstance(alpha, torch.Tensor):
            if alpha.numel() != 1:
                raise ValueError(f"RQ takes one alpha, not a tensor of shape {tuple(alpha.shape)}")
            self.alpha = alpha if alpha.dim() == 0 else alpha.reshape(())
        else:
            a = np.asarray(alpha, np.float64)
            if a.size != 1:
                raise ValueError(f"RQ takes one alpha, not an array of shape {a.shape}")
            self.alpha = float(a.reshape(()))
        if not _value(self.alpha) > 0:
            raise ValueError("RQ needs alpha > 0")

    def flat_terms(self):
        return [(1.0, [("rq", None, self.alpha)])]

    def render(self):
        return f"RQ({_fmt(self.alpha)})"


class Linear(_Elementary):
    """``<x, y>``.  ``Linear()(x)`` stays a :class:`matrix.LowRank` (``x x^T``), so ``GP(Linear())(x, noise)`` is a
    Woodbury matrix and ``logpdf`` costs ``O(n d^2)`` (SURVEY.md 8f rank 2)."""

    kind = "linear"

    def _matrix(self, x, y, same):
        if same:
            return M.LowRank(x.t, x.origin)
        return M.Dense(self._pairwise_dev(x, y, same), x.origin)


class Delta(_Elementary):
    """Kronecker delta: identity when both arguments are the same object, else ``r^2 < 1e-10``."""

    kind = "delta"

    def _matrix(self, x, y, same):
        if same:
            ones = torch.ones(x.batch_shape + (x.n,), dtype=x.t.dtype, device=x.t.device)
            return M.Diagonal(ones, x.origin, scalar=1.0)
        return M.Dense(self._pairwise_dev(x, y, same), x.origin)


class OneKernel(_Elementary):
    kind = "one"

    def render(self):
        return "1"


class ZeroKernel(Kernel):
    def flat_terms(self):
        return []

    def _matrix(self, x, y, same):
        return M.Zero(x.t.dtype, x.n, y.n, x.t.device, x.batch_shape, x.origin)

    def render(self):
        return "0"

    @property
    def stationary(self):
        return True


class ScaledKernel(Kernel):
    def __init__(self, k, scale):
        self.k, self.scale = k, scale

    @property
    def symmetric(self):
        return self.k.symmetric

    def flat_terms(self):
        t = self.k.flat_terms()
        if t is None:
            return None
        s = self.scale if isinstance(self.scale, torch.Tensor) else float(self.scale)
        return [(c * s, fs) for c, fs in t]

    def _pairwise_dev(self, x, y, same):
        if self._flattenable():
            return super()._pairwise_dev(x, y, same)
        return self.scale * M.dense(pairwise(self.k, x, y if not same else None))

    def _elwise_dev(self, x, y, same):
        if self._flattenable():
            return super()._elwise_dev(x, y, same)
        return self.scale * elwise_dev(self.k, x, y, same)

    def _matrix(self, x, y, same):
        if not self._flattenable():
            return M.Dense(self._pairwise_dev(x, y, same), x.origin)
        inner = self.k
        # a scale that carries a graph must not be detached by the structured shortcuts (ADVICE r1): keep it as a tensor
        st = self.scale if (isinstance(self.scale, torch.Tensor) and self.scale.requires_grad and torch.is_grad_enabled()) else None
        sv = float(self.scale.detach()) if isinstance(self.scale, torch.Tensor) else float(self.scale)
        if same and isinstance(inner, Linear) and sv > 0:
            if st is not None:
                return M.LowRank(x.t * st.to(device=x.t.device, dtype=x.t.dtype).sqrt(), x.origin)
            return M.LowRank(x.t * sv ** 0.5, x.origin)
        if same and isinstance(inner, Delta):
            if st is not None:
                d = st.to(device=x.t.device, dtype=x.t.dtype).expand(x.batch_shape + (x.n,))
                return M.Diagonal(d, x.origin, scalar=sv, scalar_t=st)
            return M.fill_diag(sv, x.n, x.t.dtype, x.t.device, x.origin) if not x.batch_shape else M.Diagonal(
                torch.full(x.batch_shape + (x.n,), sv, dtype=x.t.dtype, device=x.t.device), x.origin, scalar=sv)
        return super()._matrix(x, y, same)

    def render(self):
        return f"{_fmt(self.scale)} * {_paren(self.k)}"

    @property
    def stationary(self):
        return self.k.stationary


class _Join(Kernel):
    def __init__(self, a, b):
        self.a, self.b = a, b

    @property
    def symmetric(self):
        return self.a.symmetric and self.b.symmetric

    @property
    def stationary(self):
        return self.a.stationary and self.b.stationary


class SumKernel(_Join):
    def flat_terms(self):
        ta, tb = self.a.flat_terms(), self.b.flat_terms()
        if ta is None or tb is None:
            return None
        return ta + tb

    def _pairwise_dev(self, x, y, same):
        if self._flattenable():
            return super()._pairwise_dev(x, y, same)
        yy = None if same else y
        return M.dense(M.add(pairwise(self.a, x, yy), pairwise(self.b, x, yy)))

    def _elwise_dev(self, x, y, same):
        if self._flattenable():
            return super()._elwise_dev(x, y, same)
        return elwise_dev(self.a, x, y, same) + elwise_dev(self.b, x, y, same)

    def _matrix(self, x, y, same):
        if self._flattenable():
            # keep Delta parts diagonal: k + s2 * Delta  ->  KernelDense + Diagonal (stays symbolic)
            if same and isinstance(_strip_scale(self.b)[0], Delta):
                return M.add(self.a._matrix(x, y, same), self.b._matrix(x, y, same))
            return super()._matrix(x, y, same)
        yy = None if same else y
        return M.add(pairwise(self.a, x, yy), pairwise(self.b, x, yy))

    def render(self):
        return f"{self.a.render()} + {self.b.render()}"


class ProductKernel(_Join):
    def flat_terms(self):
        ta, tb = self.a.flat_terms(), self.b.flat_terms()
        if ta is None or tb is None:
            return None
        return [(ca * cb, fa + fb) for (ca, fa), (cb, fb) in itertools.product(ta, tb)]

    def _pairwise_dev(self, x, y, same):
        if self._flattenable():
            return super()._pairwise_dev(x, y, same)
        yy = None if same else y
        return M.dense(pairwise(self.a, x, yy)) * M.dense(pairwise(self.b, x, yy))

    def _elwise_dev(self, x, y, same):
        if self._flattenable():
            return super()._elwise_dev(x, y, same)
        return elwise_dev(self.a, x, y, same) * elwise_dev(self.b, x, y, same)

    def render(self):
        return f"{_paren(self.a)} * {_paren(self.b)}"


class StretchedKernel(Kernel):
    """``k.stretch(l)``: ``k(x / l, y / l)``.  Flattened by composing length scales multiplicatively."""

    def __init__(self, k, stretch):
        self.k, self.stretch_ = k, stretch

    @property
    def symmetric(self):
        return self.k.symmetric

    def flat_terms(self):
        t = self.k.flat_terms()
        if t is None:
            return None
        return [(c, [(f[0], _mul_scale(f[1], self.stretch_)) + tuple(f[2:3]) for f in fs]) for c, fs in t]

    def _scaled_inputs(self, x, y, same):
        s = self.stretch_
        xs = Input.__new__(Input)
        xs.origin, xs._groups = x.origin, {}
        sv = s if isinstance(s, torch.Tensor) else torch.as_tensor(np.asarray(s, np.float64), dtype=x.t.dtype,
                                                                   device=x.t.device)
        xs.t = x.t / sv
        if same:
            return xs, xs
        ys = Input.__new__(Input)
        ys.origin, ys._groups = y.origin, {}
        ys.t = y.t / sv
        return xs, ys

    def _pairwise_dev(self, x, y, same):
        if self._flattenable():
            return super()._pairwise_dev(x, y, same)
        xs, ys = self._scaled_inputs(x, y, same)
        return self.k._pairwise_dev(xs, ys, same)

    def _elwise_dev(self, x, y, same):
        if self._flattenable():
            return super()._elwise_dev(x, y, same)
        xs, ys = self._scaled_inputs(x, y, same)
        return self.k._elwise_dev(xs, ys, same)

    def render(self):
        return f"{_paren(self.k)} > {_fmt(self.stretch_)}"

    @property
    def stationary(self):
        return self.k.stationary


class ReversedKernel(Kernel):
    """``reversed(k)(x, y) = k(y, x)^T`` (``stheno/model/measure.py:112-114``)."""

    def __init__(self, k):
        self.k = k

    symmetric = False

    def reversed(self):
        return self.k

    def _pairwise_dev(self, x, y, same):
        return self.k._pairwise_dev(y, x, same).transpose(-1, -2)

    def _elwise_dev(self, x, y, same):
        return self.k._elwise_dev(y, x, same)

    def render(self):
        return f"Reversed({self.k.render()})"


# ------------------------------------------------------------------------------------------------------------
# input maps: shift / select / transform / per-argument stretch  (``GP.shift/select/transform``,
# ``stheno/model/measure.py:272-345``; mlkernels ShiftedKernel / SelectedKernel / InputTransformedKernel)
# ------------------------------------------------------------------------------------------------------------
class InputMap:
    """A transformation of the input points applied on the device before the kernel / mean is evaluated:
    ``shift``: ``x - c``; ``stretch``: ``x / l``; ``select``: ``x[:, dims]``; ``transform``: ``f(x)``."""

    def __init__(self, kind, param):
        self.kind, self.param = kind, param

    def __call__(self, x):
        t = x.t
        p = self.param
        if self.kind == "shift":
            v = p if isinstance(p, torch.Tensor) else torch.as_tensor(np.asarray(p, np.float64), dtype=t.dtype, device=t.device)
            out = t - v.to(device=t.device, dtype=t.dtype)
        elif self.kind == "stretch":
            v = p if isinstance(p, torch.Tensor) else torch.as_tensor(np.asarray(p, np.float64), dtype=t.dtype, device=t.device)
            out = t / v.to(device=t.device, dtype=t.dtype)
        elif self.kind == "select":
            out = t[..., list(p)]
        elif self.kind == "periodic":
            v = p if isinstance(p, torch.Tensor) else torch.as_tensor(np.asarray(p, np.float64), dtype=t.dtype, device=t.device)
            ang = t * (2 * np.pi) / v.to(device=t.device, dtype=t.dtype)
            out = torch.cat([torch.sin(ang), torch.cos(ang)], dim=-1)
        else:
            out = p(t)
            if not isinstance(out, torch.Tensor):
                out = to_dev(out, t.dtype)
            out = uprank(out.to(t.dtype))
        y = Input.__new__(Input)
        y.origin, y._groups, y.src = x.origin, {}, None
        y.t = out.contiguous()
        return y

    def same_as(self, other):
        if other is None or self.kind != other.kind:
            return False
        a, b = self.param, other.param
        if a is b:
            return True
        if self.kind == "transform" or isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
            return False
        return np.array_equal(np.asarray(a, dtype=object), np.asarray(b, dtype=object))

    def render(self):
        sym = {"shift": "shift", "stretch": ">", "select": ":", "transform": "transform", "periodic": "per"}[self.kind]
        if self.kind == "transform":
            return f"{sym} {getattr(self.param, '__name__', 'f')}"
        if self.kind == "select":
            return f"{sym} {list(self.param)}"
        return f"{sym} {_fmt(self.param)}"


def _same_map(a, b):
    return (a is None and b is None) or (a is not None and a.same_as(b))


class MappedKernel(Kernel):
    """``k(m1(x), m2(y))`` for input maps ``m1``, ``m2`` (``None`` = identity).  With equal maps on the same points the inner
    kernel keeps its fused path (symbolic :class:`KernelDense`: K1 writes straight into the Cholesky workspace)."""

    def __init__(self, k, m1, m2):
        self.k, self.m1, self.m2 = k, m1, m2

    @property
    def symmetric(self):
        return self.k.symmetric and _same_map(self.m1, self.m2)

    def reversed(self):
        return self if self.symmetric else MappedKernel(self.k.reversed(), self.m2, self.m1)

    def _mapped(self, x, y, same):
        xs = x if self.m1 is None else self.m1(x)
        if same and _same_map(self.m1, self.m2):
            return xs, xs, True
        ys = y if self.m2 is None else self.m2(y)
        return xs, ys, False

    def _pairwise_dev(self, x, y, same):
        return self.k._pairwise_dev(*self._mapped(x, y, same))

    def _elwise_dev(self, x, y, same):
        return self.k._elwise_dev(*self._mapped(x, y, same))

    def _matrix(self, x, y, same):
        xs, ys, still_same = self._mapped(x, y, same)
        if still_same:
            return self.k._matrix(xs, xs, True)
        return M.Dense(self.k._pairwise_dev(xs, ys, False), x.origin)

    def render(self):
        if _same_map(self.m1, self.m2):
            return f"{_paren(self.k)} {self.m1.render()}"
        r = lambda m: "id" if m is None else m.render()
        return f"{_paren(self.k)} ({r(self.m1)}, {r(self.m2)})"

    @property
    def stationary(self):
        return (self.k.stationary and _same_map(self.m1, self.m2) and self.m1 is not None
                and self.m1.kind in ("shift", "stretch", "periodic"))


def _map_kernel(k, kind, params):
    """``k.shift(c)`` / ``k.shift(c1, c2)`` etc.: one parameter maps both arguments, two map them separately and ``None`` (or, for
    stretches, 1 / for shifts, 0) leaves an argument untouched."""
    if isinstance(k, ZeroKernel):
        return k
    if len(params) == 1:
        m = InputMap(kind, params[0])
        return MappedKernel(k, m, m)
    if len(params) != 2:
        raise ValueError(f"{kind}: one parameter (both inputs) or two (one per input) expected")

    def one(p):
        if p is None:
            return None
        if kind == "shift" and np.isscalar(p) and p == 0:
            return None
        if kind == "stretch" and np.isscalar(p) and p == 1:
            return None
        return InputMap(kind, p)

    m1, m2 = one(params[0]), one(params[1])
    if m1 is None and m2 is None:
        return k
    return MappedKernel(k, m1, m2)


def k1_block(k, x, y=None, *, through_maps=False, zero=False):
    """``k(x, y)`` as one K1 descriptor: ``(flat, scales, xm, ym)`` with ``flat, scales`` the :meth:`Kernel._flat` of the
    kernel and ``xm``, ``ym`` the :class:`Input` s it reads (not yet stretched by ``scales``: :meth:`Input.scaled`).  ``y=None``:
    the square ``k(x, x)`` (then ``ym is xm``).  None for multi-output inputs, for a kernel that does not flatten to one
    descriptor (sums or products of differently mapped kernels, derivatives, ...) and, unless ``zero``, for one without
    terms (a zero block).

    ``through_maps``: a chain of :class:`MappedKernel` s (``shift``, ``stretch``, ``select``, ``periodic``, ``transform``,
    nested in any order) around a flat kernel resolves to that kernel at the points the chain makes of ``x`` and ``y``, with
    their torch graph to the raw points and to the maps' parameters: only the analytic gradient routes differentiate through
    the maps.  A square block needs equal maps at every link; a cross block maps each argument by its own."""
    if _is_multi(x) or (y is not None and _is_multi(y)):
        return None
    maps = []
    while through_maps and isinstance(k, MappedKernel):
        if y is None and not _same_map(k.m1, k.m2):
            return None
        maps.append((k.m1, k.m2))
        k = k.k
    flat, scales = k._flat()
    if flat is None or not (flat.terms or zero):
        return None
    xm = as_input(x)
    ym = xm if y is None else as_input(y)
    for m1, m2 in maps:  # outermost first: MappedKernel(k, m1, m2)(x, y) = k(m1(x), m2(y))
        if y is None:
            xm = ym = xm if m1 is None else m1(xm)
        else:
            xm, ym = (xm if m1 is None else m1(xm)), (ym if m2 is None else m2(ym))
    return flat, scales, xm, ym


def _children(k):
    return [c for c in (getattr(k, "k", None), getattr(k, "a", None), getattr(k, "b", None)) if isinstance(c, Kernel)]


def _maps(k):
    """The input maps anywhere inside the kernel expression ``k``."""
    out = [m for m in ((k.m1, k.m2) if isinstance(k, MappedKernel) else ()) if m is not None]
    for c in _children(k):
        out += _maps(c)
    return out


def map_output_grads(k, x, y):
    """The points that ``k``'s ``transform`` maps produce from the arguments of ``k(x, y)`` and that require grad.  A transform's
    parameters (a network's weights) hide in its closure, so only its output shows that the kernel depends on them: the maps
    are evaluated here (O(n d)).  Empty when grad mode is off or ``k`` has no transform; the other maps' parameters are
    tensors :func:`_grad_tensors` finds."""
    if not torch.is_grad_enabled() or not any(m.kind == "transform" for m in _maps(k)):
        return []
    out = []

    def walk(k, x, y):
        if isinstance(k, MappedKernel):
            x, y = (x if k.m1 is None else k.m1(x)), (y if k.m2 is None else k.m2(y))
            out.extend(t for t in (x.t, y.t) if t.requires_grad)
        elif isinstance(k, ReversedKernel):
            x, y = y, x
        for c in _children(k):
            if _maps(c):
                walk(c, x, y)

    walk(k, as_input(x), as_input(y))
    return out


class DerivativeKernel(Kernel):
    """``d^a/dx_{d1} d^b/dy_{d2} k(x, y)`` (``a, b`` in {0, 1}; mlkernels ``DerivativeKernel`` behind ``GP.diff``,
    ``stheno/model/measure.py:343-360``).  Evaluated by forward-mode differentiation (``torch.func.jvp``, nested for the mixed
    second derivative) of the differentiable restatement of the flattened inner kernel (``generic_grad.kernel_torch``):
    ``K[i, j]`` depends on ``x`` only through row ``i``, so ONE tangent with ``e_{d1}`` in every row gives every
    ``dK[i, j] / dx_i[d1]`` at once.  SURVEY 8f rank 3 (off the benchmarked path; the result is an ordinary dense matrix that
    the hand-written factorisation / solves then consume)."""

    def __init__(self, k, d1, d2):
        self.k, self.d1, self.d2 = k, d1, d2

    @property
    def symmetric(self):
        return self.k.symmetric and self.d1 == self.d2

    def reversed(self):
        return self if self.symmetric else DerivativeKernel(self.k.reversed(), self.d2, self.d1)

    def _deriv(self, fn, xt, yt):
        from torch.func import jvp

        def tangent(t, d):
            e = torch.zeros_like(t)
            e[..., d] = 1.0
            return e

        if self.d1 is not None and self.d2 is not None:
            def inner(yv):
                return jvp(lambda xv: fn(xv, yv), (xt,), (tangent(xt, self.d1),))[1]

            return jvp(inner, (yt,), (tangent(yt, self.d2),))[1]
        if self.d1 is not None:
            return jvp(lambda xv: fn(xv, yt), (xt,), (tangent(xt, self.d1),))[1]
        return jvp(lambda yv: fn(xt, yv), (yt,), (tangent(yt, self.d2),))[1]

    def _pairwise_dev(self, x, y, same):
        from .generic_grad import kernel_torch

        with torch.enable_grad():
            out = self._deriv(lambda a, b: kernel_torch(self.k, a, b), x.t.detach(), (x if same else y).t.detach().clone())
        return out.detach()

    def _elwise_dev(self, x, y, same):
        from .generic_grad import kernel_torch

        def fn(a, b):  # elementwise: pair i with i
            return kernel_torch(self.k, a.unsqueeze(-2), b.unsqueeze(-2))[..., 0, 0]

        with torch.enable_grad():
            out = self._deriv(fn, x.t.detach(), (x if same else y).t.detach().clone())
        return out.detach().unsqueeze(-1)

    def _matrix(self, x, y, same):
        return M.Dense(self._pairwise_dev(x, y, same), x.origin)

    def render(self):
        if self.d1 == self.d2:
            return f"d({self.d1}) {_paren(self.k)}"
        return f"d({self.d1}, {self.d2}) {_paren(self.k)}"

    @property
    def stationary(self):
        return self.k.stationary


class FunctionScaledKernel(Kernel):
    """``g1(x) k(x, y) g2(y)`` for user functions ``g`` (``None`` = 1): ``f * k`` and the one-sided
    ``TensorProductKernel(f, ones) * k`` of ``GP * function`` (``stheno/model/measure.py:241-251``).  The inner kernel is
    evaluated by K1; the row / column factors are applied to its dense result."""

    def __init__(self, k, g1, g2):
        self.k, self.g1, self.g2 = k, g1, g2

    @property
    def symmetric(self):
        return self.k.symmetric and self.g1 is self.g2

    def reversed(self):
        return self if self.symmetric else FunctionScaledKernel(self.k.reversed(), self.g2, self.g1)

    @staticmethod
    def _factor(g, x):
        return None if g is None else FunctionMean(g)._dev(x)  # [..., n, 1]

    def _pairwise_dev(self, x, y, same):
        K = self.k._pairwise_dev(x, y, same)
        gx, gy = self._factor(self.g1, x), self._factor(self.g2, x if same else y)
        if gx is not None:
            K = K * gx
        if gy is not None:
            K = K * gy.transpose(-1, -2)
        return K

    def _elwise_dev(self, x, y, same):
        k = self.k._elwise_dev(x, y, same)
        gx, gy = self._factor(self.g1, x), self._factor(self.g2, x if same else y)
        if gx is not None:
            k = k * gx
        if gy is not None:
            k = k * gy
        return k

    def _matrix(self, x, y, same):
        return M.Dense(self._pairwise_dev(x, y, same), x.origin)

    def render(self):
        n = lambda g: "1" if g is None else getattr(g, "__name__", "f")
        if self.g1 is self.g2:
            return f"{n(self.g1)} * {_paren(self.k)}"
        return f"({n(self.g1)} x {n(self.g2)}) * {_paren(self.k)}"

    @property
    def stationary(self):
        return False


def _strip_scale(k):
    c = 1.0
    while isinstance(k, ScaledKernel):
        c = c * k.scale
        k = k.k
    return k, c


def _simplify_stretch(k, s1, s2):
    if isinstance(k, (ZeroKernel, OneKernel)):
        return k
    if s1 is not s2 and not (np.isscalar(s1) and np.isscalar(s2) and s1 == s2):
        return _map_kernel(k, "stretch", (s1, s2))  # per-argument stretch (cross-kernels of a stretched GP, measure.py:305)
    return StretchedKernel(k, s1)


def _fmt(v):
    if isinstance(v, torch.Tensor):
        v = v.detach().cpu().numpy()
    a = np.asarray(v)
    return f"{float(a):g}" if a.ndim == 0 else np.array2string(a, precision=3)


def _paren(k):
    return f"({k.render()})" if isinstance(k, (SumKernel,)) else k.render()


# ------------------------------------------------------------------------------------------------------------
# pairwise / elwise entry points with the multi-output (tuple / FDD) input rules of ``stheno/mo/input.py:7-36``
# ------------------------------------------------------------------------------------------------------------
def pairwise(k, x, y=None):
    """``k(x, y)`` -> structured matrix.  ``y=None`` (or ``y is x``) means the same object."""
    from .mo.kernel import mo_pairwise

    same = y is None or y is x
    if hasattr(k, "_pairwise_multi") or _is_multi(x) or (not same and _is_multi(y)):
        return mo_pairwise(k, x, x if same else y, same)
    xi = as_input(x)
    yi = xi if same else as_input(y)
    if not same and getattr(xi, "src", None) is not None and getattr(yi, "src", None) is xi.src:
        same, yi = True, xi  # two wrappers of the caller's same array (e.g. f1(x), f2(x)): the same points
    return k._matrix(xi, yi, same)


def elwise_dev(k, x, y, same):
    return _elwise_any(k, x, None if same else y, same)


def elwise(k, x, y=None):
    """``k.elwise(x, y)`` -> column ``(n, 1)`` in the caller's array type."""
    same = y is None or y is x
    return from_dev(_elwise_any(k, x, None if same else y, same), _origin_of_input(x))


# ------------------------------------------------------------------------------------------------------------
# posterior objects (mlkernels.PosteriorKernel / SubspaceKernel / PosteriorMean)
# ------------------------------------------------------------------------------------------------------------
def _cross_rows(k_zi, z, x, ch):
    """``k_zi(z, x)^T`` as a zero-padded ``[B, m_pad, n_pad]`` row buffer (rows = points of ``x``)."""
    blk = k1_block(k_zi, z, x)
    if blk is not None:
        flat, scales, zi, xi = blk
        return ops.kernel_rows_padded(flat, xi.scaled(scales), zi.scaled(scales), ch), xi.n
    Kzx = M.dense(pairwise(k_zi, z, x))  # [..., n, m]
    K3, _ = batch_flatten(Kzx, 2)
    buf = ch.new_rows(K3.shape[2])
    ops.transpose(K3, K3.shape[1], K3.shape[2], out=buf)
    return buf, K3.shape[2]


def _grad_tensors(*objs):
    """The tensors that require grad reachable from the kernels, K1 descriptors, means, inputs, matrices and tensors ``objs``
    (empty when grad mode is off): what a result depends on through raw-pointer kernels.  Every choice between the raw route
    and a differentiable one asks this."""
    from .model.fdd import FDD

    out, seen = [], set()
    if not torch.is_grad_enabled():
        return out

    def walk(o):
        if o is None or id(o) in seen:
            return
        seen.add(id(o))
        if isinstance(o, torch.Tensor):
            if o.requires_grad:
                out.append(o)
        elif isinstance(o, (list, tuple)):
            for v in o:
                walk(v)
        elif isinstance(o, Input):
            walk(o.t)
        elif isinstance(o, FDD):
            walk(o.x)
        elif isinstance(o, ops.FlatKernel):
            walk([getattr(o, "coef_raw", None), getattr(o, "param_raw", None)])
        elif isinstance(o, M.KernelDense):
            walk([o.flat, o.xg, o.noise_t, o.noise_vec])
        elif isinstance(o, (Kernel, Mean, InputMap, M.AbstractMatrix)):
            for k, v in vars(o).items():
                if k not in ("_chol", "_b"):
                    walk(v)

    for o in objs:
        walk(o)
    return out


def _prediction_grads(post, x, *others):
    """The tensors that require grad behind a prediction of the exact posterior ``post`` (a :class:`PosteriorKernel` or
    :class:`PosteriorMean`) at ``x``; ``others``: what else the prediction reads.  Empty when grad mode is off."""
    maps = [] if _is_multi(x) or _is_multi(post.z) else map_output_grads(post.k_zi, post.z, x)
    return _grad_tensors(post.K_z, post.k_zi, post.z, x, *others) + maps


def _exact_args(post, x):
    """``(flat, coefs_x, xg_x, ns, nv, coefs_c, xsg, zg, params_x, params_c)``: the cross kernel's descriptor and the tensor
    inputs of :func:`autograd.exact_posterior` for a prediction of ``post`` at ``x``, or None when it has no analytic route.
    Covered: exact observations with a symbolic ``K_z``, a cross kernel that is one K1 descriptor under input maps, and
    single-output inputs of the factor's batch."""
    K_z = post.K_z
    blk = k1_block(post.k_zi, post.z, x, through_maps=True) if isinstance(K_z, M.KernelDense) else None
    if blk is None:
        return None
    flat, scales, zi, xi = blk
    xsg, zg = xi.scaled(scales), zi.scaled(scales)
    if xsg.shape[1] != K_z.xg.shape[1] or zg.shape[1] != K_z.xg.shape[1] or zg.shape[2] != K_z.n:
        return None
    from .autograd import coef_tensor, param_tensor

    return (flat, coef_tensor(K_z.flat, K_z.xg), K_z.xg, K_z.noise, K_z.noise_vec, coef_tensor(flat, xsg), xsg, zg,
            param_tensor(K_z.flat, K_z.xg), param_tensor(flat, xsg))


def _posterior_call(post, x, fwd, what, *others, mean=False, P=None, cross=None):
    """``(dot, sq, cov)`` as ``fwd()`` computes them -- the launches of a prediction of the exact posterior ``post`` at ``x``,
    None for outputs not formed -- on the prediction's gradient route:

    * nothing requires grad (:func:`_prediction_grads`; ``others``: what else the prediction reads): ``fwd()`` as it is;
    * the prediction is covered (:func:`_exact_args`): the analytic backward of ``autograd.exact_posterior``.  ``mean``:
      ``post`` is a :class:`PosteriorMean` whose mean the prediction forms; ``P``: the prior covariance of ``cov``;
    * else: each output attached by ``autograd.no_gradient`` to those tensors, named ``"{what} of a <posterior kind>"``
      (:func:`_route_name`), or ``cross`` when it is given (a cross-covariance) and only the prediction is not covered;
      ``what=None``: None instead, for a caller that falls back to predictions that name themselves."""
    # y - m_z(z) itself: a mean given as a user function hides its parameters in a closure
    ybar = post._ybar() if mean and torch.is_grad_enabled() else None
    ts = _prediction_grads(post, x, *others, *((post.y, ybar) if mean else ()))
    if not ts:
        return fwd()
    from .autograd import PosteriorSpec, exact_posterior, no_gradient

    args = _exact_args(post, x)
    if args is None and what is None:
        return None
    if args is None or cross is not None:
        route = f"{what} of a {_route_name(post)}" if args is None else cross
        return tuple(None if t is None else no_gradient(route, t, ts) for t in fwd())
    flat, coefs_x, xg_x, ns, nv, coefs_c, xsg, zg, params_x, params_c = args
    spec = PosteriorSpec(post.K_z.chol(), post.K_z.flat, flat, post._half_y() if mean else None, fwd)
    return exact_posterior(spec, coefs_x, xg_x, ns, nv, ybar, coefs_c, xsg, zg, P, params_x, params_c)


class PosteriorKernel(Kernel):
    """``k_ij(x, y) - k_zi(z, x)^T K_z^-1 k_zj(z, y)`` (``stheno/model/observations.py:148-154``)."""

    symmetric = False

    def __init__(self, k_ij, k_zi, k_zj, z, K_z):
        self.k_ij, self.k_zi, self.k_zj, self.z, self.K_z = k_ij, k_zi, k_zj, z, M._densify(K_z, full=True)

    def _half(self, k_z, x):
        ch = self.K_z.chol()
        V, m = _cross_rows(k_z, self.z, x, ch)
        ch.solve_rows_(V)
        return V, m

    def _pairwise_any(self, x, y, same):
        prior = M.dense(pairwise(self.k_ij, x, None if same else y))
        _, _, C = _posterior_call(self, x, lambda: (None, None, self._cov(x, y, same, prior)), "the posterior covariance",
                                  self.k_zj, None if same else y, P=prior,
                                  cross=None if self._same_half(same) else
                                  "a posterior cross-covariance between different inputs or processes")
        return M.Dense(C, _origin_of_input(x))

    def _same_half(self, same):
        return same and self.k_zi is self.k_zj

    def _cov(self, x, y, same, prior, V=None, m=None):
        """``prior - V_x V_y^T`` (``V``: the solved rows at ``x`` when already formed); with one half for both sides, from the
        lower triangle of the product, mirrored.  The copy of ``prior`` keeps its graph: when nothing behind ``V`` requires
        grad, the result's gradient is the prior's alone."""
        same_half = self._same_half(same)
        if V is None:
            V, m = self._half(self.k_zi, x)
        Vy, my = (V, m) if same_half else self._half(self.k_zj, x if same else y)
        P3, bs = batch_flatten(prior, 2)
        C = torch.zeros(P3.shape[0], V.shape[1], Vy.shape[1], dtype=P3.dtype, device=P3.device)
        C[:, :m, :my] = P3
        ops.gemm_nt(V, Vy, C, alpha=-1.0, beta=1.0, lower=same_half)
        if same_half:
            ops.symmetrize_(C, m)
        return C[:, :m, :my].reshape(bs + (m, my))

    def _elwise_any(self, x, y, same):
        prior = _elwise_any(self.k_ij, x, y, same)
        same_half = self._same_half(same)
        _, corr, _ = _posterior_call(self, x, lambda: (None, self._sq(x) if same_half else self._corr(x, y, same), None),
                                     "the posterior variance", self.k_zj, None if same else y,
                                     cross=None if same_half else
                                     "the posterior variance of a cross-covariance between different inputs")
        return prior - corr.reshape(prior.shape[:-1]).unsqueeze(-1)

    def _sq(self, x):
        Vx, mx = self._half(self.k_zi, x)
        return ops.row_dot_sq(Vx, mx, Vx.shape[2], None)[1]

    def _corr(self, x, y, same):
        Vx, mx = self._half(self.k_zi, x)
        Vy, _ = self._half(self.k_zj, x if same else y)
        return (Vx[:, :mx] * Vy[:, :mx]).sum(-1)

    def _matrix(self, x, y, same):
        return self._pairwise_any(x, y, same)

    def _pairwise_dev(self, x, y, same):
        return M.dense(self._pairwise_any(x, y, same))

    def _elwise_dev(self, x, y, same):
        return self._elwise_any(x, y, same)

    def render(self):
        return "PosteriorKernel()"


class SubspaceKernel(Kernel):
    """``k_zi(z, x)^T A^-1 k_zj(z, y)`` (``stheno/model/observations.py:261-266``)."""

    symmetric = False

    def __init__(self, k_zi, k_zj, z, A):
        self.k_zi, self.k_zj, self.z, self.A = k_zi, k_zj, z, M._densify(A, full=True)

    def _half(self, k_z, x):
        ch = self.A.chol()
        V, m = _cross_rows(k_z, self.z, x, ch)
        ch.solve_rows_(V)
        return V, m

    def _pairwise_any(self, x, y, same):
        org = _origin_of_input(x)
        same_half = same and (self.k_zi is self.k_zj)

        def fwd():
            Vx, mx = self._half(self.k_zi, x)
            Vy, my = (Vx, mx) if same_half else self._half(self.k_zj, x if same else y)
            C = ops.gemm_nt(Vx, Vy, lower=False)
            return C[:, :mx, :my].reshape(_batch_shape_of_input(x) + (mx, my)), Vx

        route = self._xs_route(x) if same_half else None
        if route is not None:
            from .autograd import subspace_cov

            return M.Dense(subspace_cov(self.A.chol(), *route, fwd), org)
        return M.Dense(self._no_grad(fwd()[0], x, y), org)

    def _xs_route(self, x):
        """``(flat, zg, xsg)`` when the covariance at ``x`` has an analytic gradient in ``x``: only ``x`` requires grad, the
        cross kernel flattens to one descriptor, and ``x``, ``z`` and ``A`` are single-output and unbatched; else None."""
        if _grad_tensors(self.A, self.k_zi, self.z) or not _grad_tensors(x):
            return None
        blk = k1_block(self.k_zi, self.z, x)
        if blk is None or blk[2].batch_shape or blk[3].batch_shape or self.A.chol().batch != 1:
            return None
        flat, scales, zi, xi = blk
        return flat, zi.scaled(scales), xi.scaled(scales)

    def _elwise_any(self, x, y, same):
        Vx, mx = self._half(self.k_zi, x)
        same_half = same and (self.k_zi is self.k_zj)
        Vy = Vx if same_half else self._half(self.k_zj, x if same else y)[0]
        out = (Vx[:, :mx] * Vy[:, :mx]).sum(-1)
        return self._no_grad(out.reshape(_batch_shape_of_input(x) + (mx, 1)), x, y)

    def _no_grad(self, value, x, y):
        ts = _grad_tensors(self.A, self.k_zi, self.k_zj, self.z, x, y)
        if not ts:
            return value
        from .autograd import no_gradient

        return no_gradient("a sparse (pseudo-observation) posterior", value, ts)

    def _matrix(self, x, y, same):
        return self._pairwise_any(x, y, same)

    def _pairwise_dev(self, x, y, same):
        return M.dense(self._pairwise_any(x, y, same))

    def _elwise_dev(self, x, y, same):
        return self._elwise_any(x, y, same)

    def render(self):
        return "SubspaceKernel()"


def _origin_of_input(x):
    from .model.fdd import FDD

    if isinstance(x, Input):
        return x.origin
    if isinstance(x, FDD):
        return _origin_of_input(x.x)
    if isinstance(x, tuple):
        return _origin_of_input(x[0])
    return origin_of(x)


def _batch_shape_of_input(x):
    from .model.fdd import FDD

    if isinstance(x, FDD):
        return _batch_shape_of_input(x.x)
    if isinstance(x, tuple):
        return _batch_shape_of_input(x[0])
    return as_input(x).batch_shape


def _elwise_any(k, x, y, same):
    """Device column ``[..., n, 1]`` of ``k.elwise(x, y)`` for any input kind."""
    from .mo.kernel import mo_elwise_dev

    if hasattr(k, "_elwise_multi") or _is_multi(x) or (not same and _is_multi(y)):
        return mo_elwise_dev(k, x, x if same else y, same)
    xi = as_input(x)
    return k._elwise_dev(xi, xi if same else as_input(y), same)


# ------------------------------------------------------------------------------------------------------------
# means
# ------------------------------------------------------------------------------------------------------------
class Mean:
    def __call__(self, x):
        return from_dev(self.dev(x), _origin_of_input(x))

    def dev(self, x):
        """Device column ``[..., n, 1]`` for any input kind (numeric, FDD, tuple)."""
        from .model.fdd import FDD

        if isinstance(x, tuple):
            return torch.cat([self.dev(xi) for xi in x], dim=-2)
        if isinstance(x, FDD):
            raise ValueError(f"{type(self).__name__} cannot be evaluated at an FDD")
        return self._dev(as_input(x))

    def _dev(self, x):
        raise NotImplementedError

    is_zero = False

    def __add__(self, other):
        other = _as_mean(other)
        if other.is_zero:
            return self
        if self.is_zero:
            return other
        return SumMean(self, other)

    __radd__ = __add__

    def __mul__(self, other):
        if isinstance(other, Mean):
            if self.is_zero or other.is_zero:
                return ZeroMean()
            return ProductMean(self, other)
        if isinstance(other, FunctionType):
            return ProductMean(FunctionMean(other), self)
        if self.is_zero:
            return self
        return ScaledMean(self, other)

    __rmul__ = __mul__

    def __neg__(self):
        return self * -1.0

    def __sub__(self, other):
        return self + (-_as_mean(other))

    def stretch(self, stretch):
        return self if self.is_zero else StretchedMean(self, stretch)

    def shift(self, shift):
        return self if self.is_zero else MappedMean(self, InputMap("shift", shift))

    def select(self, dims):
        return self if self.is_zero else MappedMean(self, InputMap("select", tuple(np.atleast_1d(dims).tolist())))

    def transform(self, f):
        return self if self.is_zero else MappedMean(self, InputMap("transform", f))

    def diff(self, dim=0):
        """``m.diff(dim)``: ``dm/dx_dim`` (``stheno/model/measure.py:357``)."""
        return self if self.is_zero else DerivativeMean(self, dim)

    def render(self):
        return type(self).__name__ + "()"

    def display(self, formatter=lambda v: v):
        return self.render()

    def __str__(self):
        return self.render()

    __repr__ = __str__


def _as_mean(m):
    if isinstance(m, Mean):
        return m
    if isinstance(m, FunctionType):
        return FunctionMean(m)
    if isinstance(m, (int, float)) and m == 0:
        return ZeroMean()
    return m * OneMean()


class ZeroMean(Mean):
    is_zero = True

    def _dev(self, x):
        return torch.zeros(x.batch_shape + (x.n, 1), dtype=x.t.dtype, device=x.t.device)

    def render(self):
        return "0"


class OneMean(Mean):
    def _dev(self, x):
        return torch.ones(x.batch_shape + (x.n, 1), dtype=x.t.dtype, device=x.t.device)

    def render(self):
        return "1"


class ScaledMean(Mean):
    def __init__(self, m, scale):
        self.m, self.scale = m, scale

    def dev(self, x):
        return self.scale * self.m.dev(x)

    def render(self):
        return f"{_fmt(self.scale)} * {self.m.render()}"


class SumMean(Mean):
    def __init__(self, a, b):
        self.a, self.b = a, b

    def dev(self, x):
        return self.a.dev(x) + self.b.dev(x)

    def render(self):
        return f"{self.a.render()} + {self.b.render()}"


class ProductMean(Mean):
    def __init__(self, a, b):
        self.a, self.b = a, b

    def dev(self, x):
        return self.a.dev(x) * self.b.dev(x)

    def render(self):
        return f"{self.a.render()} * {self.b.render()}"


class StretchedMean(Mean):
    def __init__(self, m, stretch):
        self.m, self.stretch_ = m, stretch

    def _dev(self, x):
        xs = Input.__new__(Input)
        xs.origin, xs._groups = x.origin, {}
        s = self.stretch_
        sv = s if isinstance(s, torch.Tensor) else torch.as_tensor(np.asarray(s, np.float64), dtype=x.t.dtype,
                                                                   device=x.t.device)
        xs.t = x.t / sv
        xs.src = None
        return self.m.dev(xs)  # ``dev``: composite means (scaled / sum / product / posterior) only define that


class MappedMean(Mean):
    """``m(map(x))`` (``GP.shift/select/transform`` on the mean, ``stheno/model/measure.py:284,322,341``)."""

    def __init__(self, m, imap):
        self.m, self.imap = m, imap

    def _dev(self, x):
        return self.m.dev(self.imap(x))

    def render(self):
        return f"{self.m.render()} {self.imap.render()}"


class DerivativeMean(Mean):
    """``dm/dx_dim`` by forward-mode differentiation of the mean's torch evaluation (user functions, constants, sums /
    products / scalings of those)."""

    def __init__(self, m, dim):
        self.m, self.dim = m, dim

    def _dev(self, x):
        from torch.func import jvp

        def fn(t):
            xi = Input.__new__(Input)
            xi.origin, xi._groups, xi.src, xi.t = x.origin, {}, None, t
            return self.m.dev(xi)

        e = torch.zeros_like(x.t)
        e[..., self.dim] = 1.0
        with torch.enable_grad():
            out = jvp(fn, (x.t.detach(),), (e,))[1]
        return out.detach()

    def render(self):
        return f"d({self.dim}) {self.m.render()}"


class FunctionMean(Mean):
    """A user function ``f(x) -> (n, 1)`` or ``(n,)`` used as a mean (``GP(lambda x: x ** 2, EQ())``)."""

    def __init__(self, f):
        self.f = f

    def _dev(self, x):
        out = self.f(x.t)
        if not isinstance(out, torch.Tensor):
            out = to_dev(out, x.t.dtype)
        return uprank(out.to(x.t.dtype))

    def render(self):
        return getattr(self.f, "__name__", "f")


class PosteriorMean(Mean):
    """``m_i(x) + k_zi(z, x)^T K_z^-1 (y - m_z(z))`` (``stheno/model/observations.py:160-167``).

    ``rhs_key``: key under which ``(y - m_z(z))^T`` was attached to ``K_z`` so that ``L^-1 (y - m_z(z))`` comes out
    of the factorisation itself."""

    def __init__(self, m_i, m_z, k_zi, z, K_z, y, rhs_key=None):
        self.m_i, self.m_z, self.k_zi, self.z, self.K_z, self.y = m_i, m_z, k_zi, z, M._densify(K_z, full=True), y
        self.rhs_key = rhs_key
        self._b = None

    def _half_y(self):
        """``(L^-1 (y - m_z(z)))^T`` padded to ``[B, n_pad]``."""
        if self._b is None:
            ch = self.K_z.chol()
            hb = self.K_z.half_rhs(self.rhs_key) if self.rhs_key is not None else None
            if hb is None:
                diff = self.y - self.m_z.dev(self.z)
                d3, _ = batch_flatten(diff, 2)
                hb = ch.half_solve(d3.transpose(1, 2).contiguous())
            b = torch.zeros(ch.batch, ch.n_pad, dtype=ch.dtype, device=ch.device)
            b[:, : ch.n] = hb[:, 0]
            self._b = b
        return self._b

    def _dot(self, x, V=None, m=None):
        """``k(x, z) K_z^-1 (y - m_z(z))`` ``[B, m]`` (``V``: the solved rows at ``x`` when already formed)."""
        ch = self.K_z.chol()
        if V is None:
            V, m = _cross_rows(self.k_zi, self.z, x, ch)
            ch.solve_rows_(V)
        return ops.row_dot_sq(V, m, ch.n_pad, self._half_y(), want_sq=False)[0]

    def _ybar(self):
        """``y - m_z(z)`` as ``[B, n]`` (with its graph)."""
        d3, _ = batch_flatten(self.y - self.m_z.dev(self.z), 2)
        return d3[..., 0]

    def dev(self, x):
        prior = self.m_i.dev(x)
        dot, _, _ = _posterior_call(self, x, lambda: (self._dot(x), None, None), "the posterior mean", mean=True)
        return prior + dot.reshape(prior.shape[:-1]).unsqueeze(-1)

    def render(self):
        return "PosteriorMean()"


def _route_name(post):
    """The posterior kind named by the error of an uncovered gradient route."""
    from .model.fdd import FDD

    K_z = post.K_z
    if isinstance(K_z, M.BlockDense) or isinstance(post.z, (tuple, FDD)):
        return "multi-output posterior"
    if isinstance(K_z, M.KernelDense):
        return "posterior whose cross kernel is not one flat kernel expression under input maps (derivatives, " \
               "function-scaled, reversed, sums of differently mapped kernels) or whose inputs are multi-output or of another batch"
    return "sparse (pseudo-observation) or non-kernel posterior"


def _shared_posterior(mean, kernel):
    return (
        isinstance(mean, PosteriorMean)
        and isinstance(kernel, PosteriorKernel)
        and mean.K_z is kernel.K_z
        and mean.k_zi is kernel.k_zi
        and kernel.k_zi is kernel.k_zj
        and mean.z is kernel.z
    )


def _sparse_posterior(mean, kernel, x):
    """The sparse counterpart of :func:`_shared_posterior`: the ``PosteriorMean`` and ``PosteriorKernel + SubspaceKernel`` of
    one ``PseudoObs*`` problem (``AbstractPseudoObservations``) at numeric, single-output, unbatched ``x``, with one cross
    kernel that flattens to one descriptor and nothing that requires grad except ``x`` itself -- the marginals
    :func:`_sparse_marginals` streams, differentiable in ``x``.  That cross kernel as :func:`k1_block` gives it, else None."""
    if not (isinstance(mean, PosteriorMean) and isinstance(kernel, SumKernel)):
        return None
    pk, sk, k = kernel.a, kernel.b, mean.k_zi
    if not (isinstance(pk, PosteriorKernel) and isinstance(sk, SubspaceKernel)):
        return None
    if not (pk.K_z is mean.K_z and pk.z is mean.z and sk.z is mean.z):
        return None
    if not (pk.k_zi is k and pk.k_zj is k and sk.k_zi is k and sk.k_zj is k):
        return None
    blk = k1_block(k, mean.z, x)
    if blk is None or blk[2].batch_shape or blk[3].batch_shape or _grad_tensors(mean, kernel):
        return None
    return blk if mean.K_z.chol().batch == 1 and sk.A.chol().batch == 1 else None


def _sparse_marginals(mean, kernel, x, blk, want_dot):
    """``(mean or None, var)`` of a posterior :func:`_sparse_posterior` accepts (``blk``: what it returned), each ``[n, 1]``:
    the K1 rows at ``x`` are formed once per chunk of test points and solved against ``L_z`` and against the factor of ``A``
    (the mean only with ``want_dot``); differentiable in ``x`` (``autograd.sparse_posterior_marginals``)."""
    from .autograd import SparsePosteriorSpec, sparse_posterior_marginals

    flat, scales, zi, xi = blk
    spec = SparsePosteriorSpec(flat, zi.scaled(scales), mean.K_z.chol(), kernel.b.A.chol(),
                               mean._half_y()[0] if want_dot else None)
    prior_m = mean.m_i.dev(x) if want_dot else None
    mu, var = sparse_posterior_marginals(spec, xi.scaled(scales), prior_m, _elwise_any(kernel.a.k_ij, x, None, True))
    return (mu if want_dot else None), var


def marginal_var(mean, kernel, x):
    """``k.elwise(x)`` of a posterior process with mean ``mean``, ``[..., n, 1]``: the streamed sparse marginals where
    :func:`_sparse_posterior` holds, else the kernel's own element-wise evaluation."""
    blk = _sparse_posterior(mean, kernel, x)
    if blk is not None:
        return _sparse_marginals(mean, kernel, x, blk, want_dot=False)[1]
    return _elwise_any(kernel, x, None, True)


def mean_var(mean, kernel, x):
    """``mlkernels.mean_var``: mean ``[..., n, 1]`` (device) and variance (matrix), sharing ``L^-1 k(z, x)`` between
    the two for an exact posterior (``stheno/model/fdd.py:68-70``)."""
    if _shared_posterior(mean, kernel) and not _is_multi(x):
        prior_m = mean.m_i.dev(x)
        prior = M.dense(pairwise(kernel.k_ij, x))

        def fwd():
            V, m = kernel._half(kernel.k_zi, x)
            return mean._dot(x, V, m), None, kernel._cov(x, x, True, prior, V, m)

        out = _posterior_call(mean, x, fwd, None, mean=True, P=prior)
        if out is None:
            return mean.dev(x), pairwise(kernel, x)  # each raises on backward, naming itself
        dot, _, C = out
        mu = prior_m + dot.reshape(prior_m.shape[:-1]).unsqueeze(-1)
        return mu, M.Dense(C, _origin_of_input(x))
    return mean.dev(x), pairwise(kernel, x)


def mean_var_diag(mean, kernel, x):
    """``mlkernels.mean_var_diag``: mean and marginal variances ``[..., n, 1]`` from ONE pass over
    ``V = k(x*, z) L^-T`` (``stheno/model/fdd.py:72-74``; call pattern pinned by ``tests/model/test_model.py:335-365``)."""
    if _shared_posterior(mean, kernel) and not _is_multi(x):
        ch = kernel.K_z.chol()
        prior_m = mean.m_i.dev(x)
        prior_v = _elwise_any(kernel.k_ij, x, None, True)
        shp = prior_m.shape[:-1]
        blk = k1_block(kernel.k_zi, kernel.z, x) if ch.batch == 1 else None

        def fwd():
            if blk is not None and not blk[2].batch_shape and not blk[3].batch_shape:
                # K3 in ONE call: kernel rows -> tensor-core solve -> both reductions, test points streamed through a
                # bounded buffer
                flat, scales, zi, xi = blk
                return ops.posterior_marginals(flat, xi.scaled(scales), zi.scaled(scales), ch, mean._half_y()[0]) + (None,)
            V, m = kernel._half(kernel.k_zi, x)
            return ops.row_dot_sq(V, m, ch.n_pad, mean._half_y()) + (None,)

        dot, sq, _ = _posterior_call(mean, x, fwd, "the posterior marginals", mean=True)
        return prior_m + dot.reshape(shp).unsqueeze(-1), prior_v - sq.reshape(shp).unsqueeze(-1)
    blk = _sparse_posterior(mean, kernel, x)
    if blk is not None:
        return _sparse_marginals(mean, kernel, x, blk, want_dot=True)
    return mean.dev(x), _elwise_any(kernel, x, None, True)
