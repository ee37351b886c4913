"""``GP``: a handle into a :class:`Measure` (``stheno/model/gp.py:58-274``; hot-path subset: construction,
``f(x, noise)``, conditioning, ``+``, ``* scalar``, ``stretch``)."""
from types import FunctionType

import numpy as np
import torch

from ..kernels import Kernel, Mean, OneKernel, OneMean, ZeroMean, FunctionMean
from ..random import RandomProcess
from .fdd import FDD

__all__ = ["assert_same_measure", "intersection_measure_group", "cross", "GP"]


def assert_same_measure(*ps):
    for p in ps[1:]:
        if ps[0].measure != p.measure:
            raise AssertionError(f"Processes {ps[0]} and {p} are associated to different measures.")


def intersection_measure_group(*ps):
    assert_same_measure(*ps)
    inter = list(ps[0]._measures)
    for p in ps[1:]:
        inter = [m for m in inter if any(m is q for q in p._measures)]
    return inter


def cross(*ps):
    """Cartesian product of processes: a multi-output GP (``gp.py:43-55``)."""
    p_cross = GP()
    for measure in intersection_measure_group(*ps):
        measure.cross(p_cross, *ps)
    return p_cross


def _is_numeric(v):
    return isinstance(v, (int, float, np.number, np.ndarray, torch.Tensor))


def _central_fdm(order, deriv, factor=1e8):
    """Grid, coefficients and step of ``fdm.central_fdm(order, deriv, adapt=0, factor=factor)`` [UPSTREAM-RECALLED: fdm is an
    un-vendored dependency].  Central integer grid of ``order`` points (even orders skip the centre); the coefficients solve the Taylor conditions
    ``sum_i c_i g_i^k = k! [k == deriv]``, ``k < order``; the step minimises the bound ``c1 / h^deriv + c2 h^(order - deriv)`` with
    ``c1 = 1e-16 * factor * sum|c|`` (round-off of the function values) and ``c2 = sum|c g^order| / order!`` (truncation)."""
    import math

    half = order // 2
    if order % 2 == 0:  # even: integer points without the centre (order 2 -> [-1, 1]: pinned by README.md:292-293)
        grid = np.concatenate([np.arange(-half, 0), np.arange(1, half + 1)]).astype(np.float64)
    else:
        grid = np.arange(-half, half + 1).astype(np.float64)
    V = np.vander(grid, order, increasing=True).T  # V[k, i] = g_i^k
    rhs = np.zeros(order)
    rhs[deriv] = math.factorial(deriv)
    coefs = np.linalg.solve(V, rhs)
    c1 = 1e-16 * factor * np.sum(np.abs(coefs))
    c2 = np.sum(np.abs(coefs * grid**order)) / math.factorial(order)
    step = (deriv / (order - deriv) * c1 / c2) ** (1.0 / order)
    return grid, coefs, step


class GP(RandomProcess):
    """``GP([mean,] kernel, *, measure=None, name=None)``; ``GP()`` makes an unattached handle."""

    def __init__(self, *args, measure=None, name=None):
        self._measures = []
        if len(args) == 0:
            return
        from .measure import Measure

        if len(args) == 1:
            mean, kernel = ZeroMean(), args[0]
        elif len(args) == 2:
            mean, kernel = args
        else:
            raise TypeError("GP([mean,] kernel)")
        if measure is None:
            measure = Measure.default if Measure.default is not None else Measure()
        if isinstance(mean, FunctionType):
            mean = FunctionMean(mean)
        elif _is_numeric(mean):
            mean = mean * OneMean()
        if isinstance(kernel, FunctionType):
            raise NotImplementedError("function-valued kernels are outside the hot-path scope")
        if _is_numeric(kernel):
            kernel = kernel * OneKernel()
        measure.add_independent_gp(self, mean, kernel)
        if name:
            measure.name(self, name)

    @property
    def measure(self):
        if len(self._measures) == 0:
            raise RuntimeError("GP is not associated to a measure.")
        return self._measures[0]

    @property
    def kernel(self):
        return self.measure.kernels[self]

    @property
    def mean(self):
        return self.measure.means[self]

    @property
    def name(self):
        return self.measure[self]

    @name.setter
    def name(self, name):
        for measure in self._measures:
            measure.name(self, name)

    def __call__(self, x, noise=None):
        """``f(x, noise)`` -> :class:`FDD` (``gp.py:134-144``)."""
        return FDD(self, x, noise)

    def condition(self, *args):
        posterior = self.measure.condition(*args)
        return posterior(self)

    def __or__(self, args):
        """``f | (f(x), y)``, ``f | ((f1(x1), y1), (f2(x2), y2))``, ``f | Obs(...)`` (``gp.py:146-160``)."""
        if isinstance(args, tuple):
            return self.condition(*args)
        return self.condition(args)

    def __add__(self, other):
        res = GP()
        if isinstance(other, GP):
            for measure in intersection_measure_group(self, other):
                measure.sum(res, self, other)
        else:
            for measure in self._measures:
                measure.sum(res, self, other)
        return res

    def __mul__(self, other):
        res = GP()
        if isinstance(other, GP):  # moment-matched product (``measure.py:253-270``)
            for measure in intersection_measure_group(self, other):
                measure.mul(res, self, other)
            return res
        for measure in self._measures:
            measure.mul(res, self, other)
        return res

    def stretch(self, stretch):
        res = GP()
        for measure in self._measures:
            measure.stretch(res, self, stretch)
        return res

    def shift(self, shift):
        """``f.shift(c)``: ``x -> f(x - c)`` (``gp.py:190-195``)."""
        res = GP()
        for measure in self._measures:
            measure.shift(res, self, shift)
        return res

    def select(self, *dims):
        """``f.select(*dims)``: a GP of only those input dimensions (``gp.py:211-216``)."""
        res = GP()
        for measure in self._measures:
            measure.select(res, self, *dims)
        return res

    def transform(self, f):
        """``f.transform(g)``: ``x -> f(g(x))`` (``gp.py:204-209``)."""
        res = GP()
        for measure in self._measures:
            measure.transform(res, self, f)
        return res

    def diff(self, dim=0):
        """``f.diff(dim)``: the derivative process (``gp.py:218-223``)."""
        res = GP()
        for measure in self._measures:
            measure.diff(res, self, dim)
        return res

    def diff_approx(self, deriv=1, order=6):
        """Finite-difference approximation of the ``deriv``-th derivative as a linear combination of shifted copies of this
        GP (``gp.py:225-244``).  The reference takes grid, coefficients and step from ``fdm.central_fdm(order, deriv, adapt=0,
        factor=1e8)``; restated here (``_central_fdm``) and pinned on the README literal (``README.md:292-293``: order 2 ->
        step 1.414213562373095e-4, coefficients -0.5 / 0.5)."""
        grid, coefs, step = _central_fdm(order, deriv)
        df = 0
        for g, c in zip(grid, coefs):
            df = df + float(c) * self.shift(float(-g * step))
        return df / step**deriv

    def sample_function(self, num=1, features=4096, state=None):
        """``num`` functions drawn from this GP -- prior or exact posterior -- as one
        :class:`~stheno_b200.pathwise.FunctionSample`: call it at any points, any number of times, and it evaluates the same
        functions (pathwise conditioning of a ``features``-feature random-Fourier prior sample).  ``state``: a
        ``torch.Generator`` that makes the draw reproducible.  Refuses with ``ValueError`` what it does not cover (products of
        kernel factors, Delta terms, derivative or function-scaled kernels, multi-output, sparse and cross-process posteriors)."""
        from ..pathwise import FunctionSample

        return FunctionSample(self, num=num, features=features, state=state)

    @property
    def stationary(self):
        return self.kernel.stationary

    def display(self, formatter=lambda v: v):
        if self._measures:
            return f"GP({self.mean.display(formatter)}, {self.kernel.display(formatter)})"
        return "GP()"

    def __str__(self):
        return self.display()

    __repr__ = __str__
