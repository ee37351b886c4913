"""The value and the gradient of every route-selection case against fp64 references.

``tests/test_route_selection.py`` pins which entry points each case runs; this module checks what those entry points
compute.  The cases are its ``CASES``, run through its recorder (``_observe``) so the calls are asserted against the same
``EXPECTED`` table at every size, with the builders restated here so the data can grow:

- ``route``: exactly the data of ``test_route_selection`` (n = 40, 12 test points, 8 inducing points, d = 1): one K1 tile,
  one chunk.
- ``tile``: ragged multi-tile shapes -- n = 1153 data points and 389 test points (2 x 389 batched) uniform on [-3, 3]^3,
  130 inducing points, noise 0.3, ``B.sparse_chunk`` = 500 (three ragged data chunks) and, for the exact ``marginals``
  cases, 4500 test points (two chunks of ``ops.posterior_marginals``).
- ``emulated``: the exact ``marginals``, ``mean_var`` and ``logpdf`` cases of the six plain kernel families at n = 4100
  under ``B.precision = "auto"``, where the factorisation and the solves run on the int8-slice emulation.

Every output is compared with a NumPy fp64 evaluation through ``oracle/gp_oracle.py``; every gradient the route offers
(grad not ``off`` and no ``no_gradient`` text) with torch fp64 autograd on the host through the restatement below
(``torch.exp``, ``torch.linalg.cholesky``, ``solve_triangular`` and the VFE / FITC / DTC formulas), which shares no code
with the package.  Every output under grad is also compared with its ``off`` twin.  The bars are in ``BARS``; they rest
on the condition-number cap that ``test_condition_cap`` asserts for every matrix the references factorise."""
import functools
import math

import numpy as np
import pytest
import scipy.linalg as sla
import torch

from oracle import gp_oracle as O
from tests import test_route_selection as R
from tests.test_route_selection import CASES, EXPECTED, GPU_ONLY

# One table of bars, fixed for every case and size.  They rest on n u kappa <= 1.3e-9 (u = 2^-53, fp64's unit roundoff; n
# the order) with kappa <= COND_CAP for every matrix the references factorise -- K_x + sigma^2 I (or the joint), K_z + eps I,
# the stored A and the posterior covariance a log-pdf factorises -- which ``test_condition_cap`` asserts at every size.
BARS = {
    "value": 1e-9,  # |out - ref| / scale; scale = max |ref|, for variances and covariances the prior variance
    "grad": 1e-7,  # |grad - ref grad| / max(max |ref grad|, 1e-6 |sum(w * ref out)|) (a shift of a stationary kernel: 0)
    "twin": 1e-12,  # |out under grad - out of the grad-off twin| / scale
    # The one exception, with fixed bars: at the route size the posterior covariance that a posterior-FDD log-pdf factorises
    # has kappa up to 7.3e8 (two of the 12 pinned test points nearly coincide; ``ROUTE_OVER_CAP``).  The largest errors
    # measured there on an H100: values 1.3e-8 (EQ, VFE), gradients 3.5e-6 (EQ, VFE, xs), grad-on vs grad-off 2.5e-9 (EQ, VFE,
    # theta, where the route under grad forms the covariance another way).
    "route_logpdf": {"value": 1e-7, "grad": 1e-5, "twin": 1e-8},
}
COND_CAP = 1e4
COND_PREMISE = 1.3e-9  # n u kappa
# Matrices of the pinned route data above COND_CAP, each with a fixed ceiling over its measured kappa.
ROUTE_OVER_CAP = {
    "A": 2e5,  # the stored L_z A L_z^T of the sparse data sets: up to 1.7e5 (n u kappa = 1.6e-10 at its order 8)
    "K_z periodic": 4e10,  # inducing points 0 and 4 coincide modulo the period 2: singular to the 1e-10 jitter (3.5e10)
    "A periodic": 3e12,  # the stored A on that K_z: up to 2.5e12
    "posterior covariance": 1e9,  # two of the 12 test points nearly coincide: up to 7.3e8 (the ``route_logpdf`` bars)
}

EPS = 1e-10  # ``B.epsilon`` of the route cases
# Data of the larger sizes, chosen to keep every factorised matrix under the cap: observation noise 0.3 (the stored A),
# test points spread over [-4.5, 4.5]^3 (the posterior covariance of a log-pdf), the source cases' data over [-2, 2]^3
# (the Linear kernel's K_x) and the emulated size's data over [-4.5, 4.5]^3 (n u kappa at n = 4100).
NOISE = {"route": 0.1, "tile": 0.3, "emulated": 0.3}
TILE = {"n": 1153, "m": 389, "m_marginals": 4500, "chunk": 500, "x": 3.0, "xs": 4.5, "x_source": 2.0}
EMULATED = {"n": 4100, "calls": ("marginals", "mean_var", "logpdf"), "grads": ("off", "xs"), "x": 4.5, "slices": 8}
F64 = torch.float64


def _key(case):
    return "-".join(case)


# --------------------------------------------------------------------------------------------------------------------
# data and builders, by size
# --------------------------------------------------------------------------------------------------------------------
def _inducing(kernel):
    """130 inducing points: a 5 x 5 x 5 grid over [-4, 4]^3 and five cell centres, spaced at least ~1.4 length scales
    apart (for the periodic kernel over one period, where its effective length scale is period x 0.7 / 2 pi)."""
    lo, h = (0.0, 0.4) if kernel == "periodic" else (-4.0, 2.0)
    t = lo + h * torch.arange(5, dtype=F64)
    grid = torch.cartesian_prod(t, t, t)
    cells = torch.tensor([(0, 0, 0), (1, 2, 3), (3, 1, 0), (2, 3, 1), (0, 3, 2)], dtype=F64)
    return torch.cat([grid, lo + h * (cells + 0.5)])


def _data(dev, size, kernel="eq", batched=False, many=False):
    """``(x, xs, z, y)`` of ``size``; ``many``: the tile size's 4500 test points."""
    if size == "route":
        return R._data(dev, batched)
    g = torch.Generator().manual_seed(11)
    n, r = (TILE["n"], TILE["x"]) if size == "tile" else (EMULATED["n"], EMULATED["x"])
    x = (torch.rand(n, 3, dtype=F64, generator=g) * 2 - 1) * r
    xs = (torch.rand(2, TILE["m_marginals"] if many else TILE["m"], 3, dtype=F64, generator=g) * 2 - 1) * TILE["xs"]
    y = torch.sin(3 * x[:, 0])
    return x.to(dev), (xs if batched else xs[0]).to(dev), _inducing(kernel).to(dev), y.to(dev)


def _many(size, case):
    return size == "tile" and case[:1] == ("plain",) and case[2:4] == ("exact", "marginals")


def _leaf(v, dev, on):
    return torch.tensor(v, dtype=F64, device=dev, requires_grad=on)


def _run(S, dev, size, kernel, post_kind, call, grad, batched=False, many=False):
    """``test_route_selection._run`` at ``size``: ``(outputs, leaf requiring grad or None)``."""
    x, xs, z, y = _data(dev, size, kernel, batched, many)
    v = _leaf(1.3, dev, grad == "theta")
    if grad == "xs":
        xs.requires_grad_(True)
    f = S.GP(R._kernel(S, kernel, v))
    if post_kind == "exact":
        obs = S.Obs(f(x, NOISE[size]), y)
    else:
        obs = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[post_kind](f(z), f(x, NOISE[size]), y)
    leaf = {"theta": v, "xs": xs}.get(grad)
    if call == "elbo":
        return [obs.elbo(f.measure)], leaf
    fdd = (f | obs)(xs)
    if call == "logpdf":
        return [fdd.logpdf(torch.cos(xs[..., 0]).detach())], leaf
    return R._predict(S, fdd, call), leaf


def _run_derivative(S, dev, size, call, grad):
    x, xs, _, y = _data(dev, size)
    v = _leaf(1.3, dev, grad == "theta")
    if grad == "xs":
        xs.requires_grad_(True)
    f = S.GP(v * S.EQ().stretch(0.8))
    post = f.measure | (f.diff()(x, NOISE[size]), y)
    return R._predict(S, post(f)(xs), call), {"theta": v, "xs": xs}.get(grad)


def _run_multi(S, dev, size, call, grad):
    x, xs, _, y = _data(dev, size)
    v = _leaf(1.3, dev, grad == "theta")
    if grad == "xs":
        xs.requires_grad_(True)
    f1 = S.GP(v * S.EQ().stretch(0.8))
    f2 = 2.0 * f1
    post = f1 | ((f1(x, NOISE[size]), y), (f2(x + 0.5, NOISE[size]), y))
    return R._predict(S, post(xs), call), {"theta": v, "xs": xs}.get(grad)


def _run_cross(S, dev, size, call, grad):
    x, xs, _, y = _data(dev, size)
    xs2 = xs + 0.25
    v = _leaf(1.3, dev, grad == "theta")
    if grad == "xs":
        xs.requires_grad_(True)
    f = S.GP(v * S.EQ().stretch(0.8))
    k = (f | (f(x, NOISE[size]), y)).kernel
    out = S.B.dense(k(xs, xs2)) if call == "pairwise" else k.elwise(xs, xs2)
    return [out], {"theta": v, "xs": xs}.get(grad)


def _source_data(size, layout):
    """``(x, z, W)`` of a source case on the host: ``test_route_selection._run_source``'s data at the route size."""
    g = torch.Generator().manual_seed(5)
    bs = (3,) if layout == "materialised" else ()
    if size == "route":
        x = torch.rand(bs + (30, 1), dtype=F64, generator=g) * 4
        z = torch.linspace(0, 4, 8, dtype=F64).repeat(bs + (1,)).unsqueeze(-1)
        return x, z, torch.tensor([[0.9]], dtype=F64)
    x = (torch.rand(bs + (TILE["n"], 3), dtype=F64, generator=g) * 2 - 1) * TILE["x_source"]
    return x, _inducing("rq").expand(bs + (-1, -1)).clone(), 0.9 * torch.eye(3, dtype=F64)


def _source_leaves(size, call, source, dev):
    """The tensors of a source case (on ``dev``), the one named by ``source`` requiring grad."""
    layout = call.split("-")[1]
    x, z, W = _source_data(size, layout)

    def leaf(v, *names):
        return torch.as_tensor(v, dtype=F64).to(dev).requires_grad_(source in names)

    x, z = x.to(dev), z.to(dev)
    t = {"v": leaf(1.3, "variance", "fk"), "ell": leaf(0.8, "scale"), "alpha": leaf(1.5, "alpha"), "c": leaf(0.3, "shift"),
         "m": leaf(0.4, "mean"), "W": leaf(W, "transform"), "x": x, "z": z, "y": torch.sin(3 * x[..., :1])}
    t["noise"] = leaf(torch.full(x.shape[:-1], NOISE[size]), "noise_vec") if source == "noise_vec" else leaf(NOISE[size], "noise")
    x.requires_grad_(source == "x")
    t["y"].requires_grad_(source == "y")
    names = {"variance": "v", "fk": "v", "scale": "ell", "alpha": "alpha", "shift": "c", "mean": "m", "transform": "W",
             "noise": "noise", "noise_vec": "noise", "x": "x", "y": "y"}
    return t, (t[names[source]] if source in names else None)


def _fk(u):
    """The function of ``f * k``: ``1 + 0.1 u`` on the first input dimension (the only one at the route size)."""
    return 1 + 0.1 * u[..., :1]


def _run_source(S, dev, size, call, source):
    """``test_route_selection._run_source`` at ``size``."""
    what, layout = call.split("-")
    t, leaf = _source_leaves(size, call, source, dev)
    v, x, y, noise = t["v"], t["x"], t["y"], t["noise"]
    k = {"woodbury": lambda: v * S.Linear(), "diagonal": lambda: v * S.Delta()}.get(
        layout, lambda: v * S.RQ(t["alpha"]).stretch(t["ell"]))()
    if source == "shift":
        k = k.shift(t["c"])
    elif source == "transform":
        k = k.transform(lambda u: u @ t["W"])
    elif source == "fk":
        k = _fk * k
    f = S.GP(t["m"] * S.OneMean(), k)
    if what == "logpdf":
        if layout == "block":
            fdd, yy = S.combine((f(x, noise), y), ((2.0 * f)(x + 0.5, noise), y))
            return [fdd.logpdf(yy)], leaf
        return [f(x, noise).logpdf(y)], leaf
    obs = S.PseudoObs(f(t["z"]), f(x, noise), y)
    out = {"elbo": obs.elbo, "mu": obs.mu, "A": obs.A}[what](f.measure)
    return [S.B.dense(out)], leaf


_BUILDERS = {"_run": _run, "_run_derivative": _run_derivative, "_run_multi": _run_multi, "_run_cross": _run_cross,
             "_run_source": _run_source}


def _observe(S, dev, monkeypatch, case, size):
    """Run ``case`` at ``size`` through ``test_route_selection._observe`` (its recorder, its backward checks): returns
    ``(calls, texts)`` and ``(outputs, leaf)``, outputs ``None`` when the forward refuses."""
    box = {}

    def at_size(fn):
        def run(S_, dev_, *args, **kwargs):
            if fn is _run and _many(size, case):
                kwargs["many"] = True
            box["outs"], box["leaf"] = fn(S_, dev_, size, *args, **kwargs)
            return box["outs"]

        return run

    for name, fn in _BUILDERS.items():
        monkeypatch.setattr(R, name, at_size(fn))
    monkeypatch.setattr(S.B, "epsilon", EPS)
    monkeypatch.setattr(S.Measure, "default", None)
    if size == "tile":
        monkeypatch.setattr(S.B, "sparse_chunk", TILE["chunk"])
    observed = R._observe(S, dev, monkeypatch, case)
    return observed, (box.get("outs"), box.get("leaf"))


# --------------------------------------------------------------------------------------------------------------------
# references: NumPy fp64 through the oracle (values), torch fp64 autograd on the host (gradients)
# --------------------------------------------------------------------------------------------------------------------
def _eq(ell):
    return ("stretched", ell, ("eq",))


def _spec(name, v):
    """``test_route_selection._kernel`` as an oracle kernel spec (``v`` a float or a torch scalar)."""
    return {
        "eq": ("scaled", v, _eq(0.8)),
        "rq": ("scaled", v, ("stretched", 0.9, ("rq", 1.5))),
        "sumprod": ("sum", ("scaled", v, _eq(0.8)), ("scaled", 0.5, ("product", ("stretched", 1.3, ("matern32",)), _eq(2.0)))),
        "stretched": ("stretched", 1.4, ("scaled", v, ("matern52",))),
        "shifted": ("shifted", 0.3, ("scaled", v, _eq(0.8))),
        "periodic": ("periodic", 2.0, ("scaled", v, _eq(0.7))),
    }[name]


class _NP:
    """NumPy fp64 through the oracle."""

    @staticmethod
    def k(spec, a, b=None):
        return O.kernel_matrix(spec, a, b)

    @staticmethod
    def kdiag(spec, a, b=None):
        return O.kernel_elwise(spec, a, b)[:, 0]

    chol = staticmethod(lambda K: O.chol_eps(K, EPS))
    tri = staticmethod(lambda L, B: sla.solve_triangular(L, B, lower=True))
    cho_solve = staticmethod(lambda L, B: sla.cho_solve((L, True), B))
    logpdf = staticmethod(lambda mean, cov, y: O.normal_logpdf(mean, cov, y, EPS))
    eye = staticmethod(lambda n: np.eye(n))

    @staticmethod
    def sparse(spec, z, x, noise, y, method, mean=None):
        mx = None if mean is None else np.full((x.shape[0], 1), mean)
        mz = None if mean is None else np.full((z.shape[0], 1), mean)
        c = O.sparse_compute(spec, z, x, noise, y, method, mean_x=mx, mean_z=mz, eps=EPS)
        return c["elbo"], c["mu"], c["A"], c["K_z"]


def _tk(spec, a, b=None, ew=False):
    """Torch restatement of the oracle's kernel specs (parameters may be tensors)."""
    b = a if b is None else b
    kind = spec[0]
    if kind == "scaled":
        return spec[1] * _tk(spec[2], a, b, ew)
    if kind == "sum":
        return _tk(spec[1], a, b, ew) + _tk(spec[2], a, b, ew)
    if kind == "product":
        return _tk(spec[1], a, b, ew) * _tk(spec[2], a, b, ew)
    if kind == "stretched":
        return _tk(spec[2], a / spec[1], b / spec[1], ew)
    if kind == "shifted":
        return _tk(spec[2], a - spec[1], b - spec[1], ew)
    if kind == "transformed":
        return _tk(spec[2], spec[1](a), spec[1](b), ew)
    if kind == "periodic":
        def u(t):
            t = t * (2 * math.pi / spec[1])
            return torch.cat([torch.sin(t), torch.cos(t)], -1)

        return _tk(spec[2], u(a), u(b), ew)
    if kind == "linear":
        return (a * b).sum(-1) if ew else a @ b.mT
    diff = a - b if ew else a[..., :, None, :] - b[..., None, :, :]
    d2 = (diff * diff).sum(-1)
    if kind == "eq":
        return torch.exp(-0.5 * d2)
    if kind == "rq":
        return (1 + d2 / (2 * spec[1])) ** (-spec[1])
    if kind == "delta":
        return (d2 < O.DELTA_EPSILON).to(d2.dtype)
    r = torch.sqrt(torch.clamp_min(d2, 1e-30))
    if kind == "matern32":
        s = math.sqrt(3.0) * r
        return (1 + s) * torch.exp(-s)
    if kind == "matern52":
        s = math.sqrt(5.0) * r
        return (1 + s + 5.0 / 3.0 * d2) * torch.exp(-s)
    raise ValueError(kind)


class _T:
    """Torch fp64 on the host, differentiable."""

    k = staticmethod(lambda spec, a, b=None: _tk(spec, a, b))
    kdiag = staticmethod(lambda spec, a, b=None: _tk(spec, a, b, ew=True))
    tri = staticmethod(lambda L, B: torch.linalg.solve_triangular(L, B, upper=False))
    eye = staticmethod(lambda n: torch.eye(n, dtype=F64))

    @staticmethod
    def chol(K):
        return torch.linalg.cholesky(K + EPS * torch.eye(K.shape[-1], dtype=F64))

    cho_solve = staticmethod(lambda L, B: torch.cholesky_solve(B, L))

    @staticmethod
    def logpdf(mean, cov, y):
        L = _T.chol(cov)
        r = _T.tri(L, y.reshape(-1, 1) - mean.reshape(-1, 1))
        return -(2 * torch.log(torch.diagonal(L)).sum() + L.shape[0] * math.log(2 * math.pi) + (r * r).sum()) / 2

    @staticmethod
    def sparse(spec, z, x, noise, y, method, mean=None):
        """``observations.py:279-336`` (VFE / FITC / DTC): ``(elbo, mu, L_z A L_z^T, K_z)``."""
        mean = 0.0 if mean is None else mean
        K_z = _tk(spec, z)
        L_z = _T.chol(K_z)
        W = _T.tri(L_z, _tk(spec, z, x))
        kn = torch.broadcast_to(torch.as_tensor(noise, dtype=F64), (x.shape[0],))
        trace = 0.0
        if method in ("vfe", "fitc"):
            corr = _tk(spec, x, ew=True) - (W * W).sum(0)
            if method == "vfe":
                trace = (corr / kn).sum()
            else:
                kn = kn + corr
        A = _T.eye(z.shape[0]) + (W / kn) @ W.T
        L_A = _T.chol(A)
        ybar = y.reshape(-1, 1) - mean
        prod = (W / kn) @ ybar
        mu = mean + L_z @ torch.cholesky_solve(prod, L_A)
        t = _T.tri(L_A, prod)
        det = torch.log(2 * math.pi * kn).sum() + 2 * torch.log(torch.diagonal(L_A)).sum()
        elbo = -0.5 * (det + (ybar[:, 0] ** 2 / kn).sum() - (t * t).sum() + trace)
        return elbo, mu, L_z @ A @ L_z.T, K_z


class _Post:
    """A Gaussian posterior of ``f``: ``mean(s) = cross(s)^T alpha``, ``cov(s, s2) = prior(s, s2) + sum_i sign_i
    (L_i^-1 cross(s))^T (L_i^-1 cross(s2))``; exact: one factor of ``K_x + sigma^2 I`` with sign -1; sparse: ``L_z`` with
    -1 and the factor of the stored ``A`` with +1."""

    def __init__(self, X, prior, cross, alpha, factors):
        self.X, self.prior, self.cross, self.alpha, self.factors = X, prior, cross, alpha, factors

    def mean(self, s):
        return self.cross(s).T @ self.alpha

    def _terms(self, s, s2):
        c = self.cross(s)
        for sign, L in self.factors:
            v = self.X.tri(L, c)
            yield sign, v, (v if s2 is None else self.X.tri(L, self.cross(s2)))

    def cov(self, s, s2=None):
        out = self.X.k(self.prior, s, s2)
        for sign, v, v2 in self._terms(s, s2):
            out = out + sign * (v.T @ v2)
        return out

    def diag(self, s, s2=None):
        out = self.X.kdiag(self.prior, s, s2)
        for sign, v, v2 in self._terms(s, s2):
            out = out + sign * (v * v2).sum(0)
        return out


def _posterior(X, kind, kernel, post, x, z, y, v, noise):
    """The posterior of a value case (``kind`` plain / batched / derivative / multi / cross) in arithmetic ``X``."""
    spec = _spec("eq" if kind != "plain" and kind != "batched" else kernel, v)
    y = y.reshape(-1, 1)
    if post in ("vfe", "fitc", "dtc"):
        _, mu, A, K_z = X.sparse(spec, z, x, noise, y, post)
        L_z = X.chol(K_z)
        return _Post(X, spec, lambda s: X.k(spec, z, s), X.cho_solve(L_z, mu), [(-1, L_z), (1, X.chol(A))])
    if kind == "derivative":  # NumPy only: every derivative case refuses its gradient, so ``_tk`` has no ``diff`` spec
        inner = _eq(0.8)
        K = X.k(("scaled", v, ("diff", (0, 0), inner)), x)
        cross = lambda s: X.k(("scaled", v, ("diff", (0, None), inner)), x, s)  # cov(f'(x), f(s))
    elif kind == "multi":
        x2 = x + 0.5
        K = _block([[X.k(spec, x), 2 * X.k(spec, x, x2)], [2 * X.k(spec, x2, x), 4 * X.k(spec, x2)]], X)
        cross = lambda s: _block([[X.k(spec, x, s)], [2 * X.k(spec, x2, s)]], X)
        y = _block([[y], [y]], X)
    else:
        K = X.k(spec, x)
        cross = lambda s: X.k(spec, x, s)
    L = X.chol(K + noise * X.eye(K.shape[0]))
    return _Post(X, spec, cross, X.cho_solve(L, y), [(-1, L)])


def _block(rows, X):
    cat = np.concatenate if X is _NP else torch.cat
    return cat([cat(r, -1) for r in rows], -2)


def _predict(X, P, call, xs):
    """The outputs of ``call`` for one (unbatched) set of test points."""
    mean = P.mean(xs)
    if call == "mean":
        return [mean]
    if call == "var":
        return [P.cov(xs)]
    if call == "marginals":
        d = P.diag(xs)
        return [mean[:, 0], np.maximum(d, 0.0) if X is _NP else torch.clamp_min(d, 0.0)]
    if call == "mean_var":
        return [mean, P.cov(xs)]
    if call == "logpdf":
        target = np.cos(xs[:, 0]) if X is _NP else torch.cos(xs[:, 0]).detach()  # the cases' y does not carry xs' gradient
        return [X.logpdf(mean, P.cov(xs), target)]
    raise ValueError(call)


# variance-valued outputs (their scale is the prior variance) by call
_VARIANCES = {"var": (0,), "marginals": (1,), "mean_var": (1,), "pairwise": (0,), "elwise": (0,)}


def _host(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


@functools.lru_cache(maxsize=None)
def _np_data(size, kernel, batched, many):
    return tuple(_host(t) for t in _data("cpu", size, kernel, batched, many))


@functools.lru_cache(maxsize=None)
def _np_posterior(size, kind, kernel, post):
    """The oracle factorisation of one data set, once per (kernel, posterior kind, size)."""
    x, _, z, y = _np_data(size, kernel, False, False)
    return _posterior(_NP, kind, kernel, post, x, z, y, 1.3, NOISE[size])


def _parts(case):
    """``(kind, kernel, post, call, grad)`` of a non-source case (derivative, multi and cross cases use the EQ kernel)."""
    return case if case[0] in ("plain", "batched") else (case[0], "eq", "exact", case[1], case[2])


def _reference(case, size):
    """``(reference outputs, scales)``; a batched output's reference is the list of its members'."""
    if case[0] == "source":
        return _source_reference(_NP, case, size, None)
    kind, kernel, post, call, _ = _parts(case)
    batched = kind == "batched"
    x, xs, z, y = _np_data(size, kernel, batched, _many(size, case))
    if call == "elbo":
        return [np.asarray(_NP.sparse(_spec(kernel, 1.3), z, x, NOISE[size], y.reshape(-1, 1), post)[0])], None
    P = _np_posterior(size, kind, kernel, post)
    if kind == "cross":
        out = P.cov(xs, xs + 0.25) if call == "pairwise" else P.diag(xs, xs + 0.25)
        return [out], _prior_var(P, xs)
    if batched:
        members = [_predict(_NP, P, call, s) for s in xs]
        return [np.stack(o) for o in zip(*members)], _prior_var(P, xs.reshape(-1, xs.shape[-1]))
    return _predict(_NP, P, call, xs), _prior_var(P, xs)


def _prior_var(P, xs):
    return float(np.max(_NP.kdiag(P.prior, xs)))


def _source_spec(X, t, layout, source):
    """The kernel of a source case as a spec, and the function ``f`` of ``f * k`` (or None)."""
    v = t["v"]
    if layout == "woodbury":
        spec = ("scaled", v, ("linear",))
    elif layout == "diagonal":
        spec = ("scaled", v, ("delta",))
    else:
        spec = ("scaled", v, ("stretched", t["ell"], ("rq", t["alpha"])))
    if source == "shift":
        spec = ("shifted", t["c"], spec)
    elif source == "transform":
        W = t["W"]
        spec = ("transformed", lambda u: u @ W, spec) if X is _T else ("transformed", lambda u: u @ _host(W), spec)
    return spec, (_fk if source == "fk" else None)


def _source_outputs(X, t, call, source):
    """The outputs of a source case in arithmetic ``X`` from its tensors ``t`` (unbatched)."""
    what, layout = call.split("-")
    spec, fs = _source_spec(X, t, layout, source)
    x, y, noise, m = t["x"], t["y"], t["noise"], t["m"]

    def K(a, b=None):
        k = X.k(spec, a, b)
        if fs is not None:
            b = a if b is None else b
            k = fs(a) * k * fs(b).T
        return k

    def noise_mat(n):
        return noise * X.eye(n) if np.ndim(_host(noise)) == 0 else (np.diag(noise) if X is _NP else torch.diag(noise))

    if what == "logpdf":
        if layout == "block":
            x2 = x + 0.5
            Kj = _block([[K(x), 2 * K(x, x2)], [2 * K(x2, x), 4 * K(x2)]], X)
            n2 = noise if np.ndim(_host(noise)) == 0 else (np.concatenate if X is _NP else torch.cat)([noise, noise])
            cat = np.concatenate if X is _NP else torch.cat
            Kj = Kj + (n2 * X.eye(Kj.shape[0]) if np.ndim(_host(n2)) == 0 else (np.diag(n2) if X is _NP else torch.diag(n2)))
            mean = cat([m + 0 * y, 2 * m + 0 * y])
            return [X.logpdf(mean, Kj, cat([y, y]))]
        return [X.logpdf(m + 0 * y, K(x) + noise_mat(x.shape[0]), y)]
    elbo, mu, A, _ = X.sparse(spec, t["z"], x, noise, y, "vfe", mean=m)
    return [{"elbo": elbo, "mu": mu, "A": A}[what]]


def _source_reference(X, case, size, leaf_t):
    """The reference outputs of a source case (members of a materialised batch stacked) and their scales."""
    _, call, source = case
    layout = call.split("-")[1]
    if leaf_t is None:
        t, _ = _source_leaves(size, call, source, "cpu")
        t = {k: (_host(v) if X is _NP else v) for k, v in t.items()}
    else:
        t = leaf_t
    if layout != "materialised":
        return _source_outputs(X, t, call, source), None
    per = t["noise"].shape[0] if np.ndim(_host(t["noise"])) == 2 else None
    members = []
    for b in range(t["x"].shape[0]):
        tb = dict(t, x=t["x"][b], z=t["z"][b], y=t["y"][b])
        if per is not None:
            tb["noise"] = t["noise"][b]
        members.append(_source_outputs(X, tb, call, source))
    stack = np.stack if X is _NP else torch.stack
    return [stack(o) for o in zip(*members)], None


# --------------------------------------------------------------------------------------------------------------------
# gradient references
# --------------------------------------------------------------------------------------------------------------------
def _weights(outs):
    g = torch.Generator().manual_seed(3)
    return [torch.randn(o.shape, dtype=F64, generator=g) for o in outs]


def _loss(outs, ws):
    return sum((w.to(o.device) * o).sum() for o, w in zip(outs, ws))


def _grad_reference(case, size, ws):
    """``d sum(w * out) / d leaf`` through torch fp64 autograd on the host."""
    if case[0] == "source":
        _, call, source = case
        t, leaf = _source_leaves(size, call, source, "cpu")
        outs, _ = _source_reference(_T, case, size, t)
    else:
        kind, kernel, post, call, grad = _parts(case)
        x, xs, z, y = _data("cpu", size, kernel, False, _many(size, case))
        v = _leaf(1.3, "cpu", grad == "theta")
        leaf = v if grad == "theta" else xs.requires_grad_(True)
        if call == "elbo":
            outs = [_T.sparse(_spec(kernel, v), z, x, NOISE[size], y, post)[0]]
        else:
            outs = _predict(_T, _posterior(_T, kind, kernel, post, x, z, y, v, NOISE[size]), call, xs)
    loss = _loss(outs, ws)
    (g,) = torch.autograd.grad(loss, leaf, allow_unused=True) if loss.requires_grad else (None,)
    return (torch.zeros_like(leaf) if g is None else g), float(loss)


# --------------------------------------------------------------------------------------------------------------------
# the checks
# --------------------------------------------------------------------------------------------------------------------
def _rel(a, b, scale):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.size == b.size, (a.shape, b.shape)
    scale = max(scale, 1e-300)
    return float(np.max(np.abs(a.reshape(b.shape) - b)) / scale) if b.size else 0.0


def _scales(case, refs, prior):
    call = case[-2] if case[0] in ("plain", "batched") else (case[1] if case[0] != "source" else None)
    var = _VARIANCES.get(call, ()) if prior is not None else ()
    return [prior if i in var else float(np.max(np.abs(r))) for i, r in enumerate(refs)]


def _bar(name, case, size):
    """``BARS[name]``, or ``BARS["route_logpdf"][name]`` for a posterior-FDD log-pdf at the route size."""
    route_logpdf = size == "route" and case[0] == "plain" and case[3] == "logpdf"
    return BARS["route_logpdf"][name] if route_logpdf else BARS[name]


def _check_values(case, size, outs):
    refs, prior = _reference(case, size)
    assert len(outs) == len(refs)
    scales = _scales(case, refs, prior)
    bar, worst = _bar("value", case, size), 0.0
    batched = case[0] == "batched" or case[1:2] in (("elbo-materialised",), ("mu-materialised",), ("A-materialised",))
    for i, (o, r, s) in enumerate(zip(outs, refs, scales)):
        o = _host(o)
        members = zip(o.reshape((r.shape[0], -1)), r) if batched else [(o, r)]
        for b, (ob, rb) in enumerate(members):
            err = _rel(ob, rb, s)
            worst = max(worst, err)
            assert err <= bar, f"output {i} member {b}: {err:.3e} relative to {s:.3e}"
    return scales, worst


def _check_twin(S, dev, case, size, outs, scales):
    """The outputs under grad equal those of the same call with grad mode off: ``"bit-identical"`` or the largest error."""
    if dev == "cpu" and _key(case[:-1] + ("off",)) in GPU_ONLY:
        return "twin on the GPU"
    builder = _BUILDERS[{"plain": "_run", "batched": "_run"}.get(case[0], "_run_" + case[0])]
    args = case[1:]
    kwargs = {"batched": True} if case[0] == "batched" else {}
    if case[0] == "plain" and _many(size, case):
        kwargs["many"] = True
    if case[0] != "source":
        args = args[:-1] + ("off",)
    with torch.no_grad():
        twin, _ = builder(S, dev, size, *args, **kwargs)
    same, worst = [], 0.0
    for i, (o, t, s) in enumerate(zip(outs, twin, scales)):
        o, t = _host(o), _host(t)
        same.append(np.array_equal(o, t))
        err = _rel(o, t, s)
        worst = max(worst, err)
        assert err <= _bar("twin", case, size), f"output {i}: {err:.3e} from the off twin"
    return "bit-identical" if all(same) else f"{worst:.1e}"


def _wants_grad(case, texts):
    return case[-1] not in ("off", "none") and not texts


def _value_case(S, dev, monkeypatch, case, size):
    calls, texts = EXPECTED[_key(case)]
    if dev == "cpu":
        calls, texts = R.EXPECTED_HOST.get(_key(case), (calls, texts))
    observed, (outs, leaf) = _observe(S, dev, monkeypatch, case, size)
    assert observed == (calls, sorted(texts))
    if outs is None:  # the forward refuses: the refusal is the route (asserted above), there is no value
        assert any(t.startswith("NotImplementedError") for t in texts)
        return
    scales, value_err = _check_values(case, size, outs)
    twin = _check_twin(S, dev, case, size, outs, scales) if case[-1] != "off" else "-"
    print(f"\n{size} {_key(case)}: value {value_err:.1e} twin {twin}", end="")
    if _wants_grad(case, texts):
        ws = _weights(outs)
        try:
            loss = _loss(outs, ws)  # an output that does not depend on the leaf (Delta's inputs, A's y) has gradient zero
            (g,) = torch.autograd.grad(loss, leaf, allow_unused=True) if loss.requires_grad else (None,)
        except AttributeError as e:
            if dev == "cpu" and _stand_in(e.obj):
                pytest.skip(f"values checked; the gradient needs the GPU backward ({e.name} is not in the host stand-in)")
            raise
        g = torch.zeros_like(leaf) if g is None else g
        ref, loss = _grad_reference(case, size, ws)
        ref = _host(ref)
        scale = max(float(np.max(np.abs(ref))), 1e-6 * abs(loss))
        err = _rel(_host(g), ref, scale)
        print(f" grad {err:.1e}", end="")
        assert err <= _bar("grad", case, size), f"gradient: {err:.3e} relative to {scale:.3e}"


def _stand_in(obj):
    """Whether ``obj`` is the host stand-in of ``ops`` or one of its objects (which have no analytic backward kernels)."""
    return getattr(obj, "__name__", None) == "tests._cpu_backend" or type(obj).__module__ == "tests._cpu_backend"


def _emulated(case):
    return (case[0] == "plain" and case[2] == "exact" and case[3] in EMULATED["calls"]
            and case[4] in EMULATED["grads"])


def _value_case_list():
    """The cases this module's builders and references cover, built from their own axes."""
    kernels, grads = ("eq", "rq", "sumprod", "stretched", "shifted", "periodic"), ("off", "theta", "xs")
    calls = ("mean", "var", "marginals", "mean_var")
    out = []
    for k in kernels:
        out += [("plain", k, p, c, g) for p in ("exact", "vfe") for c in calls + ("logpdf",) for g in grads]
        out += [("plain", k, p, "elbo", g) for p in ("vfe", "fitc", "dtc") for g in ("off", "theta")]
    out += [("batched", "eq", p, c, g) for p in ("exact", "vfe") for c in calls for g in grads]
    for c in calls:
        out += [("derivative", c, g) for g in grads] + [("multi", c, g) for g in grads]
    out += [("cross", c, g) for c in ("pairwise", "elwise") for g in grads]
    sources = ("off", "none", "variance", "scale", "alpha", "shift", "transform", "noise", "noise_vec", "y", "x", "mean", "fk")
    for what in ("logpdf-kernel", "logpdf-block", "logpdf-woodbury", "logpdf-diagonal"):
        skip = ("scale", "alpha", "fk") if what in ("logpdf-woodbury", "logpdf-diagonal") else ()
        out += [("source", what, s) for s in sources if s not in skip]
    for what in ("elbo", "mu", "A"):
        for layout in ("streamed", "materialised"):
            out += [("source", f"{what}-{layout}", s) for s in sources]
    return out


def test_cases_are_the_route_cases():
    """Every route case has a value check: the cases this module covers are exactly ``test_route_selection.CASES`` (a
    route case added there fails here until its builder and reference are added)."""
    assert sorted(map(_key, _value_case_list())) == sorted(map(_key, CASES))
    assert set(map(_key, CASES)) == set(EXPECTED)


VALUE_CASES = list(CASES)


@pytest.mark.parametrize("case", [c for c in VALUE_CASES if _key(c) not in GPU_ONLY], ids=_key)
def test_values_on_host(cpu_backend, monkeypatch, case):
    import stheno_b200 as S

    _value_case(S, "cpu", monkeypatch, case, "route")


@pytest.mark.gpu
@pytest.mark.parametrize("size", ("route", "tile"))
@pytest.mark.parametrize("case", VALUE_CASES, ids=_key)
def test_values_on_gpu(monkeypatch, case, size):
    """Every case at the route and tile sizes.  The batched cases (two sets of test points, one unbatched problem) caught
    ``ops.kernel_rows_padded``, ``Chol.solve_rows_`` / ``solve_rows_t_`` and ``ops.row_dot_sq`` stepping through the data,
    the factor and the right-hand vector with their own batch strides: the second set read past those buffers (wrong means
    and variances at the route size, an illegal address at the tile size).  They now broadcast the one problem."""
    import stheno_b200 as S

    _value_case(S, "cuda", monkeypatch, case, size)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in VALUE_CASES if _emulated(c)], ids=_key)
def test_values_emulated(monkeypatch, case):
    """n = 4100 under ``B.precision = "auto"``: the factorisation, solves and products run on the int8-slice emulation."""
    import stheno_b200 as S
    from stheno_b200 import ops

    monkeypatch.setattr(S.B, "precision", "auto")
    assert ops._oz_slices() == EMULATED["slices"]  # "auto" emulates a posterior's factor and solves with 8 slices
    ops.gemm_profile(True)
    try:
        _value_case(S, "cuda", monkeypatch, case, "emulated")
        emulated = ops.gemm_profile_read(1)[2]
    finally:
        ops.gemm_profile(False)
    assert emulated > 0


# --------------------------------------------------------------------------------------------------------------------
# the condition numbers the bars rest on
# --------------------------------------------------------------------------------------------------------------------
def _factorised(size, what):
    """``(name, matrix)`` for every matrix the references factorise for the data set ``what`` at ``size``."""
    if what.startswith("source-"):
        layout = what.split("-")[1]
        t, _ = _source_leaves(size, f"x-{layout}", "none", "cpu")
        t = {k: _host(v) for k, v in t.items()}
        out = []
        xb = t["x"] if t["x"].ndim == 3 else t["x"][None]
        zb = t["z"] if t["z"].ndim == 3 else t["z"][None]
        spec = ("scaled", 1.3, ("stretched", 0.8, ("rq", 1.5)))
        noise = NOISE[size]
        for x, z in zip(xb, zb):
            eye = noise * np.eye(x.shape[0])
            if layout == "block":
                x2 = x + 0.5
                K = O.mo_block_kernel([[spec, ("scaled", 2.0, spec)], [("scaled", 2.0, spec), ("scaled", 4.0, spec)]], [x, x2])
                out.append(("joint", K + noise * np.eye(K.shape[0])))
            elif layout == "kernel":
                out.append(("K_x", O.kernel_matrix(spec, x) + eye))
            elif layout == "woodbury":
                out.append(("K_x", O.kernel_matrix(("scaled", 1.3, ("linear",)), x) + eye))
            elif layout == "diagonal":
                out.append(("K_x", O.kernel_matrix(("scaled", 1.3, ("delta",)), x) + eye))
            else:
                _, _, A, K_z = _NP.sparse(spec, z, x, noise, np.sin(3 * x[:, :1]), "vfe", mean=0.4)
                out += [("K_z", K_z + EPS * np.eye(z.shape[0])), ("A", A + EPS * np.eye(z.shape[0]))]
        return out
    kind, kernel, post = what.split("-")
    x, xs, z, y = _np_data(size, kernel, False, False)
    if kind == "logpdf":  # the posterior covariance at the test points of the log-pdf cases
        C = _np_posterior(size, "plain", kernel, post).cov(xs)
        return [("posterior covariance", C + EPS * np.eye(C.shape[0]))]
    if post in ("vfe", "fitc", "dtc"):
        _, _, A, K_z = _NP.sparse(_spec(kernel, 1.3), z, x, NOISE[size], y.reshape(-1, 1), post)
        tag = " periodic" if kernel == "periodic" else ""
        return [("K_z" + tag, K_z + EPS * np.eye(z.shape[0])), ("A" + tag, A + EPS * np.eye(z.shape[0]))]
    L = _np_posterior(size, kind, kernel, post).factors[0][1]
    return [("K_x + sigma^2 I", L @ L.T)]


def _data_sets(size):
    if size == "emulated":
        return [f"{kind}-{k}-exact" for kind in ("plain", "logpdf") for k in R.KERNELS]
    return ([f"plain-{k}-{p}" for k in R.KERNELS for p in ("exact", "vfe", "fitc", "dtc")]
            + [f"logpdf-{k}-{p}" for k in R.KERNELS for p in ("exact", "vfe")]
            + ["derivative-eq-exact", "multi-eq-exact"]
            + [f"source-{layout}" for layout in ("kernel", "block", "woodbury", "diagonal", "streamed", "materialised")])


@pytest.mark.parametrize("size, what", [(s, w) for s in ("route", "tile", "emulated") for w in _data_sets(s)])
def test_condition_cap(size, what):
    """Every matrix the references factorise has ``kappa_2 <= COND_CAP`` and ``n u kappa <= COND_PREMISE`` (n its order):
    the bars rest on it.  The route size's data are pinned by ``test_route_selection``; its matrices above the cap are the
    named entries of ``ROUTE_OVER_CAP``, each under its fixed ceiling."""
    u = 2.0 ** -53
    for name, K in _factorised(size, what):
        lam = np.linalg.eigvalsh(K)  # symmetric positive definite: kappa_2 = lambda_max / lambda_min
        kappa = lam[-1] / lam[0]
        cap = min(COND_CAP, COND_PREMISE / (K.shape[0] * u))
        if size == "route" and name in ROUTE_OVER_CAP:
            cap = ROUTE_OVER_CAP[name]
        assert 0 < kappa <= cap, f"{name}: kappa = {kappa:.3e} > {cap:.3e}"
