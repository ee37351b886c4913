"""Which route each posterior prediction and sparse objective takes.

Every entry point that picks a route on the hot path is wrapped by a recorder that calls through to the real function:
the K1 row builders (``ops.kernel_rows_padded``, ``ops.posterior_marginals``, ``ops.SparseAccumulator``) and the autograd
routes (``autograd.exact_posterior``, ``no_gradient``, ``subspace_cov``, ``sparse_posterior_marginals``, ``sparse_elbo``).
Each case pins the calls the model layer makes (calls an entry point makes from inside its own module are not counted) and,
where ``no_gradient`` nodes are attached, that ``backward()`` raises and the exact text each node raises.

The cases cover ``mean``, ``var``, ``marginals``, ``mean_var`` and ``logpdf`` of exact posteriors and ``PseudoObs*``
posteriors and ELBOs, over plain, stretched, shifted, periodic and derivative kernels, multi-output observations and
batched test points and cross-covariances, with nothing, a kernel variance or the test inputs requiring grad.  The host test runs the cases that
the CPU stand-in backend covers; the GPU test runs every case.

The ``source`` cases pin which route ``Normal.logpdf`` (on a kernel matrix, an assembled multi-output joint, a Woodbury and a
diagonal covariance; ``BlockDense.eligible`` decides whether the joint stays a grid) and ``PseudoObs`` (``elbo``, ``mu``,
``A``; streamed and, for a batched problem, materialised) take for each tensor that can require grad: a kernel variance,
a length scale, RQ's alpha, a shift, a transform's output, the scalar and the vector noise, ``y``, the inputs, a mean
parameter, a variance inside ``f * k`` -- or nothing, with and without grad mode."""
import collections
import sys

import pytest
import torch

KERNELS = ("eq", "rq", "sumprod", "stretched", "shifted", "periodic")
GRADS = ("off", "theta", "xs")

_OPS = ("kernel_rows_padded", "posterior_marginals", "SparseAccumulator")
_AUTOGRAD = ("exact_posterior", "no_gradient", "subspace_cov", "sparse_posterior_marginals", "sparse_elbo")
# also recorded in the source cases: the raw factorisations, the differentiable log-pdfs and kernel matrices, the restatements
_SOURCE_OPS = ("chol_from_kernel", "chol_from_dense", "_potrf")
_SOURCE_AUTOGRAD = ("kernel_logpdf", "dense_logpdf", "kernel_matrix_grad", "kernel_cross_grad")
_SOURCE_GENERIC = ("sparse_compute_torch", "woodbury_terms_torch")


def _kernel(S, name, v):
    return {
        "eq": lambda: v * S.EQ().stretch(0.8),
        "rq": lambda: v * S.RQ(1.5).stretch(0.9),
        "sumprod": lambda: v * S.EQ().stretch(0.8) + 0.5 * S.Matern32().stretch(1.3) * S.EQ().stretch(2.0),
        "stretched": lambda: (v * S.Matern52()).stretch(1.4),
        "shifted": lambda: (v * S.EQ().stretch(0.8)).shift(0.3),
        "periodic": lambda: (v * S.EQ().stretch(0.7)).periodic(2.0),
    }[name]()


def _data(dev, batched=False):
    g = torch.Generator().manual_seed(11)
    x = torch.rand(40, 1, dtype=torch.float64, generator=g) * 4
    xs = torch.rand(2, 12, 1, dtype=torch.float64, generator=g) * 4
    z = torch.linspace(0, 4, 8, dtype=torch.float64)[:, None]
    y = torch.sin(3 * x[:, 0])
    return x.to(dev), (xs if batched else xs[0]).to(dev), z.to(dev), y.to(dev)


def _run(S, dev, kernel, post_kind, call, grad, batched=False):
    """The outputs of one prediction; ``grad``: ``off`` (no grad mode), ``theta`` (the kernel variance) or ``xs``."""
    x, xs, z, y = _data(dev, batched)
    v = torch.tensor(1.3, dtype=torch.float64, device=dev, requires_grad=grad == "theta")
    if grad == "xs":
        xs.requires_grad_(True)
    f = S.GP(_kernel(S, kernel, v))
    if post_kind == "exact":
        obs = S.Obs(f(x, 0.1), y)
    else:
        obs = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[post_kind](f(z), f(x, 0.1), y)
    if call == "elbo":
        return [obs.elbo(f.measure)]
    fdd = (f | obs)(xs)
    if call == "logpdf":
        return [fdd.logpdf(torch.cos(xs[..., 0]).detach())]
    return _predict(S, fdd, call)


def _predict(S, fdd, call):
    if call == "mean":
        return [fdd.mean]
    if call == "var":
        return [S.B.dense(fdd.var)]
    if call == "marginals":
        return list(fdd.marginals())
    m, v = fdd.mean_var
    return [m, S.B.dense(v)]


def _run_derivative(S, dev, call, grad):
    """The posterior of ``f`` given observations of ``f'``: a ``DerivativeKernel`` cross kernel."""
    x, xs, _, y = _data(dev)
    v = torch.tensor(1.3, dtype=torch.float64, device=dev, requires_grad=grad == "theta")
    if grad == "xs":
        xs.requires_grad_(True)
    f = S.GP(v * S.EQ().stretch(0.8))
    post = f.measure | (f.diff()(x, 0.1), y)
    return _predict(S, post(f)(xs), call)


def _run_multi(S, dev, call, grad):
    """Observations of two processes: a multi-output ``z``."""
    x, xs, _, y = _data(dev)
    v = torch.tensor(1.3, dtype=torch.float64, device=dev, requires_grad=grad == "theta")
    if grad == "xs":
        xs.requires_grad_(True)
    f1 = S.GP(v * S.EQ().stretch(0.8))
    f2 = 2.0 * f1
    post = f1 | ((f1(x, 0.1), y), (f2(x + 0.5, 0.1), y))
    return _predict(S, post(xs), call)


def _run_cross(S, dev, call, grad):
    """The posterior kernel between two sets of test points: a cross-covariance."""
    x, xs, _, y = _data(dev)
    xs2 = xs + 0.25
    v = torch.tensor(1.3, dtype=torch.float64, device=dev, requires_grad=grad == "theta")
    if grad == "xs":
        xs.requires_grad_(True)
    f = S.GP(v * S.EQ().stretch(0.8))
    k = (f | (f(x, 0.1), y)).kernel
    return [S.B.dense(k(xs, xs2)) if call == "pairwise" else k.elwise(xs, xs2)]


SOURCES = ("off", "none", "variance", "scale", "alpha", "shift", "transform", "noise", "noise_vec", "y", "x", "mean", "fk")
SOURCE_CALLS = ("logpdf-kernel", "logpdf-block", "logpdf-woodbury", "logpdf-diagonal", "elbo-streamed", "mu-streamed",
                "A-streamed", "elbo-materialised", "mu-materialised", "A-materialised")


def _run_source(S, dev, call, source):
    """The outputs of ``call`` (``<what>-<covariance or layout>``) with the tensor named by ``source`` requiring grad."""
    what, layout = call.split("-")
    g = torch.Generator().manual_seed(5)
    bs = (3,) if layout == "materialised" else ()
    x = (torch.rand(bs + (30, 1), dtype=torch.float64, generator=g) * 4).to(dev)
    z = torch.linspace(0, 4, 8, dtype=torch.float64).repeat(bs + (1,)).unsqueeze(-1).to(dev)
    y = torch.sin(3 * x)

    def leaf(v, *names):
        return torch.as_tensor(v, dtype=torch.float64).to(dev).requires_grad_(source in names)

    v, ell, alpha, c, m = leaf(1.3, "variance", "fk"), leaf(0.8, "scale"), leaf(1.5, "alpha"), leaf(0.3, "shift"), leaf(0.4, "mean")
    W = leaf([[0.9]], "transform")
    noise = leaf(torch.full(x.shape[:-1], 0.1), "noise_vec") if source == "noise_vec" else leaf(0.1, "noise")
    x.requires_grad_(source == "x")
    y.requires_grad_(source == "y")
    k = {"woodbury": lambda: v * S.Linear(), "diagonal": lambda: v * S.Delta()}.get(layout, lambda: v * S.RQ(alpha).stretch(ell))()
    if source == "shift":
        k = k.shift(c)
    elif source == "transform":
        k = k.transform(lambda t: t @ W)
    elif source == "fk":
        k = (lambda t: 1 + 0.1 * t) * k
    f = S.GP(m * S.OneMean(), k)
    if what == "logpdf":
        if layout == "block":
            fdd, yy = S.combine((f(x, noise), y), ((2.0 * f)(x + 0.5, noise), y))
            return [fdd.logpdf(yy)]
        return [f(x, noise).logpdf(y)]
    obs = S.PseudoObs(f(z), f(x, noise), y)
    out = {"elbo": obs.elbo, "mu": obs.mu, "A": obs.A}[what](f.measure)
    return [S.B.dense(out)]


def _source_cases():
    out = []
    for call in SOURCE_CALLS:
        skip = ("scale", "alpha", "fk") if call in ("logpdf-woodbury", "logpdf-diagonal") else ()
        out += [("source", call, s) for s in SOURCES if s not in skip]
    return out


def _observe(S, dev, monkeypatch, case):
    """``(calls per entry point, sorted backward error texts)`` of one case."""
    from stheno_b200 import autograd, generic_grad, kernels
    from stheno_b200 import matrix as M

    calls = collections.Counter()

    def wrap(owner, name):
        fn = getattr(owner, name)

        def rec(*args, **kwargs):
            if sys._getframe(1).f_globals.get("__name__") != owner.__name__:
                calls[name] += 1
            return fn(*args, **kwargs)

        monkeypatch.setattr(owner, name, rec)

    kind, grad = case[0], case[-1]
    for name in _OPS + (_SOURCE_OPS if kind == "source" else ()):
        wrap(kernels.ops, name)
    for name in _AUTOGRAD + (_SOURCE_AUTOGRAD if kind == "source" else ()):
        wrap(autograd, name)
    if kind == "source":
        for name in _SOURCE_GENERIC:
            wrap(generic_grad, name)
        eligible = M.BlockDense.eligible

        def rec_eligible(rows):
            r = eligible(rows)
            calls[f"BlockDense.eligible={r}"] += 1
            return r

        monkeypatch.setattr(M.BlockDense, "eligible", staticmethod(rec_eligible))
    run = {"plain": lambda: _run(S, dev, *case[1:]), "batched": lambda: _run(S, dev, *case[1:-1], grad, batched=True),
           "derivative": lambda: _run_derivative(S, dev, *case[1:]), "multi": lambda: _run_multi(S, dev, *case[1:]),
           "cross": lambda: _run_cross(S, dev, *case[1:]), "source": lambda: _run_source(S, dev, *case[1:])}[kind]
    try:
        if grad == "off":
            with torch.no_grad():
                outs = run()
        else:
            outs = run()
    except (NotImplementedError, RuntimeError) as e:  # a refusal in the forward is a route too
        return dict(calls), [f"{type(e).__name__}: {e}"]
    errors = set()
    for t in outs:
        nodes = _no_gradient_nodes(t)
        if nodes:
            with pytest.raises(NotImplementedError):
                t.sum().backward(retain_graph=True)
        for node in nodes:  # every node's text, not only the one the backward meets first
            with pytest.raises(NotImplementedError) as e:
                node.apply(None)
            errors.add(str(e.value))
    return dict(calls), sorted(errors)


def _no_gradient_nodes(t):
    """The ``autograd.no_gradient`` nodes in ``t``'s graph."""
    stack, seen, out = [t.grad_fn], set(), []
    while stack:
        node = stack.pop()
        if node is None or node in seen:
            continue
        seen.add(node)
        if type(node).__name__ == "_NoGradientBackward":
            out.append(node)
        stack += [f for f, _ in node.next_functions]
    return out


def _case_list():
    out = []
    for k in KERNELS:
        for post in ("exact", "vfe"):
            for call in ("mean", "var", "marginals", "mean_var", "logpdf"):
                out += [("plain", k, post, call, g) for g in GRADS]
        for post in ("vfe", "fitc", "dtc"):
            out += [("plain", k, post, "elbo", g) for g in ("off", "theta")]
    for post in ("exact", "vfe"):
        for call in ("mean", "var", "marginals", "mean_var"):
            out += [("batched", "eq", post, call, g) for g in GRADS]
    for call in ("mean", "var", "marginals", "mean_var"):
        out += [("derivative", call, g) for g in GRADS] + [("multi", call, g) for g in GRADS]
    out += [("cross", call, g) for call in ("pairwise", "elwise") for g in GRADS]
    return out + _source_cases()


CASES = _case_list()


# backward texts
E0 = "gradients through the posterior marginals of a posterior whose cross kernel is not one flat kernel expression under input maps (derivatives, function-scaled, reversed, sums of differently mapped kernels) or whose inputs are multi-output or of another batch are not implemented"
E1 = "gradients through the posterior mean of a posterior whose cross kernel is not one flat kernel expression under input maps (derivatives, function-scaled, reversed, sums of differently mapped kernels) or whose inputs are multi-output or of another batch are not implemented"
E2 = "gradients through the posterior covariance of a posterior whose cross kernel is not one flat kernel expression under input maps (derivatives, function-scaled, reversed, sums of differently mapped kernels) or whose inputs are multi-output or of another batch are not implemented"
E3 = "gradients through a sparse (pseudo-observation) posterior are not implemented"
E4 = "gradients through the posterior mean of a sparse (pseudo-observation) or non-kernel posterior are not implemented"
E5 = "gradients through the posterior variance of a sparse (pseudo-observation) or non-kernel posterior are not implemented"
E6 = "gradients through the posterior variance of a posterior whose cross kernel is not one flat kernel expression under input maps (derivatives, function-scaled, reversed, sums of differently mapped kernels) or whose inputs are multi-output or of another batch are not implemented"
E7 = "gradients through the posterior covariance of a sparse (pseudo-observation) or non-kernel posterior are not implemented"
E8 = "gradients through k.elwise(x, y) with x is not y are not implemented"
E9 = "gradients through the posterior variance of a cross-covariance between different inputs are not implemented"
E10 = "gradients through a posterior cross-covariance between different inputs or processes are not implemented"
E11 = "gradients through the posterior marginals of a sparse (pseudo-observation) or non-kernel posterior are not implemented"
E12 = "gradients through the posterior marginals of a multi-output posterior are not implemented"
E13 = "gradients through the posterior mean of a multi-output posterior are not implemented"
E14 = "gradients through the posterior covariance of a multi-output posterior are not implemented"
E15 = "gradients through a sparse (pseudo-observation) approximation or posterior with input-mapped kernels are not implemented"
E16 = ("NotImplementedError: gradients through FunctionScaledKernel inside a sparse approximation are not implemented (only sums / "
       "products / stretches of the elementary kernels)")

# case -> (calls per entry point, backward texts), on the GPU
EXPECTED = {
    "batched-eq-exact-marginals-off": ({"kernel_rows_padded": 1}, ()),
    "batched-eq-exact-marginals-theta": ({"kernel_rows_padded": 1, "no_gradient": 2}, (E0, )),
    "batched-eq-exact-marginals-xs": ({"kernel_rows_padded": 1, "no_gradient": 2}, (E0, )),
    "batched-eq-exact-mean-off": ({"kernel_rows_padded": 1}, ()),
    "batched-eq-exact-mean-theta": ({"kernel_rows_padded": 1, "no_gradient": 1}, (E1, )),
    "batched-eq-exact-mean-xs": ({"kernel_rows_padded": 1, "no_gradient": 1}, (E1, )),
    "batched-eq-exact-mean_var-off": ({"kernel_rows_padded": 1}, ()),
    "batched-eq-exact-mean_var-theta": ({"kernel_rows_padded": 2, "no_gradient": 2}, (E2, E1, )),
    "batched-eq-exact-mean_var-xs": ({"kernel_rows_padded": 2, "no_gradient": 2}, (E2, E1, )),
    "batched-eq-exact-var-off": ({"kernel_rows_padded": 1}, ()),
    "batched-eq-exact-var-theta": ({"kernel_rows_padded": 1, "no_gradient": 1}, (E2, )),
    "batched-eq-exact-var-xs": ({"kernel_rows_padded": 1, "no_gradient": 1}, (E2, )),
    "batched-eq-vfe-marginals-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "batched-eq-vfe-marginals-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E4, E5, )),
    "batched-eq-vfe-marginals-xs": ({"SparseAccumulator": 1, "kernel_rows_padded": 3, "no_gradient": 3}, (E3, E1, E6, )),
    "batched-eq-vfe-mean-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 1}, ()),
    "batched-eq-vfe-mean-theta": ({"kernel_rows_padded": 1, "no_gradient": 1}, (E4, )),
    "batched-eq-vfe-mean-xs": ({"SparseAccumulator": 1, "kernel_rows_padded": 1, "no_gradient": 1}, (E1, )),
    "batched-eq-vfe-mean_var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "batched-eq-vfe-mean_var-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E7, E4, )),
    "batched-eq-vfe-mean_var-xs": ({"SparseAccumulator": 1, "kernel_rows_padded": 3, "no_gradient": 3}, (E3, E2, E1, )),
    "batched-eq-vfe-var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 2}, ()),
    "batched-eq-vfe-var-theta": ({"kernel_rows_padded": 2, "no_gradient": 2}, (E3, E7, )),
    "batched-eq-vfe-var-xs": ({"SparseAccumulator": 1, "kernel_rows_padded": 2, "no_gradient": 2}, (E3, E2, )),
    "cross-elwise-off": ({"kernel_rows_padded": 2}, ()),
    "cross-elwise-theta": ({"kernel_rows_padded": 2, "no_gradient": 2}, (E8, E9, )),
    "cross-elwise-xs": ({"kernel_rows_padded": 2, "no_gradient": 2}, (E8, E9, )),
    "cross-pairwise-off": ({"kernel_rows_padded": 2}, ()),
    "cross-pairwise-theta": ({"kernel_rows_padded": 2, "no_gradient": 1}, (E10, )),
    "cross-pairwise-xs": ({"kernel_rows_padded": 2, "no_gradient": 1}, (E10, )),
    "derivative-marginals-off": ({}, ()),
    "derivative-marginals-theta": ({"no_gradient": 2}, (E11, )),
    "derivative-marginals-xs": ({"no_gradient": 2}, (E11, )),
    "derivative-mean-off": ({}, ()),
    "derivative-mean-theta": ({"no_gradient": 1}, (E4, )),
    "derivative-mean-xs": ({"no_gradient": 1}, (E4, )),
    "derivative-mean_var-off": ({}, ()),
    "derivative-mean_var-theta": ({"no_gradient": 2}, (E7, E4, )),
    "derivative-mean_var-xs": ({"no_gradient": 2}, (E7, E4, )),
    "derivative-var-off": ({}, ()),
    "derivative-var-theta": ({"no_gradient": 1}, (E7, )),
    "derivative-var-xs": ({"no_gradient": 1}, (E7, )),
    "multi-marginals-off": ({}, ()),
    "multi-marginals-theta": ({"no_gradient": 2}, (E12, )),
    "multi-marginals-xs": ({"no_gradient": 2}, (E12, )),
    "multi-mean-off": ({}, ()),
    "multi-mean-theta": ({"no_gradient": 1}, (E13, )),
    "multi-mean-xs": ({"no_gradient": 1}, (E13, )),
    "multi-mean_var-off": ({}, ()),
    "multi-mean_var-theta": ({"no_gradient": 2}, (E14, E13, )),
    "multi-mean_var-xs": ({"no_gradient": 2}, (E14, E13, )),
    "multi-var-off": ({}, ()),
    "multi-var-theta": ({"no_gradient": 1}, (E14, )),
    "multi-var-xs": ({"no_gradient": 1}, (E14, )),
    "plain-eq-dtc-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-eq-dtc-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-eq-exact-logpdf-off": ({"kernel_rows_padded": 2}, ()),
    "plain-eq-exact-logpdf-theta": ({"exact_posterior": 2, "kernel_rows_padded": 2}, ()),
    "plain-eq-exact-logpdf-xs": ({"exact_posterior": 2, "kernel_rows_padded": 2}, ()),
    "plain-eq-exact-marginals-off": ({"posterior_marginals": 1}, ()),
    "plain-eq-exact-marginals-theta": ({"exact_posterior": 1, "posterior_marginals": 1}, ()),
    "plain-eq-exact-marginals-xs": ({"exact_posterior": 1, "posterior_marginals": 1}, ()),
    "plain-eq-exact-mean-off": ({"kernel_rows_padded": 1}, ()),
    "plain-eq-exact-mean-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-eq-exact-mean-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-eq-exact-mean_var-off": ({"kernel_rows_padded": 1}, ()),
    "plain-eq-exact-mean_var-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-eq-exact-mean_var-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-eq-exact-var-off": ({"kernel_rows_padded": 1}, ()),
    "plain-eq-exact-var-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-eq-exact-var-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-eq-fitc-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-eq-fitc-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-eq-vfe-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-eq-vfe-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-eq-vfe-logpdf-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "plain-eq-vfe-logpdf-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E7, E4, )),
    "plain-eq-vfe-logpdf-xs": ({"SparseAccumulator": 1, "exact_posterior": 2, "kernel_rows_padded": 3, "subspace_cov": 1}, ()),
    "plain-eq-vfe-marginals-off": ({"SparseAccumulator": 1, "sparse_posterior_marginals": 1}, ()),
    "plain-eq-vfe-marginals-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E4, E5, )),
    "plain-eq-vfe-marginals-xs": ({"SparseAccumulator": 1, "sparse_posterior_marginals": 1}, ()),
    "plain-eq-vfe-mean-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 1}, ()),
    "plain-eq-vfe-mean-theta": ({"kernel_rows_padded": 1, "no_gradient": 1}, (E4, )),
    "plain-eq-vfe-mean-xs": ({"SparseAccumulator": 1, "exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-eq-vfe-mean_var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "plain-eq-vfe-mean_var-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E7, E4, )),
    "plain-eq-vfe-mean_var-xs": ({"SparseAccumulator": 1, "exact_posterior": 2, "kernel_rows_padded": 3, "subspace_cov": 1}, ()),
    "plain-eq-vfe-var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 2}, ()),
    "plain-eq-vfe-var-theta": ({"kernel_rows_padded": 2, "no_gradient": 2}, (E3, E7, )),
    "plain-eq-vfe-var-xs": ({"SparseAccumulator": 1, "exact_posterior": 1, "kernel_rows_padded": 2, "subspace_cov": 1}, ()),
    "plain-periodic-dtc-elbo-off": ({}, ()),
    "plain-periodic-dtc-elbo-theta": ({"sparse_elbo": 1}, ()),
    "plain-periodic-exact-logpdf-off": ({}, ()),
    "plain-periodic-exact-logpdf-theta": ({"exact_posterior": 2}, ()),
    "plain-periodic-exact-logpdf-xs": ({"exact_posterior": 2}, ()),
    "plain-periodic-exact-marginals-off": ({}, ()),
    "plain-periodic-exact-marginals-theta": ({"exact_posterior": 1}, ()),
    "plain-periodic-exact-marginals-xs": ({"exact_posterior": 1}, ()),
    "plain-periodic-exact-mean-off": ({}, ()),
    "plain-periodic-exact-mean-theta": ({"exact_posterior": 1}, ()),
    "plain-periodic-exact-mean-xs": ({"exact_posterior": 1}, ()),
    "plain-periodic-exact-mean_var-off": ({}, ()),
    "plain-periodic-exact-mean_var-theta": ({"exact_posterior": 1}, ()),
    "plain-periodic-exact-mean_var-xs": ({"exact_posterior": 1}, ()),
    "plain-periodic-exact-var-off": ({}, ()),
    "plain-periodic-exact-var-theta": ({"exact_posterior": 1}, ()),
    "plain-periodic-exact-var-xs": ({"exact_posterior": 1}, ()),
    "plain-periodic-fitc-elbo-off": ({}, ()),
    "plain-periodic-fitc-elbo-theta": ({"sparse_elbo": 1}, ()),
    "plain-periodic-vfe-elbo-off": ({}, ()),
    "plain-periodic-vfe-elbo-theta": ({"sparse_elbo": 1}, ()),
    "plain-periodic-vfe-logpdf-off": ({}, ()),
    "plain-periodic-vfe-logpdf-theta": ({"no_gradient": 6, "sparse_elbo": 1}, (E15, E3, E7, E4, )),
    "plain-periodic-vfe-logpdf-xs": ({"exact_posterior": 2, "no_gradient": 1}, (E3, )),
    "plain-periodic-vfe-marginals-off": ({}, ()),
    "plain-periodic-vfe-marginals-theta": ({"no_gradient": 6, "sparse_elbo": 1}, (E15, E3, E4, E5, )),
    "plain-periodic-vfe-marginals-xs": ({"exact_posterior": 2, "no_gradient": 1}, (E3, )),
    "plain-periodic-vfe-mean-off": ({}, ()),
    "plain-periodic-vfe-mean-theta": ({"no_gradient": 4, "sparse_elbo": 1}, (E15, E4, )),
    "plain-periodic-vfe-mean-xs": ({"exact_posterior": 1}, ()),
    "plain-periodic-vfe-mean_var-off": ({}, ()),
    "plain-periodic-vfe-mean_var-theta": ({"no_gradient": 6, "sparse_elbo": 1}, (E15, E3, E7, E4, )),
    "plain-periodic-vfe-mean_var-xs": ({"exact_posterior": 2, "no_gradient": 1}, (E3, )),
    "plain-periodic-vfe-var-off": ({}, ()),
    "plain-periodic-vfe-var-theta": ({"no_gradient": 5, "sparse_elbo": 1}, (E15, E3, E7, )),
    "plain-periodic-vfe-var-xs": ({"exact_posterior": 1, "no_gradient": 1}, (E3, )),
    "plain-rq-dtc-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-rq-dtc-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-rq-exact-logpdf-off": ({"kernel_rows_padded": 2}, ()),
    "plain-rq-exact-logpdf-theta": ({"exact_posterior": 2, "kernel_rows_padded": 2}, ()),
    "plain-rq-exact-logpdf-xs": ({"exact_posterior": 2, "kernel_rows_padded": 2}, ()),
    "plain-rq-exact-marginals-off": ({"posterior_marginals": 1}, ()),
    "plain-rq-exact-marginals-theta": ({"exact_posterior": 1, "posterior_marginals": 1}, ()),
    "plain-rq-exact-marginals-xs": ({"exact_posterior": 1, "posterior_marginals": 1}, ()),
    "plain-rq-exact-mean-off": ({"kernel_rows_padded": 1}, ()),
    "plain-rq-exact-mean-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-rq-exact-mean-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-rq-exact-mean_var-off": ({"kernel_rows_padded": 1}, ()),
    "plain-rq-exact-mean_var-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-rq-exact-mean_var-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-rq-exact-var-off": ({"kernel_rows_padded": 1}, ()),
    "plain-rq-exact-var-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-rq-exact-var-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-rq-fitc-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-rq-fitc-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-rq-vfe-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-rq-vfe-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-rq-vfe-logpdf-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "plain-rq-vfe-logpdf-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E7, E4, )),
    "plain-rq-vfe-logpdf-xs": ({"SparseAccumulator": 1, "exact_posterior": 2, "kernel_rows_padded": 3, "subspace_cov": 1}, ()),
    "plain-rq-vfe-marginals-off": ({"SparseAccumulator": 1, "sparse_posterior_marginals": 1}, ()),
    "plain-rq-vfe-marginals-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E4, E5, )),
    "plain-rq-vfe-marginals-xs": ({"SparseAccumulator": 1, "sparse_posterior_marginals": 1}, ()),
    "plain-rq-vfe-mean-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 1}, ()),
    "plain-rq-vfe-mean-theta": ({"kernel_rows_padded": 1, "no_gradient": 1}, (E4, )),
    "plain-rq-vfe-mean-xs": ({"SparseAccumulator": 1, "exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-rq-vfe-mean_var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "plain-rq-vfe-mean_var-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E7, E4, )),
    "plain-rq-vfe-mean_var-xs": ({"SparseAccumulator": 1, "exact_posterior": 2, "kernel_rows_padded": 3, "subspace_cov": 1}, ()),
    "plain-rq-vfe-var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 2}, ()),
    "plain-rq-vfe-var-theta": ({"kernel_rows_padded": 2, "no_gradient": 2}, (E3, E7, )),
    "plain-rq-vfe-var-xs": ({"SparseAccumulator": 1, "exact_posterior": 1, "kernel_rows_padded": 2, "subspace_cov": 1}, ()),
    "plain-shifted-dtc-elbo-off": ({}, ()),
    "plain-shifted-dtc-elbo-theta": ({"sparse_elbo": 1}, ()),
    "plain-shifted-exact-logpdf-off": ({}, ()),
    "plain-shifted-exact-logpdf-theta": ({"exact_posterior": 2}, ()),
    "plain-shifted-exact-logpdf-xs": ({"exact_posterior": 2}, ()),
    "plain-shifted-exact-marginals-off": ({}, ()),
    "plain-shifted-exact-marginals-theta": ({"exact_posterior": 1}, ()),
    "plain-shifted-exact-marginals-xs": ({"exact_posterior": 1}, ()),
    "plain-shifted-exact-mean-off": ({}, ()),
    "plain-shifted-exact-mean-theta": ({"exact_posterior": 1}, ()),
    "plain-shifted-exact-mean-xs": ({"exact_posterior": 1}, ()),
    "plain-shifted-exact-mean_var-off": ({}, ()),
    "plain-shifted-exact-mean_var-theta": ({"exact_posterior": 1}, ()),
    "plain-shifted-exact-mean_var-xs": ({"exact_posterior": 1}, ()),
    "plain-shifted-exact-var-off": ({}, ()),
    "plain-shifted-exact-var-theta": ({"exact_posterior": 1}, ()),
    "plain-shifted-exact-var-xs": ({"exact_posterior": 1}, ()),
    "plain-shifted-fitc-elbo-off": ({}, ()),
    "plain-shifted-fitc-elbo-theta": ({"sparse_elbo": 1}, ()),
    "plain-shifted-vfe-elbo-off": ({}, ()),
    "plain-shifted-vfe-elbo-theta": ({"sparse_elbo": 1}, ()),
    "plain-shifted-vfe-logpdf-off": ({}, ()),
    "plain-shifted-vfe-logpdf-theta": ({"no_gradient": 6, "sparse_elbo": 1}, (E15, E3, E7, E4, )),
    "plain-shifted-vfe-logpdf-xs": ({"exact_posterior": 2, "no_gradient": 1}, (E3, )),
    "plain-shifted-vfe-marginals-off": ({}, ()),
    "plain-shifted-vfe-marginals-theta": ({"no_gradient": 6, "sparse_elbo": 1}, (E15, E3, E4, E5, )),
    "plain-shifted-vfe-marginals-xs": ({"exact_posterior": 2, "no_gradient": 1}, (E3, )),
    "plain-shifted-vfe-mean-off": ({}, ()),
    "plain-shifted-vfe-mean-theta": ({"no_gradient": 4, "sparse_elbo": 1}, (E15, E4, )),
    "plain-shifted-vfe-mean-xs": ({"exact_posterior": 1}, ()),
    "plain-shifted-vfe-mean_var-off": ({}, ()),
    "plain-shifted-vfe-mean_var-theta": ({"no_gradient": 6, "sparse_elbo": 1}, (E15, E3, E7, E4, )),
    "plain-shifted-vfe-mean_var-xs": ({"exact_posterior": 2, "no_gradient": 1}, (E3, )),
    "plain-shifted-vfe-var-off": ({}, ()),
    "plain-shifted-vfe-var-theta": ({"no_gradient": 5, "sparse_elbo": 1}, (E15, E3, E7, )),
    "plain-shifted-vfe-var-xs": ({"exact_posterior": 1, "no_gradient": 1}, (E3, )),
    "plain-stretched-dtc-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-stretched-dtc-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-stretched-exact-logpdf-off": ({"kernel_rows_padded": 2}, ()),
    "plain-stretched-exact-logpdf-theta": ({"exact_posterior": 2, "kernel_rows_padded": 2}, ()),
    "plain-stretched-exact-logpdf-xs": ({"exact_posterior": 2, "kernel_rows_padded": 2}, ()),
    "plain-stretched-exact-marginals-off": ({"posterior_marginals": 1}, ()),
    "plain-stretched-exact-marginals-theta": ({"exact_posterior": 1, "posterior_marginals": 1}, ()),
    "plain-stretched-exact-marginals-xs": ({"exact_posterior": 1, "posterior_marginals": 1}, ()),
    "plain-stretched-exact-mean-off": ({"kernel_rows_padded": 1}, ()),
    "plain-stretched-exact-mean-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-stretched-exact-mean-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-stretched-exact-mean_var-off": ({"kernel_rows_padded": 1}, ()),
    "plain-stretched-exact-mean_var-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-stretched-exact-mean_var-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-stretched-exact-var-off": ({"kernel_rows_padded": 1}, ()),
    "plain-stretched-exact-var-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-stretched-exact-var-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-stretched-fitc-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-stretched-fitc-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-stretched-vfe-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-stretched-vfe-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-stretched-vfe-logpdf-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "plain-stretched-vfe-logpdf-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E7, E4, )),
    "plain-stretched-vfe-logpdf-xs": ({"SparseAccumulator": 1, "exact_posterior": 2, "kernel_rows_padded": 3, "subspace_cov": 1}, ()),
    "plain-stretched-vfe-marginals-off": ({"SparseAccumulator": 1, "sparse_posterior_marginals": 1}, ()),
    "plain-stretched-vfe-marginals-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E4, E5, )),
    "plain-stretched-vfe-marginals-xs": ({"SparseAccumulator": 1, "sparse_posterior_marginals": 1}, ()),
    "plain-stretched-vfe-mean-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 1}, ()),
    "plain-stretched-vfe-mean-theta": ({"kernel_rows_padded": 1, "no_gradient": 1}, (E4, )),
    "plain-stretched-vfe-mean-xs": ({"SparseAccumulator": 1, "exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-stretched-vfe-mean_var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "plain-stretched-vfe-mean_var-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E7, E4, )),
    "plain-stretched-vfe-mean_var-xs": ({"SparseAccumulator": 1, "exact_posterior": 2, "kernel_rows_padded": 3, "subspace_cov": 1}, ()),
    "plain-stretched-vfe-var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 2}, ()),
    "plain-stretched-vfe-var-theta": ({"kernel_rows_padded": 2, "no_gradient": 2}, (E3, E7, )),
    "plain-stretched-vfe-var-xs": ({"SparseAccumulator": 1, "exact_posterior": 1, "kernel_rows_padded": 2, "subspace_cov": 1}, ()),
    "plain-sumprod-dtc-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-sumprod-dtc-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-sumprod-exact-logpdf-off": ({"kernel_rows_padded": 2}, ()),
    "plain-sumprod-exact-logpdf-theta": ({"exact_posterior": 2, "kernel_rows_padded": 2}, ()),
    "plain-sumprod-exact-logpdf-xs": ({"exact_posterior": 2, "kernel_rows_padded": 2}, ()),
    "plain-sumprod-exact-marginals-off": ({"posterior_marginals": 1}, ()),
    "plain-sumprod-exact-marginals-theta": ({"exact_posterior": 1, "posterior_marginals": 1}, ()),
    "plain-sumprod-exact-marginals-xs": ({"exact_posterior": 1, "posterior_marginals": 1}, ()),
    "plain-sumprod-exact-mean-off": ({"kernel_rows_padded": 1}, ()),
    "plain-sumprod-exact-mean-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-sumprod-exact-mean-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-sumprod-exact-mean_var-off": ({"kernel_rows_padded": 1}, ()),
    "plain-sumprod-exact-mean_var-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-sumprod-exact-mean_var-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-sumprod-exact-var-off": ({"kernel_rows_padded": 1}, ()),
    "plain-sumprod-exact-var-theta": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-sumprod-exact-var-xs": ({"exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-sumprod-fitc-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-sumprod-fitc-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-sumprod-vfe-elbo-off": ({"SparseAccumulator": 1}, ()),
    "plain-sumprod-vfe-elbo-theta": ({"SparseAccumulator": 1, "sparse_elbo": 1}, ()),
    "plain-sumprod-vfe-logpdf-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "plain-sumprod-vfe-logpdf-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E7, E4, )),
    "plain-sumprod-vfe-logpdf-xs": ({"SparseAccumulator": 1, "exact_posterior": 2, "kernel_rows_padded": 3, "subspace_cov": 1}, ()),
    "plain-sumprod-vfe-marginals-off": ({"SparseAccumulator": 1, "sparse_posterior_marginals": 1}, ()),
    "plain-sumprod-vfe-marginals-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E4, E5, )),
    "plain-sumprod-vfe-marginals-xs": ({"SparseAccumulator": 1, "sparse_posterior_marginals": 1}, ()),
    "plain-sumprod-vfe-mean-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 1}, ()),
    "plain-sumprod-vfe-mean-theta": ({"kernel_rows_padded": 1, "no_gradient": 1}, (E4, )),
    "plain-sumprod-vfe-mean-xs": ({"SparseAccumulator": 1, "exact_posterior": 1, "kernel_rows_padded": 1}, ()),
    "plain-sumprod-vfe-mean_var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 3}, ()),
    "plain-sumprod-vfe-mean_var-theta": ({"kernel_rows_padded": 3, "no_gradient": 3}, (E3, E7, E4, )),
    "plain-sumprod-vfe-mean_var-xs": ({"SparseAccumulator": 1, "exact_posterior": 2, "kernel_rows_padded": 3, "subspace_cov": 1}, ()),
    "plain-sumprod-vfe-var-off": ({"SparseAccumulator": 1, "kernel_rows_padded": 2}, ()),
    "plain-sumprod-vfe-var-theta": ({"kernel_rows_padded": 2, "no_gradient": 2}, (E3, E7, )),
    "plain-sumprod-vfe-var-xs": ({"SparseAccumulator": 1, "exact_posterior": 1, "kernel_rows_padded": 2, "subspace_cov": 1}, ()),
    "source-A-materialised-alpha": ({"sparse_compute_torch": 1}, ()),
    "source-A-materialised-fk": ({"sparse_compute_torch": 1}, (E16, )),
    "source-A-materialised-mean": ({"sparse_compute_torch": 1}, ()),
    "source-A-materialised-noise": ({"sparse_compute_torch": 1}, ()),
    "source-A-materialised-noise_vec": ({"sparse_compute_torch": 1}, ()),
    "source-A-materialised-none": ({"chol_from_dense": 1, "chol_from_kernel": 1, "kernel_rows_padded": 1}, ()),
    "source-A-materialised-off": ({"chol_from_dense": 1, "chol_from_kernel": 1, "kernel_rows_padded": 1}, ()),
    "source-A-materialised-scale": ({"sparse_compute_torch": 1}, ()),
    "source-A-materialised-shift": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-A-materialised-transform": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-A-materialised-variance": ({"sparse_compute_torch": 1}, ()),
    "source-A-materialised-x": ({"sparse_compute_torch": 1}, ()),
    "source-A-materialised-y": ({"sparse_compute_torch": 1}, ()),
    "source-A-streamed-alpha": ({"sparse_compute_torch": 1}, ()),
    "source-A-streamed-fk": ({"sparse_compute_torch": 1}, (E16, )),
    "source-A-streamed-mean": ({"sparse_compute_torch": 1}, ()),
    "source-A-streamed-noise": ({"sparse_compute_torch": 1}, ()),
    "source-A-streamed-noise_vec": ({"sparse_compute_torch": 1}, ()),
    "source-A-streamed-none": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1}, ()),
    "source-A-streamed-off": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1}, ()),
    "source-A-streamed-scale": ({"sparse_compute_torch": 1}, ()),
    "source-A-streamed-shift": ({"chol_from_dense": 2, "chol_from_kernel": 2, "no_gradient": 3, "sparse_elbo": 1}, (E15, )),
    "source-A-streamed-transform": ({"chol_from_dense": 2, "chol_from_kernel": 2, "no_gradient": 3, "sparse_elbo": 1}, (E15, )),
    "source-A-streamed-variance": ({"sparse_compute_torch": 1}, ()),
    "source-A-streamed-x": ({"sparse_compute_torch": 1}, ()),
    "source-A-streamed-y": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-materialised-alpha": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-materialised-fk": ({"sparse_compute_torch": 1}, (E16, )),
    "source-elbo-materialised-mean": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-materialised-noise": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-materialised-noise_vec": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-materialised-none": ({"chol_from_dense": 1, "chol_from_kernel": 1, "kernel_rows_padded": 1}, ()),
    "source-elbo-materialised-off": ({"chol_from_dense": 1, "chol_from_kernel": 1, "kernel_rows_padded": 1}, ()),
    "source-elbo-materialised-scale": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-materialised-shift": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-elbo-materialised-transform": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-elbo-materialised-variance": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-materialised-x": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-materialised-y": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-streamed-alpha": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-elbo-streamed-fk": ({"sparse_compute_torch": 1}, (E16, )),
    "source-elbo-streamed-mean": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-elbo-streamed-noise": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-elbo-streamed-noise_vec": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-elbo-streamed-none": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1}, ()),
    "source-elbo-streamed-off": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1}, ()),
    "source-elbo-streamed-scale": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-elbo-streamed-shift": ({"chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-elbo-streamed-transform": ({"chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-elbo-streamed-variance": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-elbo-streamed-x": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-elbo-streamed-y": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1, "sparse_elbo": 1}, ()),
    "source-logpdf-block-alpha": ({"BlockDense.eligible=False": 1, "chol_from_dense": 1, "dense_logpdf": 1, "kernel_cross_grad": 2, "kernel_matrix_grad": 2}, ()),
    "source-logpdf-block-fk": ({"BlockDense.eligible=False": 1, "chol_from_dense": 1, "dense_logpdf": 1, "kernel_cross_grad": 2, "kernel_matrix_grad": 2}, ()),
    "source-logpdf-block-mean": ({"BlockDense.eligible=True": 1, "chol_from_dense": 1, "dense_logpdf": 1}, ()),
    "source-logpdf-block-noise": ({"BlockDense.eligible=True": 1, "chol_from_dense": 1, "dense_logpdf": 1}, ()),
    "source-logpdf-block-noise_vec": ({"BlockDense.eligible=True": 1, "chol_from_dense": 1, "dense_logpdf": 1}, ()),
    "source-logpdf-block-none": ({"BlockDense.eligible=True": 1, "chol_from_dense": 1}, ()),
    "source-logpdf-block-off": ({"BlockDense.eligible=True": 1, "_potrf": 1}, ()),
    "source-logpdf-block-scale": ({"BlockDense.eligible=False": 1, "chol_from_dense": 1, "dense_logpdf": 1, "kernel_cross_grad": 2, "kernel_matrix_grad": 2}, ()),
    "source-logpdf-block-shift": ({"BlockDense.eligible=False": 1, "chol_from_dense": 1, "dense_logpdf": 1, "kernel_cross_grad": 2, "kernel_matrix_grad": 2}, ()),
    "source-logpdf-block-transform": ({"BlockDense.eligible=False": 1, "chol_from_dense": 1, "dense_logpdf": 1, "kernel_cross_grad": 2, "kernel_matrix_grad": 2}, ()),
    "source-logpdf-block-variance": ({"BlockDense.eligible=False": 1, "chol_from_dense": 1, "dense_logpdf": 1, "kernel_cross_grad": 2, "kernel_matrix_grad": 2}, ()),
    "source-logpdf-block-x": ({"BlockDense.eligible=False": 1, "chol_from_dense": 1, "dense_logpdf": 1, "kernel_cross_grad": 2, "kernel_matrix_grad": 2}, ()),
    "source-logpdf-block-y": ({"BlockDense.eligible=True": 1, "chol_from_dense": 1, "dense_logpdf": 1}, ()),
    "source-logpdf-diagonal-mean": ({}, ()),
    "source-logpdf-diagonal-noise": ({}, ()),
    "source-logpdf-diagonal-noise_vec": ({}, ()),
    "source-logpdf-diagonal-none": ({}, ()),
    "source-logpdf-diagonal-off": ({}, ()),
    "source-logpdf-diagonal-shift": ({}, ()),
    "source-logpdf-diagonal-transform": ({}, ()),
    "source-logpdf-diagonal-variance": ({}, ()),
    "source-logpdf-diagonal-x": ({}, ()),
    "source-logpdf-diagonal-y": ({}, ()),
    "source-logpdf-kernel-alpha": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-kernel-fk": ({"chol_from_dense": 1, "dense_logpdf": 1, "kernel_matrix_grad": 1}, ()),
    "source-logpdf-kernel-mean": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-kernel-noise": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-kernel-noise_vec": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-kernel-none": ({"chol_from_kernel": 1}, ()),
    "source-logpdf-kernel-off": ({"chol_from_kernel": 1}, ()),
    "source-logpdf-kernel-scale": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-kernel-shift": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-kernel-transform": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-kernel-variance": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-kernel-x": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-kernel-y": ({"chol_from_kernel": 1, "kernel_logpdf": 1}, ()),
    "source-logpdf-woodbury-mean": ({"woodbury_terms_torch": 1}, ()),
    "source-logpdf-woodbury-noise": ({"woodbury_terms_torch": 1}, ()),
    "source-logpdf-woodbury-noise_vec": ({"woodbury_terms_torch": 1}, ()),
    "source-logpdf-woodbury-none": ({"chol_from_dense": 1}, ()),
    "source-logpdf-woodbury-off": ({"chol_from_dense": 1}, ()),
    "source-logpdf-woodbury-shift": ({"woodbury_terms_torch": 1}, ()),
    "source-logpdf-woodbury-transform": ({"woodbury_terms_torch": 1}, ()),
    "source-logpdf-woodbury-variance": ({"woodbury_terms_torch": 1}, ()),
    "source-logpdf-woodbury-x": ({"woodbury_terms_torch": 1}, ()),
    "source-logpdf-woodbury-y": ({"woodbury_terms_torch": 1}, ()),
    "source-mu-materialised-alpha": ({"sparse_compute_torch": 1}, ()),
    "source-mu-materialised-fk": ({"sparse_compute_torch": 1}, (E16, )),
    "source-mu-materialised-mean": ({"sparse_compute_torch": 1}, ()),
    "source-mu-materialised-noise": ({"sparse_compute_torch": 1}, ()),
    "source-mu-materialised-noise_vec": ({"sparse_compute_torch": 1}, ()),
    "source-mu-materialised-none": ({"chol_from_dense": 1, "chol_from_kernel": 1, "kernel_rows_padded": 1}, ()),
    "source-mu-materialised-off": ({"chol_from_dense": 1, "chol_from_kernel": 1, "kernel_rows_padded": 1}, ()),
    "source-mu-materialised-scale": ({"sparse_compute_torch": 1}, ()),
    "source-mu-materialised-shift": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-mu-materialised-transform": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-mu-materialised-variance": ({"sparse_compute_torch": 1}, ()),
    "source-mu-materialised-x": ({"sparse_compute_torch": 1}, ()),
    "source-mu-materialised-y": ({"sparse_compute_torch": 1}, ()),
    "source-mu-streamed-alpha": ({"sparse_compute_torch": 1}, ()),
    "source-mu-streamed-fk": ({"sparse_compute_torch": 1}, (E16, )),
    "source-mu-streamed-mean": ({"sparse_compute_torch": 1}, ()),
    "source-mu-streamed-noise": ({"sparse_compute_torch": 1}, ()),
    "source-mu-streamed-noise_vec": ({"sparse_compute_torch": 1}, ()),
    "source-mu-streamed-none": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1}, ()),
    "source-mu-streamed-off": ({"SparseAccumulator": 1, "chol_from_dense": 1, "chol_from_kernel": 1}, ()),
    "source-mu-streamed-scale": ({"sparse_compute_torch": 1}, ()),
    "source-mu-streamed-shift": ({"chol_from_dense": 2, "chol_from_kernel": 2, "no_gradient": 3, "sparse_elbo": 1}, (E15, )),
    "source-mu-streamed-transform": ({"chol_from_dense": 2, "chol_from_kernel": 2, "no_gradient": 3, "sparse_elbo": 1}, (E15, )),
    "source-mu-streamed-variance": ({"sparse_compute_torch": 1}, ()),
    "source-mu-streamed-x": ({"sparse_compute_torch": 1}, ()),
    "source-mu-streamed-y": ({"sparse_compute_torch": 1}, ()),
}

# where the stand-in backend takes another route: the analytic sparse ELBO needs CUDA tensors, so on the host the ELBO
# under grad takes the torch restatement (or, under input maps, returns no-grad values)
EXPECTED_HOST = {
    "plain-eq-dtc-elbo-theta": ({}, ()),
    "plain-eq-fitc-elbo-theta": ({}, ()),
    "plain-eq-vfe-elbo-theta": ({}, ()),
    "plain-periodic-dtc-elbo-theta": ({"no_gradient": 4}, (E15, )),
    "plain-periodic-fitc-elbo-theta": ({"no_gradient": 4}, (E15, )),
    "plain-periodic-vfe-elbo-theta": ({"no_gradient": 4}, (E15, )),
    "plain-periodic-vfe-logpdf-theta": ({"no_gradient": 7}, (E15, E3, E7, E4, )),
    "plain-periodic-vfe-marginals-theta": ({"no_gradient": 7}, (E15, E3, E4, E5, )),
    "plain-periodic-vfe-mean-theta": ({"no_gradient": 5}, (E15, E4, )),
    "plain-periodic-vfe-mean_var-theta": ({"no_gradient": 7}, (E15, E3, E7, E4, )),
    "plain-periodic-vfe-var-theta": ({"no_gradient": 6}, (E15, E3, E7, )),
    "plain-rq-dtc-elbo-theta": ({}, ()),
    "plain-rq-fitc-elbo-theta": ({}, ()),
    "plain-rq-vfe-elbo-theta": ({}, ()),
    "plain-shifted-dtc-elbo-theta": ({"no_gradient": 4}, (E15, )),
    "plain-shifted-fitc-elbo-theta": ({"no_gradient": 4}, (E15, )),
    "plain-shifted-vfe-elbo-theta": ({"no_gradient": 4}, (E15, )),
    "plain-shifted-vfe-logpdf-theta": ({"no_gradient": 7}, (E15, E3, E7, E4, )),
    "plain-shifted-vfe-marginals-theta": ({"no_gradient": 7}, (E15, E3, E4, E5, )),
    "plain-shifted-vfe-mean-theta": ({"no_gradient": 5}, (E15, E4, )),
    "plain-shifted-vfe-mean_var-theta": ({"no_gradient": 7}, (E15, E3, E7, E4, )),
    "plain-shifted-vfe-var-theta": ({"no_gradient": 6}, (E15, E3, E7, )),
    "plain-stretched-dtc-elbo-theta": ({}, ()),
    "plain-stretched-fitc-elbo-theta": ({}, ()),
    "plain-stretched-vfe-elbo-theta": ({}, ()),
    "plain-sumprod-dtc-elbo-theta": ({}, ()),
    "plain-sumprod-fitc-elbo-theta": ({}, ()),
    "plain-sumprod-vfe-elbo-theta": ({}, ()),
    "source-A-streamed-shift": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-A-streamed-transform": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-elbo-streamed-alpha": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-streamed-mean": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-streamed-noise": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-streamed-noise_vec": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-streamed-scale": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-streamed-shift": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-elbo-streamed-transform": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-elbo-streamed-variance": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-streamed-x": ({"sparse_compute_torch": 1}, ()),
    "source-elbo-streamed-y": ({"sparse_compute_torch": 1}, ()),
    "source-mu-streamed-shift": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
    "source-mu-streamed-transform": ({"chol_from_dense": 1, "chol_from_kernel": 1, "no_gradient": 4}, (E15, )),
}

# cases whose routes reach GPU-only code (the streamed sparse marginals, the analytic backwards)
GPU_ONLY = {
    "plain-eq-vfe-marginals-off",
    "plain-eq-vfe-marginals-xs",
    "plain-periodic-vfe-logpdf-xs",
    "plain-rq-vfe-marginals-off",
    "plain-rq-vfe-marginals-xs",
    "plain-shifted-vfe-logpdf-xs",
    "plain-stretched-vfe-marginals-off",
    "plain-stretched-vfe-marginals-xs",
    "plain-sumprod-vfe-marginals-off",
    "plain-sumprod-vfe-marginals-xs",
}


def _check(S, dev, monkeypatch, case, expected):
    monkeypatch.setattr(S.B, "epsilon", 1e-10)
    monkeypatch.setattr(S.Measure, "default", None)
    calls, texts = expected
    assert _observe(S, dev, monkeypatch, case) == (calls, sorted(texts))


@pytest.mark.parametrize("case", [c for c in CASES if "-".join(c) not in GPU_ONLY], ids="-".join)
def test_routes_on_host(cpu_backend, monkeypatch, case):
    import stheno_b200 as S

    key = "-".join(case)
    _check(S, "cpu", monkeypatch, case, EXPECTED_HOST.get(key, EXPECTED[key]))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids="-".join)
def test_routes_on_gpu(monkeypatch, case):
    import stheno_b200 as S

    _check(S, "cuda", monkeypatch, case, EXPECTED["-".join(case)])
