"""Analytic gradients of cross-covariances and exact posterior predictions (``autograd._KernelCross`` / ``_ExactPosterior``,
``csrc/kernel_matrix_bwd.cu``: ``gpk_kernel_cross_bwd``) against torch fp64 autograd of plain torch restatements: the
kernel written out in torch, the posterior through ``cholesky`` / ``solve_triangular`` as the reference computes it."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


# ---- the rectangular K1-backward --------------------------------------------------------------------------------------
def _phi(kind, a, b, param):
    """``phi(a_i, b_j)`` ``[B, m, n]`` (differentiable; K1's cross convention: Delta = [r^2 < 1e-10])."""
    if kind == "linear":
        return a @ b.transpose(1, 2)
    if kind == "one":
        return torch.ones(a.shape[0], a.shape[1], b.shape[1], dtype=a.dtype, device=a.device)
    diff = a[:, :, None, :] - b[:, None, :, :]
    d2 = (diff * diff).sum(-1)
    if kind == "delta":
        return (d2 < 1e-10).to(a.dtype)
    if kind == "eq":
        return torch.exp(-0.5 * d2)
    if kind == "rq":
        return (1 + d2 / (2 * param)) ** (-param)
    r = diff.abs()[..., 0] if a.shape[-1] == 1 else torch.sqrt(torch.clamp_min(d2, 1e-30))
    if kind == "matern12":
        return torch.exp(-r)
    if kind == "matern32":
        s = math.sqrt(3.0) * r
        return (1 + s) * torch.exp(-s)
    s = math.sqrt(5.0) * r
    return (1 + s + 5.0 / 3.0 * d2) * torch.exp(-s)


def _k_ref(terms, coefs, a, b):
    out = 0.0
    for (_, fs), c in zip(terms, coefs):
        prod = 1.0
        for f in fs:
            prod = prod * _phi(f[0], a[f[1]], b[f[1]], f[2] if len(f) > 2 else None)
        out = out + c * prod
    return out


ALL = [("eq", 0), ("matern12", 0), ("matern32", 0), ("matern52", 0), ("rq", 0, 1.7), ("linear", 0), ("delta", 0),
       ("one", 0)]
CROSS_CASES = [
    ([(1.0, [f])], 1, 37, 300, 3, 1) for f in ALL
] + [
    ([(1.3, [("eq", 0), ("matern32", 1), ("linear", 0), ("rq", 1, 0.8)]), (0.7, [("matern52", 1)])], 2, 129, 1000, 8, 1),
    ([(0.9, [("matern12", 0)]), (1.1, [("eq", 1), ("linear", 1)]), (0.4, [("delta", 0)])], 2, 200, 65, 1, 3),
    ([(1.2, [("eq", 0), ("matern52", 1)])], 2, 70, 90, 40, 3),
    ([(0.8, [("matern32", 0), ("linear", 0)])], 1, 65, 130, 132, 1),
]


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("terms,groups,m,n,d,batch", CROSS_CASES)
def test_cross_covariance_backward(terms, groups, m, n, d, batch, dtype):
    """``k(x*, x)`` with ``x* is not x``: gradients w.r.t. coefficients, both point sets (and so the length scales), with
    coincident cross pairs (Matern-1/2's subgradient 0, Delta's indicator)."""
    from stheno_b200 import autograd, ops

    g = torch.Generator(device="cuda").manual_seed(m + n + d)
    x = torch.randn(groups, batch, n, d, dtype=torch.float64, device="cuda", generator=g) / math.sqrt(d)
    xs = torch.randn(groups, batch, m, d, dtype=torch.float64, device="cuda", generator=g) / math.sqrt(d)
    k = min(m, n) // 3
    xs[:, :, :k] = x[:, :, :k]  # coincident cross pairs
    G = torch.randn(batch, m, n, dtype=torch.float64, device="cuda", generator=g)
    coefs0 = torch.tensor([c for c, _ in terms], dtype=torch.float64, device="cuda")

    coefs = coefs0.to(dtype).clone().requires_grad_(True)
    xsv, xv = xs.to(dtype).clone().requires_grad_(True), x.to(dtype).clone().requires_grad_(True)
    flat = ops.FlatKernel(terms, groups)
    flat.coef_raw = list(coefs.unbind())
    K = autograd.kernel_cross_grad(flat, xsv, xv)
    (G.to(dtype) * K).sum().backward()

    cr, xsr, xr = coefs0.clone().requires_grad_(True), xs.clone().requires_grad_(True), x.clone().requires_grad_(True)
    Kr = _k_ref(terms, cr.unbind(), xsr, xr)
    ((G * Kr).sum() + 0.0 * (xsr.sum() + xr.sum())).backward()  # kinds like One and Delta have gradient 0
    tol = 1e-10 if dtype == torch.float64 else 1e-4
    for name, got, want in (("K", K.detach(), Kr.detach()), ("coefs", coefs.grad, cr.grad), ("xs", xsv.grad, xsr.grad),
                            ("x", xv.grad, xr.grad)):
        scale = max(want.abs().max().item(), 1e-300)
        err = (got.double() - want).abs().max().item()
        assert err <= tol * scale, (name, err, scale)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_elwise_backward(dtype):
    """``k.elwise(x)`` through the prior-variance term: Linear's diagonal depends on x, the stationary kinds' only on the
    coefficients."""
    from stheno_b200 import autograd, ops

    terms = [(1.3, [("eq", 0)]), (0.7, [("linear", 1), ("matern32", 0)]), (0.2, [("delta", 0)])]
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(2, 2, 301, 5, dtype=torch.float64, device="cuda", generator=g)
    w = torch.randn(2, 301, dtype=torch.float64, device="cuda", generator=g)
    coefs0 = torch.tensor([c for c, _ in terms], dtype=torch.float64, device="cuda")
    coefs, xv = coefs0.to(dtype).clone().requires_grad_(True), x.to(dtype).clone().requires_grad_(True)
    flat = ops.FlatKernel(terms, 2)
    flat.coef_raw = list(coefs.unbind())
    (w.to(dtype) * autograd.kernel_diag_grad(flat, xv)).sum().backward()
    cr, xr = coefs0.clone().requires_grad_(True), x.clone().requires_grad_(True)
    kd = cr[0] + cr[1] * (xr[1] * xr[1]).sum(-1) + cr[2]
    (w * kd).sum().backward()
    tol = 1e-10 if dtype == torch.float64 else 1e-4
    for got, want in ((coefs.grad, cr.grad), (xv.grad, xr.grad)):
        assert (got.double() - want).abs().max().item() <= tol * want.abs().max().item()


def test_public_cross_kernel_and_elwise():
    """``k(x, y)`` and ``k.elwise(x)`` of the public API carry the graph to scales, length scales and both inputs."""
    import stheno_b200 as S
    from stheno_b200 import matrix as M

    g = torch.Generator(device="cuda").manual_seed(2)
    x0 = torch.randn(80, 3, dtype=torch.float64, device="cuda", generator=g)
    y0 = torch.randn(50, 3, dtype=torch.float64, device="cuda", generator=g)
    G = torch.randn(80, 50, dtype=torch.float64, device="cuda", generator=g)

    def run(ref):
        v, l = (torch.tensor(1.4, dtype=torch.float64, device="cuda", requires_grad=True),
                torch.tensor([0.7, 1.1, 1.9], dtype=torch.float64, device="cuda", requires_grad=True))
        x, y = x0.clone().requires_grad_(True), y0.clone().requires_grad_(True)
        if ref:
            d2 = (((x / l)[:, None] - (y / l)[None]) ** 2).sum(-1)
            K, kd = v * torch.exp(-0.5 * d2), v * torch.ones(80, dtype=x.dtype, device=x.device)
        else:
            k = v * S.EQ().stretch(l)
            K, kd = M.dense(k(x, y)), k.elwise(x)[:, 0]
        ((G * K).sum() + (kd * x0[:, 0]).sum()).backward()
        return [t.grad for t in (v, l, x, y)]

    for a, b in zip(run(False), run(True)):
        assert (a - b).abs().max().item() <= 1e-10 * max(1.0, b.abs().max().item())


# ---- exact posterior predictions ----------------------------------------------------------------------------------------
def _params(extra):
    def t(v):
        return torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True)

    p = {"var": t(1.3), "scale": t(0.8), "noise": t(0.15), "var2": t(0.6), "scale2": t(1.7)}
    if "linear" in extra:
        p["lin"] = t(0.3)
    if "mean" in extra:
        p["c"] = t(0.5)
    return p


def _noise(p, n, extra):
    if "hetero" in extra:
        return p["noise"] * (1.0 + torch.linspace(0, 1, n, dtype=torch.float64, device="cuda"))
    return p["noise"]


def _model(S, p, n, extra):
    k = p["var"] * S.EQ().stretch(p["scale"]) + p["var2"] * S.Matern52().stretch(p["scale2"])
    if "linear" in extra:
        k = k + p["lin"] * S.Linear()
    if "mean" in extra:
        c = p["c"]
        return S.GP(lambda x: c * x[..., :1], k)
    return S.GP(k)


def _ref_posterior(p, x, y, xs, extra, eps):
    """``(mu [.., m], var [.., m], cov [.., m, m])`` by dense cholesky / solve_triangular in torch fp64."""

    def kern(a, b):
        d2 = lambda s: (((a / s)[..., :, None, :] - (b / s)[..., None, :, :]) ** 2).sum(-1)
        K = p["var"] * torch.exp(-0.5 * d2(p["scale"]))
        r2 = d2(p["scale2"])
        r = torch.sqrt(torch.clamp_min(r2, 1e-30))
        s = math.sqrt(5.0) * r
        K = K + p["var2"] * (1 + s + 5.0 / 3.0 * r2) * torch.exp(-s)
        if "linear" in extra:
            K = K + p["lin"] * a @ b.transpose(-1, -2)
        return K

    mean = (lambda t: p["c"] * t[..., 0]) if "mean" in extra else (lambda t: torch.zeros_like(t[..., 0]))
    n = x.shape[-2]
    nz = _noise(p, n, extra)
    K = kern(x, x) + torch.diag_embed(nz * torch.ones(n, dtype=x.dtype, device=x.device) + eps)
    L = torch.linalg.cholesky(K)
    Ks = kern(xs, x)
    A = torch.linalg.solve_triangular(L, Ks.transpose(-1, -2), upper=False)  # V^T
    h = torch.linalg.solve_triangular(L, (y - mean(x)).unsqueeze(-1), upper=False)
    mu = mean(xs) + (A * h).sum(-2)
    cov = kern(xs, xs) - A.transpose(-1, -2) @ A
    return mu, torch.diagonal(cov, dim1=-2, dim2=-1), cov


def _check(got, want, what):
    for name in want:
        a, b = got[name], want[name]
        err = (a - b).abs().max().item()
        assert err <= 1e-8 * max(1.0, b.abs().max().item()), (what, name, err, b.abs().max().item())


def _posterior_case(n, m, d, extra=(), entry="marginals", batch=None, seed=0):
    import stheno_b200 as S
    from stheno_b200 import matrix as M

    S.B.epsilon = 1e-10
    g = torch.Generator(device="cuda").manual_seed(seed + n + m)
    bs = () if batch is None else (batch,)
    x0 = torch.randn(bs + (n, d), dtype=torch.float64, device="cuda", generator=g)
    xs0 = torch.randn(bs + (m, d), dtype=torch.float64, device="cuda", generator=g)
    y0 = torch.sin(x0.sum(-1)) + 0.1 * torch.randn(bs + (n,), dtype=torch.float64, device="cuda", generator=g)
    a = torch.randn(bs + (m,), dtype=torch.float64, device="cuda", generator=g)
    b = torch.randn(bs + (m,), dtype=torch.float64, device="cuda", generator=g)  # both signs
    Gc = torch.randn(bs + (m, m), dtype=torch.float64, device="cuda", generator=g)

    def loss_of(mu, var, cov):
        out = 0.0
        if mu is not None:
            out = out + (a * mu).sum()
        if var is not None:
            out = out + (b * var).sum()
        if cov is not None:
            out = out + (Gc * cov).sum()
        return out

    def run(ref):
        p = _params(extra)
        x, xs, y = x0.clone().requires_grad_(True), xs0.clone().requires_grad_(True), y0.clone().requires_grad_(True)
        if ref:
            mu, var, cov = _ref_posterior(p, x, y, xs, extra, S.B.epsilon)
            mu, var, cov = {"mean": (mu, None, None), "var_diag": (None, var, None), "var": (None, None, cov),
                            "mean_var": (mu, None, cov), "bounds": (mu - 1.96 * var.sqrt(), mu + 1.96 * var.sqrt(), None)
                            }.get(entry, (mu, var, None))
        else:
            f = _model(S, p, n, extra)
            post = (f | (f(x, _noise(p, n, extra)), y if batch is None else y[..., None]))(xs)
            if entry == "mean":
                mu, var, cov = post.mean[..., 0], None, None
            elif entry == "var_diag":
                mu, var, cov = None, post.var_diag, None
            elif entry == "var":
                mu, var, cov = None, None, M.dense(post.var)
            elif entry == "mean_var":
                mean, v = post.mean_var
                mu, var, cov = mean[..., 0], None, M.dense(v)
            elif entry == "bounds":
                _, lo, hi = post.marginal_credible_bounds()
                mu, var, cov = lo, hi, None
            else:
                mu, var = post.marginals()
                cov = None
        loss = loss_of(mu, var, cov)
        loss.backward()
        grads = {k: v.grad for k, v in p.items()}
        grads.update(x=x.grad, xs=xs.grad, y=y.grad)
        return {k: (v if v is not None else torch.zeros(())) for k, v in grads.items()}, loss.detach()

    got, lg = run(False)
    want, lr = run(True)
    assert abs(lg.item() - lr.item()) <= 1e-8 * max(1.0, abs(lr.item()))
    _check(got, want, (n, m, d, extra, entry, batch))


@pytest.mark.parametrize("n,m,d", [(50, 40, 1), (300, 200, 3), (700, 5000, 8), (8192, 1024, 8)])
def test_posterior_marginal_gradients(n, m, d):
    _posterior_case(n, m, d)


@pytest.mark.parametrize("extra", [("linear",), ("hetero",), ("mean",), ("linear", "hetero", "mean")])
def test_posterior_gradients_model_variants(extra):
    _posterior_case(300, 200, 3, extra)


@pytest.mark.parametrize("entry", ["mean", "var_diag", "marginals", "bounds", "var", "mean_var"])
def test_posterior_entry_points(entry):
    _posterior_case(300, 120, 3, ("mean",), entry=entry)


@pytest.mark.parametrize("entry", ["mean", "var_diag", "var"])
def test_posterior_batched_inputs(entry):
    _posterior_case(120, 50, 2, entry=entry, batch=2)


def _big_posterior(n=8192, m=1024, d=8, want=("xs",)):
    import stheno_b200 as S

    S.B.epsilon = 1e-10
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    xs = torch.randn(m, d, dtype=torch.float64, device="cuda", generator=g).requires_grad_("xs" in want)
    y = torch.sin(x.sum(-1))
    f = S.GP(S.EQ().stretch(2.0))
    return f, x, xs, y


def test_values_bit_identical_with_grad_enabled():
    f, x, xs, y = _big_posterior()
    post = f | (f(x, 0.1), y)
    with torch.no_grad():
        m0, v0 = post(xs).marginals()
    m1, v1 = post(xs).marginals()
    assert m1.requires_grad and v1.requires_grad
    assert torch.equal(m0, m1.detach()) and torch.equal(v0, v1.detach())


@pytest.mark.parametrize("entry,m,bound", [("marginals", 1024, 8192 * 8192 * 8 // 2), ("mean", 4096, 4096 * 8192 * 8 // 4)])
def test_cheap_backward_memory(entry, m, bound):
    """Only x* requires grad: no n x n gradient of K_x; for the mean alone no rows x n buffer either."""
    f, x, xs, y = _big_posterior(m=m)
    post = (f | (f(x, 0.1), y))(xs)
    if entry == "mean":
        loss = post.mean.sum()
    else:
        mu, var = post.marginals()
        loss = (mu + var).sum()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert xs.grad is not None and torch.isfinite(xs.grad).all()
    assert peak < bound, (peak, bound)


def test_uncovered_routes_raise():
    """Sparse and multi-output posteriors (and posterior samples) keep their values and refuse a backward."""
    import stheno_b200 as S

    S.B.epsilon = 1e-10
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(60, 1, dtype=torch.float64, device="cuda", generator=g)
    z = torch.linspace(-2, 2, 10, dtype=torch.float64, device="cuda")[:, None]
    xs = torch.randn(20, 1, dtype=torch.float64, device="cuda", generator=g)
    y0 = torch.sin(x[:, 0])

    def sparse(grad):
        y = y0.clone().requires_grad_(grad)
        f = S.GP(S.EQ())
        return (f | S.PseudoObs(f(z), f(x, 0.1), y))(xs).marginals()

    def multi(grad):
        y = y0.clone().requires_grad_(grad)
        f1 = S.GP(S.EQ())
        f2 = 2.0 * f1
        return (f1 | ((f1(x, 0.1), y), (f2(x + 0.5, 0.1), y)))(xs).marginals()

    for build in (sparse, multi):
        with torch.no_grad():
            want = build(False)
        got = build(True)
        for a, b in zip(got, want):  # the sparse ELBO has its own differentiable route: equal up to rounding
            assert torch.allclose(a.detach(), b, rtol=1e-9, atol=1e-12)
        with pytest.raises(NotImplementedError):
            (got[0].sum() + got[1].sum()).backward()

    v = torch.tensor(1.2, dtype=torch.float64, device="cuda", requires_grad=True)
    f = S.GP(v * S.EQ())
    s = (f | (f(x, 0.1), y0))(xs).sample()
    with pytest.raises(NotImplementedError):
        s.sum().backward()


def test_bayesian_optimisation_steps():
    """Maximise mu + 2 sigma over x* with torch.optim; the first gradient matches central differences of the forward."""
    import stheno_b200 as S

    S.B.epsilon = 1e-10
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.rand(40, 2, dtype=torch.float64, device="cuda", generator=g) * 4
    y = torch.sin(x[:, 0]) * torch.cos(x[:, 1])
    f = S.GP(S.EQ().stretch(0.7))
    post = f | (f(x, 0.01), y)

    def acq(xs):
        mu, var = post(xs).marginals()
        return (mu + 2 * var.sqrt()).sum()

    xs = (torch.rand(8, 2, dtype=torch.float64, device="cuda", generator=g) * 4).requires_grad_(True)
    a0 = acq(xs)
    a0.backward()
    g0 = xs.grad.clone()
    h = 1e-6
    fd = torch.zeros_like(g0)
    with torch.no_grad():
        for i in range(xs.shape[0]):
            for j in range(xs.shape[1]):
                e = torch.zeros_like(xs)
                e[i, j] = h
                fd[i, j] = (acq(xs + e) - acq(xs - e)) / (2 * h)
    assert (g0 - fd).abs().max().item() <= 1e-6 * max(1.0, fd.abs().max().item())
    opt = torch.optim.Adam([xs], lr=0.05)
    for _ in range(10):
        opt.zero_grad()
        (-acq(xs)).backward()
        opt.step()
    with torch.no_grad():
        assert acq(xs).item() > a0.item()


@pytest.mark.parametrize("form", ["factored", "uv_only", "dense_w", "gdiag_only"])
def test_cross_backward_factored_upstream(form):
    """``gpk_kernel_cross_bwd`` driven directly with ``G = r o W + u v^T`` (W a padded view, batch 2) and the prior-variance
    term: the column pass reads W transposed, takes r as a column scale and swaps u and v."""
    from stheno_b200 import _lib, ops

    terms = [(1.1, [("eq", 0), ("linear", 1)]), (0.6, [("matern12", 1)]), (0.3, [("delta", 0)]), (0.9, [("linear", 0)])]
    g = torch.Generator(device="cuda").manual_seed(17)
    B, m, n, d = 2, 150, 333, 4
    xs = torch.randn(2, B, m, d, dtype=torch.float64, device="cuda", generator=g) / 2
    x = torch.randn(2, B, n, d, dtype=torch.float64, device="cuda", generator=g) / 2
    xs[:, :, :20] = x[:, :, :20]
    Wbuf = torch.randn(B, 256, 384, dtype=torch.float64, device="cuda", generator=g)
    W = Wbuf[:, :m, :]  # ld 384 > n
    r, u, gd = (torch.randn(B, m, dtype=torch.float64, device="cuda", generator=g) for _ in range(3))
    v = torch.randn(B, n, dtype=torch.float64, device="cuda", generator=g)
    use_w, use_r, use_uv, use_gd = {"factored": (1, 1, 1, 1), "uv_only": (0, 0, 1, 0), "dense_w": (1, 0, 0, 1),
                                    "gdiag_only": (0, 0, 0, 1)}[form]
    flat = ops.FlatKernel(terms, 2)
    ts = torch.zeros(B, _lib.GPK_MAX_TERMS, dtype=torch.float64, device="cuda")
    gxs, gx = torch.zeros_like(xs), torch.zeros_like(x)
    ops.kernel_cross_bwd(flat, xs, x, W=W if use_w else None, r=r if use_r else None, u=u if use_uv else None,
                         v=v if use_uv else None, gdiag=gd if use_gd else None, term_sum=ts, grad_xsg=gxs, grad_xg=gx)

    c = torch.tensor([t for t, _ in terms], dtype=torch.float64, device="cuda").requires_grad_(True)
    xsr, xr = xs.clone().requires_grad_(True), x.clone().requires_grad_(True)
    G = torch.zeros(B, m, n, dtype=torch.float64, device="cuda")
    if use_w:
        G = G + W[:, :, :n] * (r[:, :, None] if use_r else 1.0)
    if use_uv:
        G = G + u[:, :, None] * v[:, None, :]
    loss = (G * _k_ref(terms, c.unbind(), xsr, xr)).sum() + 0.0 * (xsr.sum() + xr.sum())
    if use_gd:
        loss = loss + (gd * torch.diagonal(_k_ref(terms, c.unbind(), xsr, xsr), dim1=1, dim2=2)).sum()
    loss.backward()
    for name, got, want in (("coefs", ts[:, : len(terms)].sum(0), c.grad), ("xs", gxs, xsr.grad), ("x", gx, xr.grad)):
        err = (got - want).abs().max().item()
        assert err <= 1e-10 * max(want.abs().max().item(), 1e-300), (name, err)


@pytest.mark.parametrize("entry", ["mean_var", "var", "var_diag"])
def test_prior_only_parameter_keeps_its_gradient(entry):
    """f = f1 + f2 with f2 = GP(theta * Matern52()) independent of f1, conditioned on f1 alone: theta reaches the posterior
    covariance of f only through the prior k_ij, and its gradient must survive."""
    import stheno_b200 as S
    from stheno_b200 import matrix as M

    S.B.epsilon = 1e-10
    g = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn(90, 2, dtype=torch.float64, device="cuda", generator=g)
    xs = torch.randn(40, 2, dtype=torch.float64, device="cuda", generator=g)
    y = torch.sin(x.sum(-1))
    Gc = torch.randn(40, 40, dtype=torch.float64, device="cuda", generator=g)

    def m52(a, b):
        d2 = ((a[:, None] - b[None]) ** 2).sum(-1)
        s = math.sqrt(5.0) * torch.sqrt(torch.clamp_min(d2, 1e-30))
        return (1 + s + 5.0 / 3.0 * d2) * torch.exp(-s)

    theta = torch.tensor(0.7, dtype=torch.float64, device="cuda", requires_grad=True)
    meas = S.Measure()
    f1 = S.GP(S.EQ(), measure=meas)
    f2 = S.GP(theta * S.Matern52(), measure=meas)
    f = f1 + f2
    post = (f | (f1(x, 0.1), y))(xs)
    if entry == "mean_var":
        _, v = post.mean_var
        loss = (Gc * M.dense(v)).sum()
    elif entry == "var":
        loss = (Gc * M.dense(post.var)).sum()
    else:
        loss = (Gc.diagonal() * post.var_diag).sum()
    loss.backward()
    want = (Gc * m52(xs, xs)).sum() if entry != "var_diag" else Gc.diagonal().sum()
    assert abs(theta.grad.item() - want.item()) <= 1e-10 * max(1.0, abs(want.item()))


@pytest.mark.parametrize("n,batch", [(3000, 1), (1500, 2)])
def test_solve_many_rows_t(n, batch):
    """The recursive backward solve of the posterior's chunks against a dense triangular solve: X L = B."""
    from stheno_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(n)
    A = torch.randn(batch, n, n, dtype=torch.float64, device="cuda", generator=g) / math.sqrt(n)
    K = A @ A.transpose(1, 2) + torch.eye(n, dtype=torch.float64, device="cuda")
    ch = ops.chol_from_dense(K)
    B = torch.randn(batch, 300, n, dtype=torch.float64, device="cuda", generator=g)
    buf = ch.new_rows(300)
    buf[:, :300, :n] = B
    ch.solve_many_rows_t_(buf, leaf=512, panel=384)
    L = torch.linalg.cholesky(K)
    want = torch.linalg.solve_triangular(L, B, upper=False, left=False)
    assert (buf[:, :300, :n] - want).abs().max().item() <= 1e-10 * want.abs().max().item()
    assert buf[:, 300:].abs().max().item() == 0.0
