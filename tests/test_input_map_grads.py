"""Gradients through input-mapped kernels (``periodic``, ``shift``, ``stretch``, ``select``, ``transform``) on the analytic
routes: exact posterior predictions (``autograd.exact_posterior``) and the single-process sparse ELBO (``autograd.sparse_elbo``).
Both see a mapped kernel as its inner flat kernel at mapped points (``kernels.k1_block`` with ``through_maps=True``); torch
chains the gradients of the mapped points through the maps.

The host tests check the resolver, the grad detection and the refusals on the CPU stand-in backend; the GPU tests compare
gradients with torch fp64 autograd of dense restatements that write each map in torch."""
import math

import numpy as np
import pytest
import torch

from stheno_b200.generic_grad import kernel_diag_torch, kernel_torch, sparse_compute_torch

METHODS = ["vfe", "fitc", "dtc"]
TWO_PI = 2 * math.pi


@pytest.fixture
def SB(monkeypatch):
    """The library on the CPU stand-in backend."""
    import stheno_b200 as s
    from tests import _cpu_backend

    _cpu_backend.install(monkeypatch)
    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.Measure, "default", None)
    return s


@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.Measure, "default", None)
    return s


def _leaf(v):
    return torch.tensor(v, dtype=torch.float64, requires_grad=True)


def _periodic(t, p):
    ang = t * TWO_PI / p
    return torch.cat([torch.sin(ang), torch.cos(ang)], dim=-1)


# ---- host: the resolver ---------------------------------------------------------------------------------------------------
def _resolve(k, *args):
    from stheno_b200.kernels import k1_block

    return k1_block(k, *args, through_maps=True)


def test_k1_block_each_map_kind(SB):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(9, 3, dtype=torch.float64, generator=g)
    y = torch.randn(5, 3, dtype=torch.float64, generator=g)
    p, c, ell = _leaf(1.7), _leaf([0.2, -0.1, 0.4]), _leaf(0.8)
    W = torch.randn(3, 4, dtype=torch.float64, generator=g).requires_grad_()
    net = lambda t: torch.tanh(t @ W)
    inner = 1.3 * SB.EQ().stretch(ell)
    cases = [
        (inner.periodic(p), lambda t: _periodic(t, p)),
        (inner.shift(c), lambda t: t - c),
        (inner.select((0, 2)), lambda t: t[:, [0, 2]]),
        (inner.transform(net), net),
        (inner.periodic(p).shift(c).select((2, 1, 0)), lambda t: _periodic(t[:, [2, 1, 0]] - c, p)),
        (inner.periodic(p).transform(net).shift(c), lambda t: _periodic(net(t - c), p)),
    ]
    for k, fmap in cases:
        for args in ((x,), (x, y)):
            res = _resolve(k, *args)
            assert res is not None, k
            flat, scales, xm, ym = res
            want_flat, want_scales = inner._flat()
            assert flat.terms == want_flat.terms and scales[0] is want_scales[0] is ell
            assert torch.equal(xm.t, fmap(x))
            assert (ym is xm) if len(args) == 1 else torch.equal(ym.t, fmap(y))
            assert xm.t.requires_grad == fmap(x).requires_grad  # the graph to the map's parameters
    # per-argument maps: the cross kernel resolves, the square one (two different maps at one link) does not
    k2 = inner.shift(c, None)
    flat, _, xm, ym = _resolve(k2, x, y)
    assert torch.equal(xm.t, x - c) and torch.equal(ym.t, y)
    assert _resolve(k2, x) is None
    s2 = SB.EQ().stretch(2.0, 0.5)
    _, _, xm, ym = _resolve(s2, x, y)
    assert torch.equal(xm.t, x / 2.0) and torch.equal(ym.t, y / 0.5)


def test_k1_block_plain_and_non_resolving(SB):
    from stheno_b200.kernels import Input

    x = torch.randn(6, 1, dtype=torch.float64)
    k = SB.Matern52().stretch(0.7) + 0.3 * SB.EQ()
    flat, scales, xm, ym = _resolve(k, x)
    assert isinstance(xm, Input) and xm.t is not None and ym is xm and torch.equal(xm.t, x)
    for bad in (SB.EQ().periodic(1.0) + SB.EQ(), SB.EQ().periodic(1.0) * SB.EQ().shift(0.5),
                2.0 * SB.EQ().periodic(1.0), SB.EQ().diff(0)):
        assert _resolve(bad, x) is None and _resolve(bad, x, x + 1) is None


# ---- host: grad detection -------------------------------------------------------------------------------------------------
def _exact_problem(SB, kernel, n=30, m=7):
    g = torch.Generator().manual_seed(3)
    x = torch.rand(n, 1, dtype=torch.float64, generator=g) * 4
    xs = torch.rand(m, 1, dtype=torch.float64, generator=g) * 4
    y = torch.sin(3 * x[:, 0])
    f = SB.GP(kernel)
    return f | (f(x, 0.1), y), xs


@pytest.mark.parametrize("which", ["period", "shift", "transform"])
def test_prediction_grads_see_through_maps(SB, which):
    """A tensor period, a tensor shift and a transform whose output requires grad (the network's weights live in its
    closure) each make the exact posterior take the analytic route and the sparse problem want a gradient."""
    from stheno_b200 import kernels

    t = _leaf(1.3)
    W = _leaf([[0.7]])
    k = {"period": SB.EQ().periodic(t), "shift": SB.EQ().shift(t), "transform": SB.EQ().transform(lambda u: u @ W)}[which]
    post, xs = _exact_problem(SB, k)
    xi = kernels.as_input(xs)
    assert kernels._exact_args(post.mean, xi) is not None and kernels._prediction_grads(post.mean, xi)
    with torch.no_grad():
        assert not kernels._prediction_grads(post.mean, xi)

    f = SB.GP(k)
    z = torch.linspace(0, 4, 5, dtype=torch.float64)[:, None]
    x = torch.rand(20, 1, dtype=torch.float64)
    obs = SB.PseudoObs(f(z), f(x, 0.1), torch.sin(x[:, 0]))
    assert obs._wants_grad(f.measure) and obs._mapped(f.measure)
    W.requires_grad_(False)
    t.requires_grad_(False)
    assert not obs._wants_grad(f.measure)


def test_exact_args_refuse_sums_of_differently_mapped_kernels(SB):
    from stheno_b200 import kernels

    p = _leaf(1.3)
    post, xs = _exact_problem(SB, SB.EQ().periodic(p) + SB.EQ())
    xi = kernels.as_input(xs)
    assert kernels._exact_args(post.mean, xi) is None and kernels._prediction_grads(post.mean, xi)
    mean, var = post(xs).marginals()
    with pytest.raises(NotImplementedError):
        mean.sum().backward()


# ---- host: the uncovered sparse route keeps its values and refuses backward ----------------------------------------------
@pytest.mark.parametrize("kernel", ["resolving", "sum"])
def test_sparse_mapped_values_and_refusal_on_host(SB, kernel):
    """On the stand-in (no analytic route off the GPU) the ELBO, mu, A and K_z under grad are the no-grad values bit for
    bit, and ``backward()`` through any of them raises: never a partial gradient."""
    g = torch.Generator().manual_seed(4)
    x = torch.rand(50, 1, dtype=torch.float64, generator=g) * 4
    z = torch.linspace(0, 4, 6, dtype=torch.float64)[:, None]
    y = torch.sin(x[:, 0])

    def run(grad):
        ell = torch.tensor(0.9, dtype=torch.float64, requires_grad=grad)
        k = SB.EQ().stretch(ell).periodic(2.0)
        if kernel == "sum":
            k = k + SB.Matern32()
        f = SB.GP(k)
        obs = SB.PseudoObs(f(z), f(x, 0.1), y)
        return obs.elbo(f.measure), obs.mu(f.measure), SB.B.dense(obs.A(f.measure)), SB.B.dense(obs.K_z(f.measure))

    with torch.no_grad():
        want = run(False)
    got = run(True)
    for a, b in zip(got, want):
        assert a.requires_grad and torch.equal(a.detach(), b)
        with pytest.raises(NotImplementedError):
            a.sum().backward()


# ---- GPU: exact posterior predictions -------------------------------------------------------------------------------------
def _mlp(T, d):
    W1, b1, W2 = T(np.linspace(-1, 1, d * 6).reshape(d, 6)), T(np.linspace(-0.3, 0.3, 6)), T(np.linspace(0.8, -0.6, 12).reshape(6, 2))
    return lambda t: torch.tanh(t @ W1 + b1) @ W2


def _mapped_case(S, name, T, d):
    """``(kernel, inner, map)``: the library's kernel, the flat kernel inside its maps and the map written in torch."""
    v, ell = T(1.3), T(0.8)
    if name == "periodic":
        p = T(1.7)
        inner = v * S.EQ().stretch(ell)
        return inner.periodic(p), inner, lambda t: _periodic(t, p)
    if name == "shift":
        c = T([0.3, -0.2, 0.5][:d])
        inner = v * S.Matern52().stretch(ell)
        return inner.shift(c), inner, lambda t: t - c
    if name == "select":
        ell2 = T([0.7, 1.3])
        inner = v * S.EQ().stretch(ell2)
        return inner.select((2, 0)), inner, lambda t: t[:, [2, 0]]
    if name == "transform":
        net = _mlp(T, d)
        inner = v * S.EQ().stretch(ell)
        return inner.transform(net), inner, net
    raise ValueError(name)


def _exact_setup(S, name, n, m, d=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    params = []

    def T(v):
        t = torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True)
        params.append(t)
        return t

    k, inner, fmap = _mapped_case(S, name, T, d)
    noise = T(0.05)
    x = T(torch.rand(n, d, dtype=torch.float64, generator=g).numpy() * 3)
    xs = T(torch.rand(m, d, dtype=torch.float64, generator=g).numpy() * 3)
    y = T(torch.sin(2 * x.detach().cpu().sum(-1)).numpy())
    return k, inner, fmap, noise, x, xs, y, params


def _exact_reference(inner, fmap, noise, x, xs, y, eps):
    """Mean, marginal variances and covariance of the posterior at ``xs`` in fp64 torch."""
    xm, xsm = fmap(x), fmap(xs)
    n = x.shape[0]
    K = kernel_torch(inner, xm, xm) + (noise + eps) * torch.eye(n, dtype=x.dtype, device=x.device)
    L = torch.linalg.cholesky(K)
    Ks = kernel_torch(inner, xsm, xm)
    V = torch.linalg.solve_triangular(L, Ks.T, upper=False)  # L^-1 K*^T
    h = torch.linalg.solve_triangular(L, y[:, None], upper=False)
    mean = (V.T @ h)[:, 0]
    var_diag = kernel_diag_torch(inner, xsm) - (V * V).sum(0)
    cov = kernel_torch(inner, xsm, xsm) - V.T @ V
    return mean, var_diag, cov


def _losses(wm, wv, G):
    return {
        "mean": lambda mean, var_diag, cov: (wm * mean).sum(),
        "var_diag": lambda mean, var_diag, cov: (wv * var_diag).sum(),
        "bounds": lambda mean, var_diag, cov: (mean + 2 * var_diag.sqrt()).sum(),
        "var": lambda mean, var_diag, cov: (G * cov).sum(),
        "mean_var": lambda mean, var_diag, cov: (wm * mean).sum() + (G * cov).sum(),
    }


def _library_loss(post, xs, name, fn):
    fdd = post(xs)
    if name == "mean":
        return fn(fdd.mean.reshape(-1), None, None)
    if name == "var_diag":
        return fn(None, fdd.var_diag.reshape(-1), None)
    if name == "bounds":
        mean, var = fdd.marginals()
        return fn(mean, var, None)
    if name == "var":
        return fn(None, None, S_dense(fdd.var))
    mean, var = fdd.mean_var
    return fn(mean.reshape(-1), None, S_dense(var))


def S_dense(a):
    from stheno_b200 import matrix as M

    return M.dense(a)


EXACT_CASES = [(name, n) for name in ("periodic", "shift", "select", "transform") for n in (300, 2500)]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
@pytest.mark.parametrize("name,n", EXACT_CASES)
def test_exact_posterior_gradients(S, monkeypatch, name, n, precision):
    """Gradients of the mean, marginal variances, ``mean + 2 sd``, the covariance and ``mean_var`` w.r.t. the variance, the
    length scales, the map's parameters (period, shift, the network's weights), the noise, ``x``, ``x*`` and ``y``, to 1e-8
    of the largest reference gradient.  At n = 2500 under "auto" / "int8x8" the solves run on the int8-slice emulation."""
    from stheno_b200 import ops

    monkeypatch.setattr(S.B, "precision", precision)
    m = 1000 if n == 2500 else 60
    k, inner, fmap, noise, x, xs, y, params = _exact_setup(S, name, n, m, seed=n)
    g = torch.Generator(device="cuda").manual_seed(1)
    wm = torch.randn(m, dtype=torch.float64, device="cuda", generator=g)
    wv = torch.randn(m, dtype=torch.float64, device="cuda", generator=g)
    G = torch.randn(m, m, dtype=torch.float64, device="cuda", generator=g) / m
    mean, var_diag, cov = _exact_reference(inner, fmap, noise, x, xs, y, S.B.epsilon)
    for lname, fn in _losses(wm, wv, G).items():
        want = torch.autograd.grad(fn(mean, var_diag, cov), params, retain_graph=True, allow_unused=True)
        f = S.GP(k)
        post = f | (f(x, noise), y)
        ops.gemm_profile(True)
        try:
            loss = _library_loss(post, xs, lname, fn)
            got = torch.autograd.grad(loss, params, allow_unused=True)
            emulated = ops.gemm_profile_read(1)[2]
        finally:
            ops.gemm_profile(False)
        if n == 2500:
            assert (emulated > 0) == (precision != "fp64"), (lname, precision, emulated)
        for i, (a, w) in enumerate(zip(got, want)):
            a = torch.zeros_like(params[i]) if a is None else a
            w = torch.zeros_like(params[i]) if w is None else w
            err = float((a - w).abs().max()) / max(1.0, float(w.abs().max()))
            assert err <= 1e-8, (lname, i, err)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["periodic", "transform"])
def test_exact_posterior_values_bit_identical_under_grad(S, name):
    k, inner, fmap, noise, x, xs, y, params = _exact_setup(S, name, 400, 50)
    f = S.GP(k)
    post = f | (f(x, noise), y)
    with torch.no_grad():
        m0, v0 = post(xs).marginals()
        mv0 = post(xs).mean_var
    m1, v1 = post(xs).marginals()
    mv1 = post(xs).mean_var
    assert m1.requires_grad and v1.requires_grad
    assert torch.equal(m0, m1.detach()) and torch.equal(v0, v1.detach())
    assert torch.equal(mv0[0], mv1[0].detach()) and torch.equal(S_dense(mv0[1]), S_dense(mv1[1]).detach())


@pytest.mark.gpu
def test_exact_posterior_non_resolving_refuses(S):
    p = torch.tensor(1.5, dtype=torch.float64, device="cuda", requires_grad=True)
    x = torch.rand(80, 1, dtype=torch.float64, device="cuda") * 4
    xs = torch.rand(10, 1, dtype=torch.float64, device="cuda") * 4
    f = S.GP(S.EQ().periodic(p) + S.Matern32())
    post = f | (f(x, 0.1), torch.sin(x[:, 0]))
    with torch.no_grad():
        want = post(xs).marginals()
    got = post(xs).marginals()
    for a, b in zip(got, want):
        assert torch.equal(a.detach(), b)
        with pytest.raises(NotImplementedError):
            a.sum().backward()


# ---- GPU: the single-process sparse ELBO ----------------------------------------------------------------------------------
def _sparse_case(S, name, T, d):
    v, ell = T(1.2), T(0.9)
    inner = v * S.Matern52().stretch(ell) if name == "shift" else v * S.EQ().stretch(ell)
    if name == "periodic":
        p = T(1.9)
        return inner.periodic(p), inner, lambda t: _periodic(t, p)
    if name == "shift":
        c = T(list(np.linspace(-0.3, 0.4, d)))
        return inner.shift(c), inner, lambda t: t - c
    net = _mlp(T, d)
    return inner.transform(net), inner, net


def _sparse_problem(S, method, name, n, m, d, seed=0):
    g = torch.Generator().manual_seed(seed)
    params = []

    def T(v):
        t = torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True)
        params.append(t)
        return t

    def leaf(t):
        t = t.to(device="cuda", dtype=torch.float64).requires_grad_()
        params.append(t)
        return t

    k, inner, fmap = _sparse_case(S, name, T, d)
    x = leaf(torch.rand(n, d, dtype=torch.float64, generator=g) * 3)
    z = leaf(torch.rand(m, d, dtype=torch.float64, generator=g) * 3)
    y = leaf(torch.sin(2 * x.detach().cpu().sum(-1)) + 0.3 * torch.randn(n, dtype=torch.float64, generator=g))
    sig = leaf(0.05 + 0.1 * torch.rand(n, dtype=torch.float64, generator=g))
    nz = leaf(1e-3 + 1e-3 * torch.rand(m, dtype=torch.float64, generator=g))
    cls = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[method]

    def elbo_fn():
        f = S.GP(k)
        return cls(f(z, nz), f(x, sig), y).elbo(f.measure)

    def ref_fn():
        return sparse_compute_torch(method, inner, inner, inner, fmap(z), fmap(x), sig, nz, y[:, None],
                                    torch.zeros(m, 1, dtype=torch.float64, device="cuda"), S.B.epsilon)[3]

    return elbo_fn, ref_fn, params


SPARSE_SHAPES = {"700x37_c96": (700, 37, 3, 96), "3000x300": (3000, 300, 8, None)}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SPARSE_SHAPES))
@pytest.mark.parametrize("name", ["periodic", "shift", "transform"])
@pytest.mark.parametrize("method", METHODS)
def test_sparse_elbo_gradients(S, monkeypatch, method, name, shape):
    n, m, d, chunk = SPARSE_SHAPES[shape]
    if chunk:
        monkeypatch.setattr(S.B, "sparse_chunk", chunk)
    elbo_fn, ref_fn, params = _sparse_problem(S, method, name, n, m, d, seed=n + m)
    ref = ref_fn()
    want = torch.autograd.grad(ref, params, allow_unused=True)
    e = elbo_fn()
    assert e.requires_grad
    got = torch.autograd.grad(e, params, allow_unused=True)
    assert abs(float(e) - float(ref)) <= 1e-10 * max(1.0, abs(float(ref))), (float(e), float(ref))
    errs = []
    for p, a, w in zip(params, got, want):
        a = torch.zeros_like(p) if a is None else a
        w = torch.zeros_like(p) if w is None else w
        errs.append(float((a - w).abs().max()) / max(1.0, float(w.abs().max())))
    print(f"\n{method} {name} {shape}: max gradient error {max(errs):.2e}")
    assert max(errs) <= 1e-8, errs


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_sparse_elbo_value_under_grad_equals_no_grad(S, monkeypatch, method):
    monkeypatch.setattr(S.B, "sparse_chunk", 96)
    for name in ("periodic", "transform"):
        elbo_fn, _, _ = _sparse_problem(S, method, name, 700, 37, 3)
        e = elbo_fn()
        with torch.no_grad():
            e0 = elbo_fn()
        assert e.requires_grad and torch.equal(e.detach(), e0), (name, float(e), float(e0))


@pytest.mark.gpu
def test_sparse_mapped_predictions_and_non_resolving_refuse(S):
    """With a covered ELBO, mu and A keep the no-grad values and refuse backward; a sum of differently mapped kernels
    refuses for the ELBO too, with its no-grad value."""
    g = torch.Generator(device="cuda").manual_seed(8)
    x = torch.rand(400, 1, dtype=torch.float64, device="cuda", generator=g) * 6
    z = torch.linspace(0, 6, 15, dtype=torch.float64, device="cuda")[:, None]
    y = torch.sin(x[:, 0])

    def run(sum_kernel, grad):
        ell = torch.tensor(0.8, dtype=torch.float64, device="cuda", requires_grad=grad)
        k = S.EQ().stretch(ell).periodic(TWO_PI)
        f = S.GP(k + S.Matern32() if sum_kernel else k)
        obs = S.PseudoObs(f(z), f(x, 0.1), y)
        e = obs.elbo(f.measure)
        return e, obs.mu(f.measure), S_dense(obs.A(f.measure)), (f | obs)(x[:7]).marginals()[0]

    for sum_kernel in (False, True):
        with torch.no_grad():
            want = run(sum_kernel, False)
        got = run(sum_kernel, True)
        for i, (a, b) in enumerate(zip(got, want)):
            assert a.requires_grad
            if i < 3:
                assert torch.equal(a.detach(), b), (sum_kernel, i)
            else:
                assert torch.allclose(a.detach(), b, rtol=1e-9, atol=1e-12)
            if i == 0 and not sum_kernel:
                continue  # the covered ELBO
            with pytest.raises(NotImplementedError):
                a.sum().backward(retain_graph=True)
        if not sum_kernel:
            got[0].backward()


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_only_hyperparameters_inside_the_map_require_grad(S, method):
    """Only the variance and length scale inside ``periodic`` require grad (the noise is a float): nothing outside the map
    asks for a gradient, yet the ELBO's gradient is the whole one."""
    g = torch.Generator().manual_seed(12)
    x = (torch.rand(900, 1, dtype=torch.float64, generator=g) * 7).cuda()
    z = torch.linspace(0, 10, 25, dtype=torch.float64, device="cuda")[:, None]
    y = torch.sin(x[:, 0]) + 0.5 * torch.randn(900, dtype=torch.float64, generator=g).cuda()
    v, ell = (torch.tensor(t, dtype=torch.float64, device="cuda", requires_grad=True) for t in (1.4, 0.8))
    inner = v * S.EQ().stretch(ell)
    f = S.GP(inner.periodic(TWO_PI))
    cls = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[method]
    got = torch.autograd.grad(cls(f(z), f(x, 0.3), y).elbo(f.measure), [v, ell])
    ref = sparse_compute_torch(method, inner, inner, inner, _periodic(z, TWO_PI), _periodic(x, TWO_PI),
                               torch.full((900,), 0.3, dtype=torch.float64, device="cuda"), None, y[:, None],
                               torch.zeros(25, 1, dtype=torch.float64, device="cuda"), S.B.epsilon)[3]
    want = torch.autograd.grad(ref, [v, ell])
    for a, w in zip(got, want):
        assert float((a - w).abs()) <= 1e-8 * max(1.0, float(w.abs())), (method, float(a), float(w))


@pytest.mark.gpu
def test_readme_example_10_against_central_differences(S):
    """The reference README's sparse example: ``EQ().periodic(2 pi)`` (here with a learnable variance and length scale inside
    the map and a learnable noise), n = 50000 observations in 1-D, m = 20 inducing points, VFE / FITC / DTC.  The gradient
    in (variance, length scale, noise) along three random directions against central differences of the ELBO.  The ELBO is
    about 5e4 in size, so the differences carry a rounding error of about 1e-13 |ELBO| / h: the point is away from the
    optimum, where the directional derivatives are large against that."""
    g = torch.Generator(device="cuda").manual_seed(10)
    n, m = 50000, 20
    x = torch.linspace(0, 7, n, dtype=torch.float64, device="cuda")
    z = torch.linspace(0, 10, m, dtype=torch.float64, device="cuda")
    y = torch.sin(x) + math.sqrt(0.5) * torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    p0 = torch.tensor([2.0, 1.0, 0.2], dtype=torch.float64, device="cuda")
    for method in METHODS:
        cls = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[method]

        def elbo(p):
            f = S.GP((p[0] * S.EQ().stretch(p[1])).periodic(2 * S.B.pi))
            return cls(f(z), f(x, p[2]), y).elbo(f.measure)

        p = p0.clone().requires_grad_()
        (gp,) = torch.autograd.grad(elbo(p), [p])
        gen = torch.Generator(device="cuda").manual_seed(11)
        for _ in range(3):
            dp = torch.randn(3, dtype=torch.float64, device="cuda", generator=gen) * p0
            ana = float((gp * dp).sum())
            h = 1e-4
            with torch.no_grad():
                fd = float(elbo(p0 + h * dp) - elbo(p0 - h * dp)) / (2 * h)
            print(f"\n{method}: analytic {ana:.12e} fd {fd:.12e} rel {abs(fd - ana) / abs(ana):.2e}")
            assert abs(fd - ana) <= 1e-6 * abs(ana), (method, ana, fd)
