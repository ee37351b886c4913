"""Gradients of pathwise function samples (``FunctionSample.__call__``) in their evaluation points, and the feature kernel's
backward (``gpk_feature_eval_bwd``, ``csrc/sample_fn.cu``).

* the kernel against its closed form in fp64 over row / feature / sample / dimension counts around its tile edges, at phases
  up to 16384, in write and accumulate mode; NaN rows; run-to-run bit equality;
* the gradient of ``sum g * f_s(x*)`` against torch fp64 autograd of the pathwise identity restated from the draws the
  sample holds (``tests/test_sample_function.restate``), for priors and posteriors, one sample (the factored update
  backward) and several, across chunks, under emulated solves and in fp32;
* the contract: the evaluation points get a gradient, nothing else does, and a backward that would reach anything else raises;
* central differences of the same sample at n = 16384, a Thompson maximisation with L-BFGS, memory at 2^20 points.

The host cases run the model layer on the torch-CPU stand-ins of ``tests/_cpu_backend.py`` with torch restatements of the
feature kernel, its backward and the rectangular K1-backward; the ``gpu`` cases run the CUDA kernels."""
import types

import numpy as np
import pytest
import torch

from tests.test_sample_function import cases, dyadic_inputs, feat_ref, restate

U32 = 2.0**-24


def feat_bwd_ref(x, omega, b, amp, W, G):
    """The feature kernel's backward in fp64: ``-(c o sin(x omega^T + b)) omega`` with ``c = (G W) o amp``, and the sum of
    |terms| per element, ``sum_j a_j |omega_je| sum_s |G_is W_sj|``."""
    x, omega, b, amp, W, G = [t.to(torch.float64) for t in (x, omega, b, amp, W, G)]
    c = (G @ W) * amp
    grad = -(c * torch.sin(x @ omega.T + b)) @ omega
    mag = ((G.abs() @ W.abs()) * amp) @ omega.abs()
    return grad, mag


@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.B, "precision", "auto")
    monkeypatch.setattr(s.Measure, "default", None)
    return s


@pytest.fixture
def host(cpu_backend, monkeypatch):
    """The CPU stand-ins, with the feature kernel, its backward and the rectangular K1-backward restated in torch."""
    from stheno_b200 import autograd, pathwise

    def feature_eval(x, omega, b, amp, W, out=None):
        v = feat_ref(x, omega, b, amp, W)[0].to(x.dtype)
        if out is None:
            return v
        out += v
        return out

    def feature_eval_bwd(x, omega, b, amp, W, G, out=None):
        v = feat_bwd_ref(x, omega, b, amp, W, G)[0].to(x.dtype)
        if out is None:
            return v
        out += v
        return out

    def kernel_cross_bwd(flat, xsg, xg, *, W=None, r=None, u=None, v=None, grad_xsg=None, **unused):
        assert r is None and not any(t is not None for t in unused.values())
        m, n = xsg.shape[2], xg.shape[2]
        G = torch.zeros(xsg.shape[1], m, n, dtype=xsg.dtype)
        if W is not None:
            G += W[:, :m, :n]
        if u is not None:
            G += u[:, :, None] * v[:, None, :]
        with torch.enable_grad():
            xs = xsg.detach().clone().requires_grad_()
            K = cpu_backend._eval(flat, xs, xg.detach(), False)
            grad_xsg += torch.autograd.grad((K * G).sum(), xs)[0]

    stand_in = types.SimpleNamespace(**{k: getattr(cpu_backend, k) for k in dir(cpu_backend) if not k.startswith("__")})
    stand_in.feature_eval, stand_in.feature_eval_bwd, stand_in.kernel_cross_bwd = feature_eval, feature_eval_bwd, \
        kernel_cross_bwd
    monkeypatch.setattr(pathwise, "ops", stand_in)
    monkeypatch.setattr(autograd, "ops", stand_in)
    return cpu_backend


# ---- the gradient against torch fp64 autograd of the restated identity ------------------------------------------------------
def grad_case(S, case, n, m, dtype, dev, num, posterior=True, features=512, seed=0, chunk=2048):
    """``(got, want, cond, values under grad, values without grad)`` for ``sum g * f_s(x*)`` with a random upstream ``g``."""
    name, k, kfun, pmap, mean, mfun, noise_kind = case
    rng = np.random.default_rng(seed)
    d = 3
    X = torch.as_tensor(rng.uniform(-2, 2, (n, d)))
    xs = torch.as_tensor(rng.uniform(-2.5, 2.5, (m, d)))
    y = torch.as_tensor(rng.standard_normal(n))
    g = torch.as_tensor(rng.standard_normal((m, num)))
    noise = torch.full((n,), 0.1, dtype=torch.float64) if noise_kind == "scalar" else \
        torch.as_tensor(rng.uniform(0.05, 0.3, n))
    f = S.GP(mean, k)
    if posterior:
        nz = 0.1 if noise_kind == "scalar" else noise.to(dev, dtype)
        f = f | (f(X.to(dev, dtype), nz), y.to(dev, dtype))
    from stheno_b200.pathwise import FunctionSample

    fs = FunctionSample(f, num=num, features=features, state=torch.Generator().manual_seed(seed), chunk=chunk)
    x = xs.to(dev, dtype).requires_grad_()
    v = fs(x)
    (got,) = torch.autograd.grad((v * g.to(dev, dtype)).sum(), x)
    with torch.no_grad():
        plain = fs(xs.to(dev, dtype))
    xr = xs.clone().requires_grad_()
    if posterior:
        want, cond = restate(fs, kfun, pmap, mfun, xr, X, y, noise, S.B.epsilon)
    else:
        want, cond = restate(fs, kfun, pmap, mfun, xr), 1.0
    (want_g,) = torch.autograd.grad((want * g).sum(), xr)
    return got.detach().cpu().to(torch.float64), want_g, cond, v.detach(), plain


@pytest.mark.parametrize("which", [0, 1, 2])
@pytest.mark.parametrize("posterior", [False, True])
@pytest.mark.parametrize("num", [1, 3])
def test_grad_host(S, host, which, posterior, num):
    got, want, _, v, plain = grad_case(S, cases(S)[which], 150, 40, torch.float64, "cpu", num, posterior, chunk=16)
    assert (got - want).abs().max() <= 1e-10 * max(1.0, want.abs().max().item())
    assert torch.equal(v, plain)


# ---- the contract: the evaluation points only ---------------------------------------------------------------------------------
def contract_models(S, dev):
    """``(name, build(detached) -> GP)``: a learnable length scale, a mean parameter, observations requiring grad and a
    transform whose closure holds a parameter.  ``build(True)`` is the same model with every such tensor detached."""
    rng = np.random.default_rng(3)
    X = torch.as_tensor(rng.uniform(-2, 2, (60, 2)), device=dev)
    y = torch.as_tensor(rng.standard_normal(60), device=dev)
    ell = torch.tensor(0.9, dtype=torch.float64, device=dev, requires_grad=True)
    a = torch.tensor(0.4, dtype=torch.float64, device=dev, requires_grad=True)
    yg = y.clone().requires_grad_()
    w = torch.tensor([1.3, 0.7], dtype=torch.float64, device=dev, requires_grad=True)

    def post(f, yy):
        return f | (f(X, 0.1), yy)

    def dt(t, detached):
        return t.detach() if detached else t

    return [
        ("length scale", lambda de: post(S.GP(S.EQ().stretch(dt(ell, de))), y)),
        ("mean parameter", lambda de: post(S.GP(lambda x: dt(a, de) * x[:, :1], S.EQ()), y)),
        ("observations", lambda de: post(S.GP(S.Matern52().stretch(1.2)), dt(yg, de))),
        ("transform", lambda de: post(S.GP(S.EQ().transform(lambda x: x * dt(w, de))), y)),
    ]


def check_contract(S, dev):
    xs0 = torch.as_tensor(np.random.default_rng(4).uniform(-2.5, 2.5, (70, 2)), device=dev)
    g = torch.as_tensor(np.random.default_rng(5).standard_normal((70, 3)), device=dev)
    for name, build in contract_models(S, dev):
        fs = build(False).sample_function(num=3, features=256, state=torch.Generator().manual_seed(7))
        ref = build(True).sample_function(num=3, features=256, state=torch.Generator().manual_seed(7))
        x = xs0.clone().requires_grad_()
        loss = (fs(x) * g).sum()
        (got,) = torch.autograd.grad(loss, x, retain_graph=True)
        x2 = xs0.clone().requires_grad_()
        (want,) = torch.autograd.grad((ref(x2) * g).sum(), x2)
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12 * want.abs().max().item()), name
        loss.backward(inputs=[x], retain_graph=True)
        assert torch.allclose(x.grad, got, rtol=1e-13, atol=1e-13 * got.abs().max().item()), name
        with pytest.raises(NotImplementedError, match="function sampling"):
            loss.backward()


def parameter_free_transform(S, dev):
    """A transform without parameters is differentiated through: the gradient of ``sum g * f_s`` against torch fp64 autograd of
    the restated identity of the mapped kernel."""
    rng = np.random.default_rng(8)
    X = torch.as_tensor(rng.uniform(-2, 2, (80, 2)))
    y = torch.as_tensor(rng.standard_normal(80))
    xs = torch.as_tensor(rng.uniform(-2.5, 2.5, (50, 2)))
    g = torch.as_tensor(rng.standard_normal((50, 2)))
    tf = lambda x: torch.cat([torch.sin(x), x**2], -1)  # noqa: E731
    f = S.GP((0.7 * S.EQ().stretch(1.1)).transform(tf))
    fs = (f | (f(X.to(dev), 0.1), y.to(dev))).sample_function(num=2, features=256, state=torch.Generator().manual_seed(1))
    x = xs.to(dev).requires_grad_()
    (got,) = torch.autograd.grad((fs(x) * g.to(dev)).sum(), x)
    xr = xs.clone().requires_grad_()
    kfun = lambda a, b: 0.7 * torch.exp(-((a[:, None] - b[None]) ** 2).sum(-1) / (2 * 1.1**2))  # noqa: E731
    want, _ = restate(fs, kfun, tf, lambda x: 0 * x[:, :1], xr, X, y, torch.full((80,), 0.1, dtype=torch.float64),
                      S.B.epsilon)
    (want_g,) = torch.autograd.grad((want * g).sum(), xr)
    assert (got.cpu() - want_g).abs().max() <= 1e-10 * max(1.0, want_g.abs().max().item())


def linear_only(S, dev):
    """``F = 0``: a kernel of ``Linear`` terms only has no features; the gradient is the linear part's and the update's."""
    rng = np.random.default_rng(9)
    X = torch.as_tensor(rng.uniform(-2, 2, (40, 2)))
    y = torch.as_tensor(rng.standard_normal(40))
    xs = torch.as_tensor(rng.uniform(-2, 2, (30, 2)))
    f = S.GP(0.5 * S.Linear().stretch(2.0))
    fs = (f | (f(X.to(dev), 0.2), y.to(dev))).sample_function(num=2, state=torch.Generator().manual_seed(2))
    x = xs.to(dev).requires_grad_()
    (got,) = torch.autograd.grad(fs(x).sum(), x)
    assert fs.omega.shape[0] == 0
    xr = xs.clone().requires_grad_()
    kfun = lambda a, b: 0.5 * (a / 2.0) @ (b / 2.0).T  # noqa: E731
    want, _ = restate(fs, kfun, lambda x: x, lambda x: 0 * x[:, :1], xr, X, y, torch.full((40,), 0.2, dtype=torch.float64),
                      S.B.epsilon)
    (want_g,) = torch.autograd.grad(want.sum(), xr)
    assert (got.cpu() - want_g).abs().max() <= 1e-9 * max(1.0, want_g.abs().max().item())


def test_contract_host(S, host):
    check_contract(S, "cpu")


def test_parameter_free_transform_host(S, host):
    parameter_free_transform(S, "cpu")


def test_linear_only_host(S, host):
    linear_only(S, "cpu")


def test_no_grad_routes_host(S, host, monkeypatch):
    """Without a tensor that requires grad the evaluation takes the no-grad route; with only a hyper-parameter, the value
    raises on ``backward()``; with the points, the differentiable route runs and the feature backward is called once."""
    from stheno_b200 import autograd, pathwise

    calls = []
    real = pathwise.ops.feature_eval_bwd
    monkeypatch.setattr(pathwise.ops, "feature_eval_bwd", lambda *a, **k: calls.append(1) or real(*a, **k))
    fs = S.GP(S.EQ()).sample_function(num=2, features=64, state=torch.Generator().manual_seed(0))
    x = torch.linspace(-1, 1, 9, dtype=torch.float64)[:, None]
    v = fs(x)
    assert not v.requires_grad
    xg = x.clone().requires_grad_()
    spy, real_fs = [], autograd.function_sample
    monkeypatch.setattr(autograd, "function_sample", lambda *a: spy.append(1) or real_fs(*a))
    w = fs(xg)
    assert spy and torch.equal(w.detach(), v)
    w.sum().backward()
    assert calls == [1] and xg.grad is not None


# ---- GPU: the kernel ------------------------------------------------------------------------------------------------------------
GRID = [(n, F, num, d) for n in (1, 127, 128, 129, 5000) for F, num, d in
        ((1, 1, 1), (64, 7, 8), (65, 8, 1), (4096, 33, 8), (65, 33, 8), (4096, 1, 1), (65, 8, 40), (100, 100, 3),
         (33, 1, 40))]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("n,F,num,d", GRID)
def test_feature_bwd_kernel_parity(n, F, num, d, dtype):
    from stheno_b200 import ops

    bound = 1e-13 if dtype == torch.float64 else 2.0**-18
    for big in (False, True):
        x, omega, b, amp, W = dyadic_inputs(n, F, num, d, big, dtype, seed=n + F + num + d)
        G = torch.randn(n, num, dtype=torch.float64, generator=torch.Generator().manual_seed(n + d)).to("cuda", dtype)
        want, mag = feat_bwd_ref(*[t.cpu() for t in (x, omega, b, amp, W, G)])
        got = ops.feature_eval_bwd(x, omega, b, amp, W, G)
        assert got.dtype == dtype and got.shape == (n, d)
        err = ((got.cpu().double() - want).abs() / mag.clamp_min(1e-300)).max().item()
        assert err <= bound, (n, F, num, d, big, err)
        base = torch.randn(n, d, dtype=dtype, device="cuda")
        acc = ops.feature_eval_bwd(x, omega, b, amp, W, G, out=base.clone())
        err = ((acc.cpu().double() - base.cpu().double() - want).abs()
               / (mag + base.cpu().double().abs())).max().item()
        assert err <= bound, (n, F, num, d, big, "accumulate", err)
        assert torch.equal(ops.feature_eval_bwd(x, omega, b, amp, W, G), got)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("num", [3, 16])
@pytest.mark.parametrize("d", [5, 40])
def test_feature_bwd_kernel_nan(dtype, num, d):
    from stheno_b200 import ops

    x, omega, b, amp, W = dyadic_inputs(300, 200, num, d, True, dtype, seed=1)
    G = torch.randn(300, num, dtype=dtype, device="cuda")
    assert torch.isfinite(ops.feature_eval_bwd(x, omega, b, amp, W, G)).all()
    others = torch.ones(300, dtype=torch.bool, device="cuda")
    x[17, 2] = float("nan")
    G[200, num - 1] = float("nan")
    others[17] = others[200] = False
    out = ops.feature_eval_bwd(x, omega, b, amp, W, G)
    assert torch.isnan(out[17]).all() and torch.isnan(out[200]).all()
    assert torch.isfinite(out[others]).all()


@pytest.mark.gpu
def test_feature_bwd_checks():
    from stheno_b200 import ops

    x, omega, b, amp, W = dyadic_inputs(10, 8, 2, 3, False, torch.float64, seed=0)
    G = torch.randn(10, 2, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="shapes"):
        ops.feature_eval_bwd(x, omega, b, amp, W, G[:, :1])
    with pytest.raises(TypeError, match="dtype"):
        ops.feature_eval_bwd(x, omega, b, amp, W, G.float())
    empty = ops.feature_eval_bwd(x, omega[:0], b[:0], amp[:0], W[:, :0], G)
    assert empty.shape == (10, 3) and not empty.any()


# ---- GPU: the gradient against torch fp64 autograd ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1, 2])
@pytest.mark.parametrize("posterior", [False, True])
@pytest.mark.parametrize("num", [1, 9])
def test_grad(S, which, posterior, num):
    got, want, _, v, plain = grad_case(S, cases(S)[which], 2500, 600, torch.float64, "cuda", num, posterior,
                                       features=2048)
    assert (got - want).abs().max() <= 1e-8 * max(1.0, want.abs().max().item())
    assert torch.equal(v, plain)


@pytest.mark.gpu
@pytest.mark.parametrize("num", [1, 9])
def test_grad_chunks(S, num):
    """m = 4100 with the default chunk of 2048: three chunks, the last one ragged."""
    got, want, _, v, plain = grad_case(S, cases(S)[1], 2500, 4100, torch.float64, "cuda", num, features=1024)
    assert (got - want).abs().max() <= 1e-8 * max(1.0, want.abs().max().item())
    assert torch.equal(v, plain)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
def test_grad_emulated(S, monkeypatch, precision):
    """n = 6000: the solves that fix V run on the int8 emulation under ``auto`` and ``int8x8``."""
    monkeypatch.setattr(S.B, "precision", precision)
    got, want, _, v, plain = grad_case(S, cases(S)[0], 6000, 300, torch.float64, "cuda", 4, features=1024)
    assert (got - want).abs().max() <= 1e-8 * max(1.0, want.abs().max().item())
    assert torch.equal(v, plain)


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 2])
@pytest.mark.parametrize("num", [1, 8])
def test_grad_fp32(S, which, num):
    got, want, cond, v, plain = grad_case(S, cases(S)[which], 1500, 300, torch.float32, "cuda", num, features=1024)
    err = (got - want).abs().max().item() / max(1.0, want.abs().max().item())
    assert err <= 16.0 * U32 * cond, (err, cond)
    assert torch.equal(v, plain)


@pytest.mark.gpu
def test_contract(S):
    check_contract(S, "cuda")


@pytest.mark.gpu
def test_parameter_free_transform(S):
    parameter_free_transform(S, "cuda")


@pytest.mark.gpu
def test_linear_only(S):
    linear_only(S, "cuda")


# ---- GPU: at scale -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_central_differences(S):
    """n = 16384, d = 8, ``auto`` precision: directional derivatives of every sample at 256 points against central
    differences of the same sample at h = 1e-5, within 1e-6 of the largest."""
    rng = np.random.default_rng(0)
    n, d, m, num, h = 16384, 8, 256, 4, 1e-5
    X = torch.as_tensor(rng.standard_normal((n, d)), device="cuda")
    y = torch.as_tensor(rng.standard_normal(n), device="cuda")
    f = S.GP(S.EQ().stretch(2.0) + 0.3 * S.Matern52().stretch(3.0))
    fs = (f | (f(X, 0.1), y)).sample_function(num=num, features=2048, state=torch.Generator().manual_seed(0))
    xs = torch.as_tensor(rng.standard_normal((m, d)), device="cuda")
    u = torch.as_tensor(rng.standard_normal((m, d)), device="cuda")
    u /= u.norm(dim=1, keepdim=True)
    x = xs.clone().requires_grad_()
    v = fs(x)
    an = torch.stack([torch.autograd.grad(v[:, s].sum(), x, retain_graph=True)[0] for s in range(num)], 1)  # [m, num, d]
    an = (an * u[:, None, :]).sum(-1)
    with torch.no_grad():
        fd = (fs(xs + h * u) - fs(xs - h * u)) / (2 * h)
    assert (fd - an).abs().max().item() <= 1e-6 * an.abs().max().item()


@pytest.mark.gpu
def test_thompson_maximisation(S):
    """A 1-D posterior, 4 samples, L-BFGS from 32 starts per sample: each sample's best value is at least its maximum over a
    2^16-point grid of the same interval, and the gradient vanishes there."""
    rng = np.random.default_rng(1)
    X = torch.as_tensor(rng.uniform(0, 10, (30, 1)), device="cuda")
    y = torch.sin(X[:, 0]) + 0.1 * torch.as_tensor(rng.standard_normal(30), device="cuda")
    f = S.GP(S.EQ())
    fs = (f | (f(X, 0.01), y)).sample_function(num=4, features=4096, state=torch.Generator().manual_seed(3))
    grid = torch.linspace(0, 10, 2**16, dtype=torch.float64, device="cuda")[:, None]
    with torch.no_grad():
        grid_max = fs(grid).max(0).values
    starts = 32
    x = torch.as_tensor(rng.uniform(0, 10, (4 * starts, 1)), device="cuda").requires_grad_()
    mask = torch.zeros(4 * starts, 4, dtype=torch.float64, device="cuda")
    for s in range(4):
        mask[s * starts : (s + 1) * starts, s] = 1.0
    opt = torch.optim.LBFGS([x], max_iter=200, tolerance_grad=1e-12, tolerance_change=1e-15, line_search_fn="strong_wolfe")

    def closure():
        opt.zero_grad()
        loss = -(fs(x) * mask).sum()
        loss.backward()
        return loss

    for _ in range(5):
        opt.step(closure)
    xo = x.detach().clone().requires_grad_()
    vals = (fs(xo) * mask).sum(1)
    (grad,) = torch.autograd.grad(vals.sum(), xo)
    for s in range(4):
        blk = slice(s * starts, (s + 1) * starts)
        i = vals[blk].argmax()
        assert vals[blk][i].item() >= grid_max[s].item() - 1e-9, (s, vals[blk][i].item(), grid_max[s].item())
        assert abs(grad[blk][i].item()) <= 1e-6, (s, grad[blk][i].item())


@pytest.mark.gpu
def test_scale_grad(S):
    """Forward and backward at 2^20 points with n = 16384, num = 16: peak device memory above the level before the sample
    stays below 1 GiB plus the factor of K."""
    rng = np.random.default_rng(0)
    n, d = 16384, 8
    X = torch.as_tensor(rng.standard_normal((n, d)), device="cuda")
    y = torch.as_tensor(rng.standard_normal(n), device="cuda")
    xs = torch.as_tensor(rng.standard_normal((2**20, d)), device="cuda").requires_grad_()
    f = S.GP(S.EQ().stretch(2.0))
    post = f | (f(X, 0.1), y)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    fs = post.sample_function(num=16, features=4096, state=torch.Generator().manual_seed(0))
    out = fs(xs)
    out.sum().backward()
    torch.cuda.synchronize()
    factor = post.mean.K_z.chol().W.numel() * 8
    assert out.shape == (2**20, 16) and torch.isfinite(xs.grad).all()
    assert torch.cuda.max_memory_allocated() - before < (1 << 30) + factor
