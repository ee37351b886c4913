"""Pathwise function samples (``GP.sample_function``, ``stheno_b200/pathwise.py``) and their feature kernel
(``gpk_feature_eval``, ``csrc/sample_fn.cu``).

* the kernel against a torch fp64 restatement over row / feature / sample counts around its tile edges, at phases up to
  16384;
* the spectral draws: random-feature inner products against ``k(x, y)`` and the moments of the frequencies;
* the pathwise identity ``f~(x*) + k(x*, X) K^-1 (y - f~(X) - eps)`` restated in torch fp64 from the draws the sample holds;
* the statistics of many samples against the exact posterior, that a sample is one function, its memory at 2^20 points and
  what it refuses.

The host cases run the model layer on the torch-CPU stand-ins of ``tests/_cpu_backend.py`` (with a torch restatement of the
feature kernel); the ``gpu`` cases run the CUDA kernels."""
import math
import types

import numpy as np
import pytest
import torch

U32 = 2.0**-24


def feat_ref(x, omega, b, amp, W):
    """The feature kernel restated in fp64: ``(cos(x omega^T + b) amp) W^T`` and the sum of |terms| per element."""
    x, omega, b, amp, W = [t.to(torch.float64) for t in (x, omega, b, amp, W)]
    phi = torch.cos(x @ omega.T + b) * amp
    return phi @ W.T, phi.abs() @ W.abs().T


@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.B, "precision", "auto")
    monkeypatch.setattr(s.Measure, "default", None)
    return s


@pytest.fixture
def host(cpu_backend, monkeypatch):
    """The CPU stand-ins, with the feature kernel restated in torch for ``pathwise``."""
    from stheno_b200 import pathwise

    def feature_eval(x, omega, b, amp, W, out=None):
        v = feat_ref(x, omega, b, amp, W)[0].to(x.dtype)
        if out is None:
            return v
        out += v
        return out

    stand_in = types.SimpleNamespace(**{k: getattr(cpu_backend, k) for k in dir(cpu_backend) if not k.startswith("__")})
    stand_in.feature_eval = feature_eval
    monkeypatch.setattr(pathwise, "ops", stand_in)
    return cpu_backend


# ---- torch fp64 restatements of the kernels and of the pathwise identity -------------------------------------------------
def k_unit(kind, a, b, alpha=None):
    d2 = ((a[:, None, :] - b[None, :, :]) ** 2).sum(-1)
    if kind == "eq":
        return torch.exp(-d2 / 2)
    if kind == "rq":
        return (1 + d2 / (2 * alpha)) ** -alpha
    r = torch.sqrt(d2.clamp_min(0))
    if kind == "matern12":
        return torch.exp(-r)
    if kind == "matern32":
        return (1 + math.sqrt(3) * r) * torch.exp(-math.sqrt(3) * r)
    if kind == "matern52":
        return (1 + math.sqrt(5) * r + 5 * d2 / 3) * torch.exp(-math.sqrt(5) * r)
    raise ValueError(kind)


def periodic(x, p):
    ang = x * 2 * math.pi / p
    return torch.cat([torch.sin(ang), torch.cos(ang)], -1)


#: (name, stheno kernel, torch restatement of (k(a, b), map of the points), mean, restated mean, noise kind)
def cases(S):
    ls = torch.tensor([0.6, 1.1, 1.7], dtype=torch.float64)
    return [
        ("eq+linear", 1.5 * S.EQ().stretch(0.8) + 0.3 * S.Linear().stretch(2.0),
         lambda a, b: 1.5 * k_unit("eq", a / 0.8, b / 0.8) + 0.3 * (a / 2.0) @ (b / 2.0).T, lambda x: x,
         0.5, lambda x: 0.5 + 0 * x[:, :1], "scalar"),
        ("matern32-ard", 0.8 * S.Matern32().stretch(ls.numpy()) + 0.2 * S.Matern52().stretch(2.5),
         lambda a, b: 0.8 * k_unit("matern32", a / ls, b / ls) + 0.2 * k_unit("matern52", a / 2.5, b / 2.5), lambda x: x,
         lambda x: 0.3 * x[:, :1] - 0.1, lambda x: 0.3 * x[:, :1] - 0.1, "hetero"),
        ("rq-periodic", (1.2 * S.RQ(1.5).stretch(0.6)).periodic(1.3),
         lambda a, b: 1.2 * k_unit("rq", a / 0.6, b / 0.6, 1.5), lambda x: periodic(x, 1.3), 0, lambda x: 0 * x[:, :1],
         "scalar"),
    ]


def restate(fs, kfun, pmap, mfun, xs, X=None, y=None, noise=None, eps=1e-12):
    """``f~(x*) (+ k(x*, X) K^-1 (y - f~(X) - eps))`` in fp64 from the draws ``fs`` holds."""
    def prior(x):
        u = pmap(x)
        out = mfun(x) + torch.cos(u @ fs.omega.cpu().T + fs.b.cpu()) * fs.amp.cpu() @ fs.W.cpu().T
        return out if fs.linear is None else out + u @ fs.linear.cpu()

    want = prior(xs)
    if X is None:
        return want
    uX = pmap(X)
    K = kfun(uX, uX) + torch.diag(noise) + eps * torch.eye(len(X), dtype=torch.float64)
    L = torch.linalg.cholesky(K)
    V = torch.cholesky_solve(y.reshape(-1, 1) - prior(X) - fs.eps.cpu(), L)
    return want + kfun(pmap(xs), uX) @ V, torch.linalg.cond(K).item()


def identity_case(S, case, n, m, dtype, dev, num=3, features=512, seed=0):
    name, k, kfun, pmap, mean, mfun, noise_kind = case
    rng = np.random.default_rng(seed)
    d = 3
    X = torch.as_tensor(rng.uniform(-2, 2, (n, d)))
    xs = torch.as_tensor(rng.uniform(-2.5, 2.5, (m, d)))
    y = torch.as_tensor(rng.standard_normal(n))
    noise = torch.full((n,), 0.1, dtype=torch.float64) if noise_kind == "scalar" else \
        torch.as_tensor(rng.uniform(0.05, 0.3, n))
    f = S.GP(mean, k)
    nz = 0.1 if noise_kind == "scalar" else noise.to(dev, dtype)
    post = f | (f(X.to(dev, dtype), nz), y.to(dev, dtype))
    fs = post.sample_function(num=num, features=features, state=torch.Generator().manual_seed(seed))
    got = fs(xs.to(dev, dtype)).cpu().to(torch.float64)
    want, cond = restate(fs, kfun, pmap, mfun, xs, X, y, noise, S.B.epsilon)
    return got, want, cond, fs


# ---- host: the spectral draws ------------------------------------------------------------------------------------------
KINDS = [("eq", None), ("matern12", None), ("matern32", None), ("matern52", None), ("rq", 0.7), ("rq", 2.5)]


def unit_kernel(S, kind, alpha):
    return {"eq": S.EQ, "matern12": S.Matern12, "matern32": S.Matern32, "matern52": S.Matern52}[kind]() if alpha is None \
        else S.RQ(alpha)


@pytest.mark.parametrize("kind,alpha", KINDS)
def test_spectral_draws(S, host, kind, alpha):
    """``phi(x)^T phi(y)`` of 2^16 features meets ``k(x, y)`` (K1's CPU stand-in) within 6 / sqrt(F) at 50 random pairs, for two
    stretches and a length-scale vector, and the frequencies have the stated distribution."""
    from scipy import stats

    F, d = 2**16, 3
    rng = np.random.default_rng(1)
    ells = [0.7, 2.0, np.array([0.5, 1.0, 3.0])]
    for j, ell in enumerate(ells):
        k = 1.3 * unit_kernel(S, kind, alpha).stretch(ell)
        fs = S.GP(k).sample_function(features=F, state=torch.Generator().manual_seed(j))
        x = torch.as_tensor(rng.uniform(-1.5, 1.5, (50, d)))
        y = x + torch.as_tensor(rng.standard_normal((50, d)) * np.asarray(ell) * 0.8)
        fs._draw(d)
        phi = lambda p: torch.cos(p @ fs.omega.T + fs.b) * fs.amp
        approx = (phi(x) * phi(y)).sum(1)
        exact = torch.as_tensor(S.B.dense(k(x, y))).diagonal()
        assert (approx - exact).abs().max() <= 6 / math.sqrt(F) * 1.3, (kind, ell)
        # the frequencies, back at unit length scale
        w = (fs.omega * torch.as_tensor(np.broadcast_to(ell, (d,)).copy())).numpy()
        if kind == "eq":
            assert stats.kstest(w[:, 0], stats.norm.cdf).pvalue > 1e-4
        elif kind.startswith("matern"):
            dof = {"matern12": 1, "matern32": 3, "matern52": 5}[kind]
            assert stats.kstest(w[:, 0], stats.t(df=dof).cdf).pvalue > 1e-4
            # multivariate t: the coordinates share one u, so |w|^2 / d is F(d, 2 nu)-distributed
            assert stats.kstest((w**2).sum(1) / d, stats.f(d, dof).cdf).pvalue > 1e-4
        else:  # sqrt(tau) z, tau ~ Gamma(alpha, rate alpha): E w^2 = 1, E w^4 = 3 (1 + 1 / alpha)
            m2, m4 = (w**2).mean(), (w**4).mean()
            se2 = math.sqrt(((w**2 - 1) ** 2).mean() / w.size)
            assert abs(m2 - 1) < 5 * se2, (m2, se2)
            assert abs(m4 / (3 * (1 + 1 / alpha)) - 1) < 0.1, m4


@pytest.mark.parametrize("noise_kind", ["scalar", "hetero"])
def test_noise_draw(S, host, noise_kind):
    """The observation-noise draw ``eps`` of a posterior sample is N(0, Sigma_noise): standardised by the noise of its point,
    its mean, variance and per-point variances match N(0, 1) within 5 standard errors (5.5 per point, over 300 points), and a
    Kolmogorov-Smirnov test does not reject it."""
    from scipy import stats

    n, num = 300, 2000
    rng = np.random.default_rng(6)
    X, y = rng.uniform(-2, 2, (n, 1)), rng.standard_normal(n)
    noise = np.full(n, 0.2) if noise_kind == "scalar" else rng.uniform(0.01, 0.5, n)
    f = S.GP(S.EQ())
    post = f | (f(X, 0.2 if noise_kind == "scalar" else noise), y)
    fs = post.sample_function(num=num, features=16, state=torch.Generator().manual_seed(2))
    z = (fs.eps / torch.as_tensor(np.sqrt(noise)).unsqueeze(1)).numpy()
    assert z.shape == (n, num)
    N = z.size
    assert abs(z.mean()) < 5 / math.sqrt(N)
    assert abs(z.var() - 1) < 5 * math.sqrt(2 / N)
    assert np.abs(z.var(1) - 1).max() < 5.5 * math.sqrt(2 / num)
    assert stats.kstest(z.reshape(-1)[:200000], stats.norm.cdf).pvalue > 1e-4


def test_one_factor_and_scale_of_features(S, host):
    """Features are split evenly over the stationary terms and each term's amplitude is sqrt(2 c_t / F_t)."""
    k = 2.0 * S.EQ() + 0.5 * S.Matern12().stretch(3.0) + S.Linear()
    fs = S.GP(k).sample_function(num=2, features=101, state=torch.Generator().manual_seed(0))
    fs(np.zeros((4, 2)))
    assert fs.omega.shape == (101, 2) and fs.W.shape == (2, 101) and fs.linear.shape == (2, 2)
    assert torch.allclose(fs.amp[:51], torch.full((51,), math.sqrt(4.0 / 51), dtype=torch.float64))
    assert torch.allclose(fs.amp[51:], torch.full((50,), math.sqrt(1.0 / 50), dtype=torch.float64))


# ---- host: the pathwise identity, one function, refusals -----------------------------------------------------------------
@pytest.mark.parametrize("which", [0, 1, 2])
def test_pathwise_identity_host(S, host, which):
    got, want, _, _ = identity_case(S, cases(S)[which], 150, 40, torch.float64, "cpu")
    assert (got - want).abs().max() <= 1e-10 * max(1.0, want.abs().max().item())


def test_prior_identity_host(S, host):
    name, k, kfun, pmap, mean, mfun, _ = cases(S)[2]
    fs = S.GP(mean, k).sample_function(num=4, features=256, state=torch.Generator().manual_seed(3))
    xs = torch.as_tensor(np.random.default_rng(0).uniform(-2, 2, (30, 3)))
    got = fs(xs)
    assert torch.allclose(got, restate(fs, kfun, pmap, mfun, xs), rtol=0, atol=1e-12)


def one_function(S, dev):
    rng = np.random.default_rng(4)
    X, y = rng.uniform(-2, 2, (200, 2)), rng.standard_normal(200)
    f = S.GP(S.EQ().stretch(0.7) + 0.2 * S.Matern32())
    post = f | (f(X, 0.05), y)
    xa = torch.as_tensor(rng.uniform(-3, 3, (300, 2)), device=dev)
    xb = torch.as_tensor(rng.uniform(-3, 3, (77, 2)), device=dev)
    fs = post.sample_function(num=5, features=1000, state=torch.Generator().manual_seed(9))
    a, b, ab = fs(xa), fs(xb), fs(torch.cat([xa, xb]))
    assert torch.allclose(torch.cat([a, b]), ab, rtol=1e-13, atol=1e-13 * ab.abs().max().item())
    assert torch.equal(fs(xa), a)
    again = post.sample_function(num=5, features=1000, state=torch.Generator().manual_seed(9))
    assert torch.equal(again(xa), a)
    other = post.sample_function(num=5, features=1000, state=torch.Generator().manual_seed(10))
    assert not torch.allclose(other(xa), a)
    # numpy in, numpy out
    out = fs(xa.cpu().numpy())
    assert isinstance(out, np.ndarray) and out.shape == (300, 5)


def test_one_function_host(S, host):
    one_function(S, "cpu")


def refusals(S):
    x = np.linspace(0, 1, 20)[:, None]
    y = np.sin(3 * x[:, 0])
    m = S.Measure()
    f = S.GP(S.EQ(), measure=m)
    g = S.GP(S.Matern12(), measure=m)
    out = [
        (lambda: S.GP(S.EQ() * S.Matern32()).sample_function(), "products of kernel factors"),
        (lambda: S.GP(S.EQ() + 0.1 * S.Delta()).sample_function(), "Delta"),
        (lambda: S.GP(S.EQ()).diff(0).sample_function(), "derivative"),
        (lambda: (lambda p: p * (lambda t: t[:, :1]))(S.GP(S.EQ())).sample_function(), "function-scaled"),
        (lambda: S.cross(f, g).sample_function(), "multi-output"),
        (lambda: (f | S.PseudoObs(f(x[::4]), f(x, 0.1), y)).sample_function(), "sparse"),
        (lambda: (f | S.Obs((f(x, 0.1), y), (g(x, 0.1), y))).sample_function(), "several observed processes"),
        (lambda: ((f + g) | (f(x, 0.1), y)).sample_function(), "another process"),
        (lambda: S.GP(S.EQ()).sample_function()(np.zeros((2, 5, 1))), "batched"),
        (lambda: S.GP(S.EQ()).sample_function()((x, x)), "multi-output"),
    ]
    return out


def test_refusals_host(S, host):
    for fn, reason in refusals(S):
        with pytest.raises(ValueError, match=reason):
            fn()


def test_grad_mode_host(S, host):
    """Under grad mode the value is the no-grad one, attached so that ``backward()`` raises."""
    ell = torch.tensor(0.8, dtype=torch.float64, requires_grad=True)
    rng = np.random.default_rng(2)
    X, y, xs = torch.as_tensor(rng.uniform(-2, 2, (50, 1))), torch.as_tensor(rng.standard_normal(50)), \
        torch.as_tensor(rng.uniform(-2, 2, (20, 1)))
    f = S.GP(S.EQ().stretch(ell))
    fs = (f | (f(X, 0.1), y)).sample_function(num=2, state=torch.Generator().manual_seed(0))
    v = fs(xs)
    with torch.no_grad():
        ref = (f | (f(X, 0.1), y)).sample_function(num=2, state=torch.Generator().manual_seed(0))(xs)
    assert torch.equal(v.detach(), ref)
    with pytest.raises(NotImplementedError, match="function sampling"):
        v.sum().backward()


# ---- GPU: the feature kernel -----------------------------------------------------------------------------------------------
def dyadic_inputs(n, F, num, d, big, dtype, seed):
    """Inputs whose phases are exact in fp64 whatever the summation order: x on a grid of 1/4, omega of 1/64, b of 2^-20.
    ``big``: phases up to 16384 (|x| <= 16, |omega| <= 1024 / d), reached in row 0 x feature 0."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-64, 65, (n, d), generator=g).double() / 4
    scale = 2**16 // d if big else 8
    omega = torch.randint(-scale, scale + 1, (F, d), generator=g).double() / 64
    if big:  # the largest phase the grid allows, 16 * 1024 = 16384, in row 0 x feature 0
        x[0], omega[0] = 16.0, scale / 64
    b = torch.randint(0, 6 * 2**20, (F,), generator=g).double() / 2**20
    amp = torch.rand(F, generator=g, dtype=torch.float64) + 0.5
    W = torch.randn(num, F, generator=g, dtype=torch.float64)
    return [t.to("cuda", dtype) for t in (x, omega, b, amp, W)]


GRID = [(n, F, num, d) for n in (1, 127, 128, 129, 5000) for F, num, d in
        ((1, 1, 1), (64, 7, 8), (65, 8, 1), (4096, 33, 8), (65, 33, 8), (4096, 1, 1))]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("n,F,num,d", GRID)
def test_feature_kernel_parity(n, F, num, d, dtype):
    from stheno_b200 import ops

    bound = 1e-13 if dtype == torch.float64 else 2.0**-20
    for big in (False, True):
        x, omega, b, amp, W = dyadic_inputs(n, F, num, d, big, dtype, seed=n + F + num)
        want, mag = feat_ref(*[t.cpu() for t in (x, omega, b, amp, W)])
        if big:
            assert (x.cpu().double() @ omega.cpu().double().T).abs().max() >= 1e4
        got = ops.feature_eval(x, omega, b, amp, W)
        assert got.dtype == dtype and got.shape == (n, num)
        err = ((got.cpu().double() - want).abs() / mag.clamp_min(1e-300)).max().item()
        assert err <= bound, (n, F, num, d, big, err)
        base = torch.randn(n, num, dtype=dtype, device="cuda")
        acc = ops.feature_eval(x, omega, b, amp, W, out=base.clone())
        err = ((acc.cpu().double() - base.cpu().double() - want).abs()
               / (mag + base.cpu().double().abs())).max().item()
        assert err <= bound, (n, F, num, d, big, "accumulate", err)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("num", [3, 16])
def test_feature_kernel_nan(dtype, num):
    from stheno_b200 import ops

    x, omega, b, amp, W = dyadic_inputs(300, 200, num, 5, True, dtype, seed=1)
    assert torch.isfinite(ops.feature_eval(x, omega, b, amp, W)).all()
    x[17, 2] = float("nan")
    out = ops.feature_eval(x, omega, b, amp, W)
    assert torch.isnan(out[17]).all()
    assert torch.isfinite(out[torch.arange(300, device="cuda") != 17]).all()


# ---- GPU: the pathwise identity ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1, 2])
def test_pathwise_identity(S, which):
    got, want, _, _ = identity_case(S, cases(S)[which], 2500, 600, torch.float64, "cuda", num=9, features=2048)
    assert (got - want).abs().max() <= 1e-10 * max(1.0, want.abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
def test_pathwise_identity_emulated(S, monkeypatch, precision):
    """n = 6000: the update's solves run on the int8 emulation (8 slices) under ``auto`` and ``int8x8``."""
    monkeypatch.setattr(S.B, "precision", precision)
    got, want, _, _ = identity_case(S, cases(S)[0], 6000, 300, torch.float64, "cuda", num=4, features=1024)
    assert (got - want).abs().max() <= 1e-10 * max(1.0, want.abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 2])
def test_pathwise_identity_fp32(S, which):
    got, want, cond, _ = identity_case(S, cases(S)[which], 1500, 300, torch.float32, "cuda", num=8, features=1024)
    err = (got - want).abs().max().item() / max(1.0, want.abs().max().item())
    assert err <= 16.0 * U32 * cond, (err, cond)


@pytest.mark.gpu
def test_one_function(S):
    one_function(S, "cuda")


@pytest.mark.gpu
def test_refusals(S):
    for fn, reason in refusals(S):
        with pytest.raises(ValueError, match=reason):
            fn()


@pytest.mark.gpu
def test_grad_mode(S):
    ell = torch.tensor(0.8, dtype=torch.float64, device="cuda", requires_grad=True)
    xs = torch.linspace(-2, 2, 30, dtype=torch.float64, device="cuda")[:, None]
    fs = S.GP(S.EQ().stretch(ell)).sample_function(num=2, state=torch.Generator().manual_seed(0))
    v = fs(xs)
    assert v.requires_grad
    with pytest.raises(NotImplementedError, match="function sampling"):
        v.sum().backward()


# ---- GPU: statistics, scale ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["eq", "matern32", "rq"])
@pytest.mark.parametrize("posterior", [False, True])
def test_statistics(S, kind, posterior):
    """4000 samples of 8192 features at 40 points: mean and covariance within 5 Monte-Carlo standard errors plus 6 / sqrt(F)
    of the prior variance of the exact (posterior) ones."""
    F, N = 8192, 4000
    k = 1.4 * {"eq": S.EQ(), "matern32": S.Matern32(), "rq": S.RQ(0.8)}[kind].stretch(0.9)
    f = S.GP(0.3, k)
    rng = np.random.default_rng(5)
    xs = torch.as_tensor(rng.uniform(-2, 2, (40, 2)), device="cuda")
    if posterior:
        X = torch.as_tensor(rng.uniform(-2, 2, (60, 2)), device="cuda")
        f = f | (f(X, 0.05), torch.as_tensor(rng.standard_normal(60), device="cuda"))
    fdd = f(xs)
    mean, cov = fdd.mean.reshape(-1).cpu(), torch.as_tensor(S.B.dense(fdd.var)).cpu()
    s = f.sample_function(num=N, features=F, state=torch.Generator().manual_seed(11))(xs).cpu()
    emp_mean, emp_cov = s.mean(1), torch.cov(s)
    var = cov.diagonal().clamp_min(0)
    se_mean = torch.sqrt(var / N)
    se_cov = torch.sqrt((var[:, None] * var[None, :] + cov**2) / N)
    feat = 6 / math.sqrt(F) * 1.4
    assert ((emp_mean - mean).abs() <= 5 * se_mean + feat).all(), (emp_mean - mean).abs().max()
    assert ((emp_cov - cov).abs() <= 5 * se_cov + feat).all(), (emp_cov - cov).abs().max()


@pytest.mark.gpu
def test_scale(S):
    """One evaluation at 2^20 points with n = 16384: peak device memory above the level before the sample stays below 1 GiB
    plus the factor of K."""
    rng = np.random.default_rng(0)
    n, d = 16384, 8
    X = torch.as_tensor(rng.standard_normal((n, d)), device="cuda")
    y = torch.as_tensor(rng.standard_normal(n), device="cuda")
    xs = torch.as_tensor(rng.standard_normal((2**20, d)), device="cuda")
    f = S.GP(S.EQ().stretch(2.0))
    post = f | (f(X, 0.1), y)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    fs = post.sample_function(num=16, features=4096, state=torch.Generator().manual_seed(0))
    out = fs(xs)
    torch.cuda.synchronize()
    factor = post.mean.K_z.chol().W.numel() * 8
    assert out.shape == (2**20, 16) and torch.isfinite(out).all()
    assert torch.cuda.max_memory_allocated() - before < (1 << 30) + factor
