"""Leave-one-out (LOO) predictive marginals and log densities: ``Normal.loo_marginals`` and ``Normal.loo_logpdf``.

For ``y ~ N(m, Sigma)``, ``Sigma = var + B.epsilon I``, ``r = y - m``, ``alpha = Sigma^-1 r`` and ``c = diag Sigma^-1``:
``mu_i = y_i - alpha_i / c_i``, ``sigma_i^2 = 1 / c_i`` and ``log p(y_i | y_-i) = -1/2 log 2 pi + 1/2 log c_i - 1/2 alpha_i^2 / c_i``.

  1. the closed form against ``n`` explicit conditionings (host, NumPy), and on the host stand-ins of the CUDA ops;
  2. values against an fp64 NumPy/SciPy restatement of the closed form (``loo_ref`` below): shapes, models, emulation, fp32,
     missing data;
  3. gradients of ``loo_logpdf`` against torch fp64 autograd of a ``torch.linalg.cholesky`` restatement;
  4. config 2 (n = 16384, d = 8) against the CPU reference;
  5. contracts: determinism, values under grad, the streamed inverse diagonal, ``gpk_loo_finish`` on its own."""
import math

import numpy as np
import pytest
import scipy.linalg as sla
import torch

from oracle import gp_oracle as O

EPS = 1e-12


# ---- fp64 references ----------------------------------------------------------------------------------------------------
def loo_ref(Sigma, r, eps=EPS):
    """The closed form in fp64 (NumPy/SciPy): ``(mean - m [n, k], var [n], lp [k])`` of ``N(0, Sigma + eps I)`` at ``r``."""
    n = Sigma.shape[0]
    L = np.linalg.cholesky(Sigma + eps * np.eye(n)) if n <= 8192 else O.chol_eps(Sigma, eps)
    alpha = sla.cho_solve((L, True), r)
    inv, info = sla.lapack.dpotri(L, lower=1)
    assert info == 0
    c = np.diag(inv).copy()
    s = alpha / c[:, None]
    lp = 0.5 * ((np.log(c)[:, None] - alpha * s).sum(0) - n * O.LOG_2_PI)
    return r - s, 1.0 / c, lp


def loo_brute(Sigma, y, m, eps=EPS):
    """``n`` explicit conditionings of ``N(m, Sigma + eps I)`` on the other ``n - 1`` entries (one column ``y``)."""
    n = Sigma.shape[0]
    S = Sigma + eps * np.eye(n)
    mean, var, lp = np.empty(n), np.empty(n), 0.0
    for i in range(n):
        o = np.arange(n) != i
        if n == 1:
            mu, v = m[i], S[i, i]
        else:
            w = np.linalg.solve(S[np.ix_(o, o)], S[o, i])
            mu, v = m[i] + w @ (y[o] - m[o]), S[i, i] - w @ S[o, i]
        mean[i], var[i] = mu, v
        lp += -0.5 * (O.LOG_2_PI + math.log(v) + (y[i] - mu) ** 2 / v)
    return mean, var, lp


def _close(got, want, bar):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    scale = max(1.0, float(np.abs(want).max()))
    err = float(np.abs(got - want).max())
    assert err <= bar * scale, (err, scale)
    return err / scale


# ---- 1. the closed form ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 7, 40])
def test_closed_form_equals_explicit_conditioning(n):
    rng = np.random.default_rng(n)
    x = rng.standard_normal((n, 2))
    Sigma = O.kernel_matrix(("stretched", 0.9, ("matern52",)), x) + 0.05 * np.diag(rng.uniform(1, 2, n))
    m = rng.standard_normal(n)
    y = rng.standard_normal(n)
    mean_r, var, lp = loo_ref(Sigma, (y - m)[:, None])
    bm, bv, blp = loo_brute(Sigma, y, m)
    np.testing.assert_allclose(mean_r[:, 0] + m, bm, rtol=1e-12, atol=1e-12 * np.abs(bm).max())
    np.testing.assert_allclose(var, bv, rtol=1e-12)
    np.testing.assert_allclose(lp[0], blp, rtol=1e-12)
    if n == 1:  # the prior marginal
        assert abs(var[0] - Sigma[0, 0] - EPS) <= 1e-15 and mean_r[0, 0] == 0.0


def _install_loo_stand_ins(monkeypatch, cpu):
    """The LOO pieces the host stand-ins of the CUDA ops lack: ``Chol.inverse_diag``, ``Chol.loo`` and ``loo_finish``."""
    def inverse_diag(self):
        L = torch.tril(self.W[:, : self.n_pad, :])
        return torch.diagonal(torch.cholesky_inverse(L), dim1=1, dim2=2)[:, : self.n].clone()

    def loo_finish(c, alpha, r=None, g=None, *, want_mean=True, want_var=True, want_lp=True):
        s = alpha / c.unsqueeze(1)
        if g is not None:
            return (g.unsqueeze(-1) * (1 + alpha * s)).sum(1) / (2 * c), g.unsqueeze(-1) * s
        lp = 0.5 * ((torch.log(c).unsqueeze(1) - alpha * s).sum(-1) - c.shape[-1] * O.LOG_2_PI)
        return (r - s) if want_mean else None, 1.0 / c, lp

    def loo(self, r, want_mean=True):
        alpha = self.full_solve(r)
        c = self.inverse_diag()
        return loo_finish(c, alpha, r, want_mean=want_mean) + (alpha, c)

    monkeypatch.setattr(cpu.Chol, "inverse_diag", inverse_diag, raising=False)
    monkeypatch.setattr(cpu.Chol, "loo", loo, raising=False)
    monkeypatch.setattr(cpu, "loo_finish", loo_finish, raising=False)


@pytest.fixture
def host(cpu_backend, monkeypatch):
    _install_loo_stand_ins(monkeypatch, cpu_backend)
    import stheno_b200 as S

    return S


def test_host_routes_against_brute_force(host):
    """Every covariance branch on the host stand-ins: kernel matrix (with a prior mean), dense, diagonal, Woodbury."""
    S = host
    rng = np.random.default_rng(3)
    n = 30
    x = rng.standard_normal((n, 2))
    y = rng.standard_normal(n)
    spec = ("sum", ("stretched", 1.1, ("eq",)), ("scaled", 0.3, ("linear",)))
    f = S.GP(lambda t: 0.5 * t.sum(-1, keepdim=True), S.EQ().stretch(1.1) + 0.3 * S.Linear())
    fdd = f(x, 0.1)
    assert type(fdd.var).__name__ == "KernelDense"
    Sigma = O.kernel_matrix(spec, x) + 0.1 * np.eye(n)
    m = 0.5 * x.sum(-1)
    bm, bv, blp = loo_brute(Sigma, y, m)
    mean, var = fdd.loo_marginals(y)
    assert mean.shape == (n,) and var.shape == (n,)
    _close(mean, bm, 1e-12)
    _close(var, bv, 1e-12)
    _close(fdd.loo_logpdf(y), blp, 1e-12)

    dense = S.Normal(m[:, None], Sigma)  # a Dense covariance
    _close(dense.loo_marginals(y)[0], bm, 1e-12)
    _close(dense.loo_logpdf(y), blp, 1e-12)

    d = rng.uniform(0.5, 2.0, n)
    diag = S.Normal(m[:, None], S.matrix.Diagonal(torch.tensor(d)))
    dm, dv = diag.loo_marginals(y)
    _close(dm, m, 1e-15)  # LOO of independent entries is their marginal
    _close(dv, d, 1e-15)
    _close(diag.loo_logpdf(y), -0.5 * (O.LOG_2_PI * n + np.log(d).sum() + ((y - m) ** 2 / d).sum()), 1e-12)

    wb = S.GP(0.7 * S.Linear())(x, 0.2)
    assert type(wb.var).__name__ == "Woodbury"
    Sw = 0.7 * x @ x.T + 0.2 * np.eye(n)
    wm, wv, wlp = loo_brute(Sw, y, np.zeros(n), eps=0.0)
    _close(wb.loo_marginals(y)[0], wm, 1e-11)
    _close(wb.loo_marginals(y)[1], wv, 1e-11)
    _close(wb.loo_logpdf(y), wlp, 1e-11)


def test_host_shapes_missing_data_and_refusal(host):
    S = host
    rng = np.random.default_rng(4)
    n, k = 20, 3
    x = rng.standard_normal((n, 1))
    fdd = S.GP(S.EQ())(x, 0.1)
    Y = rng.standard_normal((n, k))
    mean, var = fdd.loo_marginals(Y)
    assert mean.shape == (n, k) and var.shape == (n,) and fdd.loo_logpdf(Y).shape == (k,)
    for j in range(k):  # columns are independent problems
        _close(mean[:, j], fdd.loo_marginals(Y[:, j])[0], 1e-14)
    # missing data: the observed sub-problem, NaN at the missing positions
    y = Y[:, 0].copy()
    y[[2, 11]] = np.nan
    mean, var = fdd.loo_marginals(y)
    obs = ~np.isnan(y)
    sub = S.GP(S.EQ())(x[obs], 0.1)
    assert np.isnan(mean[~obs]).all() and np.isnan(var[~obs]).all()
    _close(mean[obs], sub.loo_marginals(y[obs])[0], 1e-14)
    _close(var[obs], sub.loo_marginals(y[obs])[1], 1e-14)
    _close(fdd.loo_logpdf(y), sub.loo_logpdf(y[obs]), 1e-14)
    # torch in, torch out; Woodbury and diagonal values carry torch graphs
    s = torch.tensor(0.2, dtype=torch.float64, requires_grad=True)
    lp = S.GP(s * S.Linear())(torch.tensor(x), 0.3).loo_logpdf(torch.tensor(Y[:, 0]))
    assert isinstance(lp, torch.Tensor) and lp.requires_grad
    lp.backward()
    assert s.grad is not None and torch.isfinite(s.grad)
    # the kernel-matrix marginals come from raw-pointer kernels: a backward through them raises
    l = torch.tensor(1.0, dtype=torch.float64, requires_grad=True)
    mean, _ = S.GP(S.EQ().stretch(l))(torch.tensor(x), 0.1).loo_marginals(torch.tensor(Y[:, 0]))
    with pytest.raises(NotImplementedError, match="loo_marginals"):
        mean.sum().backward()


# ---- the GPU -------------------------------------------------------------------------------------------------------------
@pytest.fixture
def S():
    import stheno_b200 as S

    before = S.B.epsilon, S.B.precision
    yield S
    S.B.epsilon, S.B.precision = before


def _dev(a, dtype=torch.float64):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device="cuda")


def _check(fdd, Sigma, y, m, bar=1e-10):
    """``fdd``'s LOO marginals and log density at ``y [n, k]`` (host) against :func:`loo_ref`."""
    mean_r, var, lp = loo_ref(Sigma, y - m[:, None])
    mean, v = fdd.loo_marginals(y)
    k = y.shape[1]
    errs = [_close(mean if k > 1 else mean[:, None], mean_r + m[:, None], bar), _close(v, var, bar),
            _close(np.atleast_1d(fdd.loo_logpdf(y)), lp, bar)]
    return max(errs)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("n", [2, 127, 128, 129, 1000, 2500])
def test_values_shapes(S, n, k):
    """EQ with a prior mean, unbatched ``(n, k)`` and batched ``(2, n, 1)``, against the fp64 closed form."""
    rng = np.random.default_rng(n + k)
    x = rng.standard_normal((2, n, 3))
    y = rng.standard_normal((2, n, k))
    spec = ("scaled", 1.3, ("stretched", 0.9, ("eq",)))
    f = S.GP(lambda t: 0.3 * t[..., :1], 1.3 * S.EQ().stretch(0.9))
    for b in range(2):
        Sigma = O.kernel_matrix(spec, x[b]) + 0.05 * np.eye(n)
        _check(f(x[b], 0.05), Sigma, y[b], 0.3 * x[b, :, 0])
    if k == 1:  # batched: (2, n) marginals, (2,) log densities
        fdd = f(x, 0.05)
        mean, var = fdd.loo_marginals(y)
        lp = fdd.loo_logpdf(y)
        assert mean.shape == (2, n) and var.shape == (2, n) and lp.shape == (2,)
        for b in range(2):
            Sigma = O.kernel_matrix(spec, x[b]) + 0.05 * np.eye(n)
            mr, vr, lr = loo_ref(Sigma, y[b] - 0.3 * x[b, :, :1])
            _close(mean[b], mr[:, 0] + 0.3 * x[b, :, 0], 1e-10)
            _close(var[b], vr, 1e-10)
            _close(lp[b], lr[0], 1e-10)


def _model(S, name, n, rng):
    """``(fdd, Sigma without eps, prior mean [n])`` of a named model."""
    x = rng.standard_normal((n, 3))
    if name == "hetero":
        nv = rng.uniform(0.01, 0.3, n)
        return S.GP(S.EQ().stretch(1.2))(x, nv), O.kernel_matrix(("stretched", 1.2, ("eq",)), x) + np.diag(nv), np.zeros(n)
    if name == "ard_sum":
        ls = np.array([0.7, 1.3, 2.1])
        k = S.Matern32().stretch(ls) + 0.5 * S.RQ(1.5).stretch(0.8) + 0.2 * S.Linear()
        spec = ("sum", ("sum", ("stretched", ls, ("matern32",)), ("scaled", 0.5, ("stretched", 0.8, ("rq", 1.5)))),
                ("scaled", 0.2, ("linear",)))
        return S.GP(k)(x, 0.1), O.kernel_matrix(spec, x) + 0.1 * np.eye(n), np.zeros(n)
    if name == "periodic":
        t = rng.uniform(0, 5, (n, 1))
        spec = ("periodic", 1.5, ("stretched", 0.8, ("eq",)))
        return (S.GP(S.EQ().stretch(0.8).periodic(1.5))(t, 0.05), O.kernel_matrix(spec, t) + 0.05 * np.eye(n),
                np.zeros(n))
    if name == "blockdense":
        from stheno_b200.model.observations import combine

        n1 = n // 3
        x1, x2 = x[:n1], x[n1:]
        m = S.Measure()
        f = S.GP(S.EQ().stretch(1.2), measure=m)
        g = S.GP(0.7 * S.Matern52(), measure=m)
        h = f + g
        var = m(combine(f(x1, 0.2), h(x2, 0.1))).var
        assert type(var).__name__ == "BlockDense"
        kf, kh = ("stretched", 1.2, ("eq",)), ("sum", ("stretched", 1.2, ("eq",)), ("scaled", 0.7, ("matern52",)))
        K = O.mo_block_kernel([[kf, kf], [kf, kh]], [x1, x2])
        K[:n1, :n1] += 0.2 * np.eye(n1)
        K[n1:, n1:] += 0.1 * np.eye(n - n1)
        return S.Normal(var), K, np.zeros(n)
    if name == "woodbury":
        fdd = S.GP(0.4 * S.Linear())(x, 0.3)
        assert type(fdd.var).__name__ == "Woodbury"
        return fdd, 0.4 * x @ x.T + 0.3 * np.eye(n), np.zeros(n)
    raise ValueError(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hetero", "ard_sum", "periodic", "blockdense", "woodbury"])
@pytest.mark.parametrize("n", [129, 1000])
def test_values_models(S, name, n):
    rng = np.random.default_rng(n)
    fdd, Sigma, m = _model(S, name, n, rng)
    y = rng.standard_normal((n, 3))
    eps = 0.0 if name == "woodbury" else EPS  # the Woodbury routes regularise the r x r Schur complement, not Sigma
    mean_r, var, lp = loo_ref(Sigma, y - m[:, None], eps)
    mean, v = fdd.loo_marginals(y)
    _close(mean, mean_r + m[:, None], 1e-10)
    _close(v, var, 1e-10)
    _close(fdd.loo_logpdf(y), lp, 1e-10)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
def test_values_emulated(S, precision):
    """n = 6000: the factor, the solves and the streamed inverse diagonal run on the int8 emulation (not under "fp64")."""
    from stheno_b200 import ops

    S.B.precision = precision
    rng = np.random.default_rng(6000)
    n = 6000
    x = rng.standard_normal((n, 4))
    y = rng.standard_normal((n, 1))
    fdd = S.GP(S.EQ().stretch(1.5))(x, 0.1)
    ops.gemm_profile(True)
    try:
        err = _check(fdd, O.kernel_matrix(("stretched", 1.5, ("eq",)), x) + 0.1 * np.eye(n), y, np.zeros(n))
        n_oz = ops.gemm_profile_read(1)[2]
    finally:
        ops.gemm_profile(False)
    print(f"\n{precision}: max error {err:.2e}, emulated launches {n_oz}")
    assert (n_oz == 0) == (precision == "fp64")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [300, 2000])
def test_values_fp32(S, n):
    """fp32 within ``16 u kappa(Sigma)`` (u = 2^-24) of the fp64 closed form on the fp32-rounded inputs."""
    S.B.epsilon = 1e-6
    rng = np.random.default_rng(n)
    x = rng.standard_normal((n, 2)).astype(np.float32)
    y = rng.standard_normal((n, 1)).astype(np.float32)
    fdd = S.GP(S.EQ().stretch(np.float32(1.1)))(_dev(x, torch.float32), 0.1)
    Sigma = O.kernel_matrix(("stretched", float(np.float32(1.1)), ("eq",)), x.astype(np.float64)) + float(
        np.float32(0.1)) * np.eye(n)
    ev = np.linalg.eigvalsh(Sigma + 1e-6 * np.eye(n))
    bar = 16 * 2.0**-24 * ev[-1] / ev[0]
    mean_r, var, lp = loo_ref(Sigma, y.astype(np.float64), 1e-6)
    mean, v = fdd.loo_marginals(_dev(y, torch.float32))
    assert mean.dtype == torch.float32
    _close(mean.cpu(), mean_r[:, 0], bar)
    _close(v.cpu(), var, bar)
    lpg = fdd.loo_logpdf(_dev(y, torch.float32)).item()
    assert abs(lpg - lp[0]) <= bar * max(1.0, abs(lp[0])), (lpg, lp[0], bar)


@pytest.mark.gpu
def test_missing_data(S):
    rng = np.random.default_rng(11)
    n = 700
    x = rng.standard_normal((n, 2))
    y = rng.standard_normal(n)
    miss = rng.choice(n, 40, replace=False)
    y[miss] = np.nan
    obs = ~np.isnan(y)
    f = S.GP(0.5 + S.Matern52().stretch(0.9))
    for yy in (y, _dev(y)):  # host (checked eagerly) and device (flag read after the work is enqueued)
        fdd = f(x, 0.1)
        mean, var = fdd.loo_marginals(yy)
        mean, var = np.asarray(torch.as_tensor(mean).cpu()), np.asarray(torch.as_tensor(var).cpu())
        Sigma = O.kernel_matrix(("sum", ("scaled", 0.5, ("one",)), ("stretched", 0.9, ("matern52",))), x[obs]) + 0.1 * np.eye(
            obs.sum())
        mr, vr, lr = loo_ref(Sigma, y[obs, None])
        assert np.isnan(mean[~obs]).all() and np.isnan(var[~obs]).all()
        _close(mean[obs], mr[:, 0], 1e-10)
        _close(var[obs], vr, 1e-10)
        _close(float(fdd.loo_logpdf(yy)), lr[0], 1e-10)


# ---- 3. gradients --------------------------------------------------------------------------------------------------------
P0 = {"v1": 1.1, "l1": 0.9, "v2": 0.6, "l2": 1.4, "alpha": 1.7, "lin": 0.2, "noise": 0.12, "mean": 0.4}


def _ref_cov(p, x):
    d = lambda s: ((x[:, None, :] - x[None, :, :]) / s).pow(2).sum(-1)  # noqa: E731
    r2 = d(p["l1"])
    s = math.sqrt(3.0) * torch.sqrt(torch.clamp_min(r2, 1e-30))
    K = p["v1"] * (1 + s) * torch.exp(-s)
    K = K + p["v2"] * (1 + d(p["l2"]) / (2 * p["alpha"])) ** (-p["alpha"])
    return K + p["lin"] * (x @ x.T)


def ref_loo_logpdf(K, r):
    """``[k]`` LOO log densities of ``N(0, K)`` at ``r [n, k]`` in torch (``cholesky``, ``cholesky_inverse``)."""
    L = torch.linalg.cholesky(K)
    alpha = torch.cholesky_solve(r, L)
    c = torch.diagonal(torch.cholesky_inverse(L))
    s = alpha / c[:, None]
    return 0.5 * ((torch.log(c)[:, None] - alpha * s).sum(0) - K.shape[0] * O.LOG_2_PI)


def _ref_grads(x0, y0, t, w, values, hetero):
    p = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in values.items()}
    x, y = x0.clone().requires_grad_(True), y0.clone().requires_grad_(True)
    nz = p["noise"] * (1 + t) if hetero else p["noise"] * torch.ones_like(t)
    K = _ref_cov(p, x) + torch.diag(nz + EPS)
    lp = ref_loo_logpdf(K, y - p["mean"] * x[:, :1])
    (w * lp).sum().backward()
    g = {k: v.grad for k, v in p.items()}
    g.update(x=x.grad, y=y.grad)
    return lp.detach(), g


def _gpu_grads(S, x0, y0, t, w, values, hetero):
    p = {k: torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True) for k, v in values.items()}
    x, y = x0.cuda().requires_grad_(True), y0.cuda().requires_grad_(True)
    k = (p["v1"] * S.Matern32().stretch(p["l1"]) + p["v2"] * S.RQ(p["alpha"]).stretch(p["l2"]) + p["lin"] * S.Linear())
    nz = p["noise"] * (1 + t.cuda()) if hetero else p["noise"]
    fdd = S.GP(lambda z: p["mean"] * z[:, :1], k)(x, nz)
    assert type(fdd.var).__name__ == "KernelDense"
    lp = fdd.loo_logpdf(y)
    lp = lp.reshape(-1)
    (w.cuda() * lp).sum().backward()
    g = {k: v.grad.cpu() for k, v in p.items()}
    g.update(x=x.grad.cpu(), y=y.grad.cpu())
    return lp.detach().cpu(), g, fdd


def _inputs(n, k, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, dtype=torch.float64, generator=g) / math.sqrt(3)
    y = torch.sin(2 * x.sum(-1, keepdim=True)) + 0.5 * torch.randn(n, k, dtype=torch.float64, generator=g)
    t = torch.linspace(0, 1, n, dtype=torch.float64)
    w = torch.tensor([1.0, -0.5, 0.75][:k], dtype=torch.float64)
    return x, y, t, w


def _graph_nodes(t):
    names, seen, stack = set(), set(), [t.grad_fn]
    while stack:
        fn = stack.pop()
        if fn is None or fn in seen:
            continue
        seen.add(fn)
        names.add(type(fn).__name__)
        stack.extend(f for f, _ in fn.next_functions)
    return names


def _grad_errors(got, want):
    return {k: (got[k] - v).abs().max().item() / max(1.0, v.abs().max().item()) for k, v in want.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("hetero", [False, True])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("n", [1500, 2500])
def test_gradients(S, n, k, hetero):
    """Every coefficient, length scale, RQ alpha, the inputs, scalar or vector noise, ``y`` and a mean parameter."""
    x, y, t, w = _inputs(n, k, n + k)
    want_lp, want = _ref_grads(x, y, t, w, P0, hetero)
    lp, got, fdd = _gpu_grads(S, x, y, t, w, P0, hetero)
    assert ((lp - want_lp).abs() <= 1e-10 * want_lp.abs().clamp_min(1)).all(), (lp, want_lp)
    errs = _grad_errors(got, want)
    print(f"\nn={n} k={k} hetero={hetero}: " + " ".join(f"{a} {e:.1e}" for a, e in errs.items()))
    for name, e in errs.items():
        assert e <= 1e-8, (name, e)


@pytest.mark.gpu
def test_gradient_graph_is_analytic(S):
    x, y, _, _ = _inputs(300, 1, 5)
    l = torch.tensor(0.9, dtype=torch.float64, device="cuda", requires_grad=True)
    lp = S.GP(S.EQ().stretch(l))(x.cuda(), 0.1).loo_logpdf(y.cuda())
    assert "_KernelLooBackward" in _graph_nodes(lp)


@pytest.mark.gpu
def test_gradients_dense_blockdense_route(S):
    """A two-output joint whose parameters require grad: assembled densely, gradient w.r.t. the assembled covariance."""
    from stheno_b200.model.observations import combine

    rng = np.random.default_rng(8)
    n1, n2 = 600, 900
    x1, x2 = torch.tensor(rng.standard_normal((n1, 2))), torch.tensor(rng.standard_normal((n2, 2)))
    y = torch.tensor(rng.standard_normal(n1 + n2))

    def gpu():
        v = torch.tensor(0.7, dtype=torch.float64, device="cuda", requires_grad=True)
        l = torch.tensor(1.2, dtype=torch.float64, device="cuda", requires_grad=True)
        m = S.Measure()
        f = S.GP(S.EQ().stretch(l), measure=m)
        g = S.GP(v * S.Matern52(), measure=m)
        lp = m(combine(f(x1.cuda(), 0.2), (f + g)(x2.cuda(), 0.1))).loo_logpdf(y.cuda())
        assert "_DenseLooBackward" in _graph_nodes(lp)
        lp.backward()
        return lp.item(), v.grad.item(), l.grad.item()

    def ref():
        v = torch.tensor(0.7, dtype=torch.float64, requires_grad=True)
        l = torch.tensor(1.2, dtype=torch.float64, requires_grad=True)
        X = torch.cat([x1, x2])
        d2 = lambda a, b: (a[:, None, :] - b[None, :, :]).pow(2).sum(-1)  # noqa: E731
        kf = lambda a, b: torch.exp(-0.5 * d2(a, b) / l**2)  # noqa: E731
        r = torch.sqrt(torch.clamp_min(d2(x2, x2), 1e-30)) * math.sqrt(5.0)
        kg = v * (1 + r + r * r / 3) * torch.exp(-r)
        K = kf(X, X)
        K = K + torch.block_diag(0.2 * torch.eye(n1, dtype=torch.float64), kg + 0.1 * torch.eye(n2, dtype=torch.float64))
        lp = ref_loo_logpdf(K + EPS * torch.eye(n1 + n2, dtype=torch.float64), y[:, None])[0]
        lp.backward()
        return lp.item(), v.grad.item(), l.grad.item()

    got, want = gpu(), ref()
    assert abs(got[0] - want[0]) <= 1e-10 * max(1, abs(want[0])), (got, want)
    for a, b in zip(got[1:], want[1:]):
        assert abs(a - b) <= 1e-8 * max(1, abs(b)), (got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("rel_noise", [1e-2, 1e-4, 1e-6])
def test_conditioning_sweep(S, rel_noise):
    """Noise = rel_noise x the variance (1.9): the library's gradient errors against torch fp64 autograd on the host, beside
    the error of the same restatement run natively in fp64 on the GPU (cuSOLVER): ``err <= 10 err_native + 1e-10``."""
    values = dict(P0, noise=rel_noise * (P0["v1"] + P0["v2"]))
    x, y, t, w = _inputs(1500, 1, 77)
    _, want = _ref_grads(x, y, t, w, values, False)
    _, got, _ = _gpu_grads(S, x, y, t, w, values, False)
    _, native = _ref_grads_cuda(x, y, t, w, values)
    e_got, e_nat = _grad_errors(got, want), _grad_errors(native, want)
    print(f"\nnoise/variance {rel_noise:.0e}: library {max(e_got.values()):.1e}, native fp64 {max(e_nat.values()):.1e}")
    assert max(e_got.values()) <= 10 * max(e_nat.values()) + 1e-10, (e_got, e_nat)


def _ref_grads_cuda(x, y, t, w, values):
    p = {k: torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True) for k, v in values.items()}
    xc, yc = x.cuda().requires_grad_(True), y.cuda().requires_grad_(True)
    K = _ref_cov(p, xc) + torch.diag(p["noise"] * torch.ones_like(t.cuda()) + EPS)
    lp = ref_loo_logpdf(K, yc - p["mean"] * xc[:, :1])
    (w.cuda() * lp).sum().backward()
    g = {k: v.grad.cpu() for k, v in p.items()}
    g.update(x=xc.grad.cpu(), y=yc.grad.cpu())
    return lp.detach().cpu(), g


# ---- 4. full size --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_config2_full_size(S):
    """Config 2: n = 16384, d = 8, EQ().stretch(2), noise 0.1, fp64 "auto"."""
    rng = np.random.default_rng(2)
    n, d = 16384, 8
    x = rng.standard_normal((n, d))
    y = rng.standard_normal((n, 1))
    fdd = S.GP(S.EQ().stretch(2.0))(_dev(x), 0.1)
    mean, var = fdd.loo_marginals(_dev(y))
    lp = fdd.loo_logpdf(_dev(y)).item()
    Sigma = O.kernel_matrix(("stretched", 2.0, ("eq",)), x) + 0.1 * np.eye(n)
    mr, vr, lr = loo_ref(Sigma, y)
    print(f"\nconfig 2: mean {_close(mean.cpu(), mr[:, 0], 1e-10):.1e} var {_close(var.cpu(), vr, 1e-10):.1e} "
          f"lp {abs(lp - lr[0]) / abs(lr[0]):.1e}")
    assert abs(lp - lr[0]) <= 1e-10 * abs(lr[0])


# ---- 5. contracts --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_deterministic_and_equal_under_grad(S):
    rng = np.random.default_rng(9)
    n = 2500
    x = _dev(rng.standard_normal((n, 3)))
    y = _dev(rng.standard_normal((n, 2)))
    l = torch.tensor(1.3, dtype=torch.float64, device="cuda", requires_grad=True)
    nz = torch.tensor(0.1, dtype=torch.float64, device="cuda", requires_grad=True)
    fdd = S.GP(S.EQ().stretch(l))(x, nz)
    a, b = fdd.loo_logpdf(y), fdd.loo_logpdf(y)
    assert torch.equal(a, b)
    m1, v1 = fdd.loo_marginals(y)
    m2, v2 = fdd.loo_marginals(y)
    assert torch.equal(m1, m2) and torch.equal(v1, v2)
    with torch.no_grad():
        c = fdd.loo_logpdf(y)
        m3, v3 = fdd.loo_marginals(y)
    assert a.requires_grad and not c.requires_grad
    assert torch.equal(a.detach(), c) and torch.equal(m1.detach(), m3) and torch.equal(v1.detach(), v3)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "fp64"])
@pytest.mark.parametrize("n", [200, 5000])
def test_streamed_inverse_diag(S, n, precision):
    """``Chol.inverse_diag`` against the row norms of a full identity solve ``L^-T``."""
    from stheno_b200 import ops

    S.B.precision = precision
    rng = np.random.default_rng(n)
    xg = _dev(rng.standard_normal((1, 1, n, 3)))
    flat = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    ch = ops.chol_from_kernel(flat, xg, noise_scalar=0.1, jitter=EPS, full_precision=True)
    V = torch.zeros(1, ch.n_pad, ch.n_pad, dtype=torch.float64, device="cuda")
    V.diagonal(dim1=1, dim2=2).fill_(1.0)
    ch.solve_rows_(V)
    want = (V[0, :n] ** 2).sum(-1)
    for chunk in (128, 2048):
        got = ch.inverse_diag(chunk=chunk)[0]
        rel = ((got - want).abs() / want).max().item()
        assert rel <= 1e-13, (chunk, rel)


def _finish_ref(c, alpha, r, g):
    c, alpha, r, g = [t.double() for t in (c, alpha, r, g)]
    s = alpha / c.unsqueeze(1)
    lp = 0.5 * ((torch.log(c).unsqueeze(1) - alpha * s).sum(-1) - c.shape[-1] * O.LOG_2_PI)
    P = (g.unsqueeze(-1) * (1 + alpha * s)).sum(1) / (2 * c)
    return r - s, 1.0 / c, lp, P, g.unsqueeze(-1) * s


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_loo_finish_kernel(dtype):
    """``gpk_loo_finish`` against a torch fp64 restatement, on strided ``alpha``, with a NaN entry and ``c`` near the
    smallest normal number (``1 / c`` overflows to inf as the restatement's does)."""
    from stheno_b200 import ops

    g0 = torch.Generator().manual_seed(1)
    B, k, n = 2, 3, 1000
    c = torch.rand(B, n, generator=g0, dtype=torch.float64) + 0.1
    tiny = torch.finfo(dtype).tiny
    c[0, 5], c[1, 7] = 4 * tiny, tiny / 2
    alpha = torch.randn(B, k, n, generator=g0, dtype=torch.float64)
    alpha[1, 2, 100] = float("nan")
    r = torch.randn(B, k, n, generator=g0, dtype=torch.float64)
    g = torch.randn(B, k, generator=g0, dtype=torch.float64)
    c, alpha, r, g = [t.to(dtype) for t in (c, alpha, r, g)]
    abuf = torch.zeros(B, 128, 1024, dtype=dtype, device="cuda")
    abuf[:, :k, :n] = alpha.cuda()
    ad = abuf[:, :k, :n]  # ld 1024, batch stride 128 x 1024, as Chol.loo hands it over
    mean, var, lp = ops.loo_finish(c.cuda(), ad, r.cuda())
    P, q = ops.loo_finish(c.cuda(), ad, g=g.cuda())
    want = _finish_ref(c, alpha, r, g)
    tol = 1e-15 if dtype == torch.float64 else 1e-6
    for got, w in zip((mean, var, lp, P, q), want):
        got = got.cpu().double()
        w = w.to(dtype).double()  # the restatement rounded once, as the kernel rounds its fp64 result
        assert torch.equal(torch.isnan(got), torch.isnan(w))
        assert torch.equal(torch.isinf(got), torch.isinf(w))
        fin = torch.isfinite(w)
        assert ((got[fin] - w[fin]).abs() <= tol * w[fin].abs().clamp_min(1)).all()
    assert torch.isnan(lp[1, 2]) and torch.isfinite(lp[1, :2]).all()
    assert torch.isnan(mean[1, 2, 100]).item() and torch.isnan(P[1, 100]).item()
    again = ops.loo_finish(c.cuda(), ad, r.cuda())[2]
    assert torch.equal(torch.nan_to_num(lp), torch.nan_to_num(again))
