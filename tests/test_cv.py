"""Multi-fold cross-validation (CV) predictive marginals and log densities: ``Normal.cv_marginals`` and ``Normal.cv_logpdf``.

For ``y ~ N(m, Sigma)``, ``Sigma = var + B.epsilon I``, ``r = y - m``, ``C = Sigma^-1``, ``alpha = C r`` and a fold ``I`` with
the block ``C_II``: ``mu_I = y_I - C_II^-1 alpha_I``, ``Cov_I = C_II^-1`` and
``log p(y_I | y_-I) = -1/2 |I| log 2 pi + 1/2 log det C_II - 1/2 alpha_I^T C_II^-1 alpha_I`` (Ginsbourger & Schaerer 2021).

  1. the closed form against explicit conditioning on ``y_-I`` (host, NumPy/SciPy), and on the host stand-ins of the CUDA
     ops: every covariance route, the singleton-fold (LOO) and one-fold (logpdf) identities, label handling, shapes;
  2. values on the GPU against the fp64 restatement: fold layouts, shapes, models, emulation, fp32, missing data, config 2;
  3. gradients of ``cv_logpdf`` against torch fp64 autograd of the dense restatement, and a conditioning sweep;
  4. contracts: determinism, values under grad, ``gpk_cv_finish`` on its own, peak memory of the forward."""
import math

import numpy as np
import pytest
import scipy.linalg as sla
import torch

from oracle import gp_oracle as O

EPS = 1e-12


# ---- fp64 references ----------------------------------------------------------------------------------------------------
def cv_ref(Sigma, r, labels, eps=EPS):
    """The closed form in fp64: ``(mean - m [n, k], var [n], lp [k])`` of ``N(0, Sigma + eps I)`` at ``r [n, k]``."""
    n = Sigma.shape[0]
    L = np.linalg.cholesky(Sigma + eps * np.eye(n)) if n <= 8192 else O.chol_eps(Sigma, eps)
    alpha = sla.cho_solve((L, True), r)
    C, info = sla.lapack.dpotri(L, lower=1)
    assert info == 0
    C = np.tril(C) + np.tril(C, -1).T
    mean_r, var, lp = np.empty_like(r), np.empty(n), np.zeros(r.shape[1])
    for lab in np.unique(labels):
        I = np.flatnonzero(labels == lab)
        Lc = np.linalg.cholesky(C[np.ix_(I, I)])
        e = sla.cho_solve((Lc, True), alpha[I])
        mean_r[I] = r[I] - e
        var[I] = np.diag(sla.cho_solve((Lc, True), np.eye(len(I))))
        lp += -0.5 * len(I) * O.LOG_2_PI + np.log(np.diag(Lc)).sum() - 0.5 * (alpha[I] * e).sum(0)
    return mean_r, var, lp


def cv_brute(Sigma, y, m, labels, eps=EPS):
    """Explicit conditioning of ``N(m, Sigma + eps I)`` on the entries outside each fold (one column ``y``)."""
    n = Sigma.shape[0]
    S = Sigma + eps * np.eye(n)
    mean, var, lp = np.empty(n), np.empty(n), 0.0
    for lab in np.unique(labels):
        I, o = labels == lab, labels != lab
        if o.any():
            W = np.linalg.solve(S[np.ix_(o, o)], S[np.ix_(o, I)])
            mu, cov = m[I] + W.T @ (y[o] - m[o]), S[np.ix_(I, I)] - S[np.ix_(I, o)] @ W
        else:
            mu, cov = m[I], S[np.ix_(I, I)]
        mean[I], var[I] = mu, np.diag(cov)
        Lc = np.linalg.cholesky(cov)
        z = sla.solve_triangular(Lc, y[I] - mu, lower=True)
        lp += -0.5 * (I.sum() * O.LOG_2_PI + z @ z) - np.log(np.diag(Lc)).sum()
    return mean, var, lp


def _close(got, want, bar):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    scale = max(1.0, float(np.abs(want).max()))
    err = float(np.abs(got - want).max())
    assert err <= bar * scale, (err, scale)
    return err / scale


def _unequal_labels(n, rng, K=4):
    """``K`` folds of unequal sizes, labels shuffled, sparse and negative."""
    cuts = np.sort(rng.choice(np.arange(1, n), K - 1, replace=False))
    lab = np.repeat(np.array([7, -3, 100, 2, 55, -40, 9, 13, 0, 4])[:K], np.diff(np.concatenate([[0], cuts, [n]])))
    return rng.permutation(lab)


# ---- 1. the closed form and the host routes ----------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 5, 23, 40])
def test_closed_form_equals_explicit_conditioning(n):
    rng = np.random.default_rng(n)
    x = rng.standard_normal((n, 2))
    Sigma = O.kernel_matrix(("stretched", 0.9, ("matern52",)), x) + 0.05 * np.diag(rng.uniform(1, 2, n))
    m, y = rng.standard_normal(n), rng.standard_normal(n)
    for lab in ([_unequal_labels(n, rng, min(4, n))] if n > 1 else []) + [np.zeros(n, int), np.arange(n)]:
        mean_r, var, lp = cv_ref(Sigma, (y - m)[:, None], lab)
        bm, bv, blp = cv_brute(Sigma, y, m, lab)
        np.testing.assert_allclose(mean_r[:, 0] + m, bm, rtol=1e-10, atol=1e-10 * np.abs(bm).max())
        np.testing.assert_allclose(var, bv, rtol=1e-10)
        np.testing.assert_allclose(lp[0], blp, rtol=1e-10)


def _install_cv_stand_ins(monkeypatch, cpu):
    """``Chol.cv`` on the host stand-ins: the fold blocks of the explicit inverse, factorised one by one."""

    def cv(self, r, sizes, want_mean=True):
        n = self.n
        C = torch.cholesky_inverse(torch.tril(self.W[:, : self.n_pad, :]))[:, :n, :n]
        alpha = self.full_solve(r)
        mean, var, lp, o = torch.empty_like(r), torch.empty(r.shape[0], n, dtype=r.dtype), 0.0, 0
        for s in sizes:
            Lc = torch.linalg.cholesky(C[:, o : o + s, o : o + s])
            aI = alpha[:, :, o : o + s].transpose(1, 2)
            e = torch.cholesky_solve(aI, Lc)
            mean[:, :, o : o + s] = r[:, :, o : o + s] - e.transpose(1, 2)
            var[:, o : o + s] = torch.diagonal(torch.cholesky_inverse(Lc), dim1=1, dim2=2)
            ldet = 2 * torch.log(torch.diagonal(Lc, dim1=1, dim2=2)).sum(-1)
            lp = lp + 0.5 * (ldet.unsqueeze(-1) - s * O.LOG_2_PI - (aI * e).sum(1))
            o += s
        return (mean if want_mean else None), var, lp, None

    monkeypatch.setattr(cpu.Chol, "cv", cv, raising=False)


@pytest.fixture
def host(cpu_backend, monkeypatch):
    from tests.test_loo import _install_loo_stand_ins

    _install_loo_stand_ins(monkeypatch, cpu_backend)
    _install_cv_stand_ins(monkeypatch, cpu_backend)
    import stheno_b200 as S

    return S


def test_host_routes_against_brute_force(host):
    """Kernel matrix (with a prior mean), dense, diagonal (= LOO) and Woodbury covariances, unequal shuffled folds."""
    S = host
    rng = np.random.default_rng(3)
    n = 30
    x = rng.standard_normal((n, 2))
    y = rng.standard_normal(n)
    lab = _unequal_labels(n, rng)
    spec = ("sum", ("stretched", 1.1, ("eq",)), ("scaled", 0.3, ("linear",)))
    fdd = S.GP(lambda t: 0.5 * t.sum(-1, keepdim=True), S.EQ().stretch(1.1) + 0.3 * S.Linear())(x, 0.1)
    assert type(fdd.var).__name__ == "KernelDense"
    Sigma = O.kernel_matrix(spec, x) + 0.1 * np.eye(n)
    m = 0.5 * x.sum(-1)
    bm, bv, blp = cv_brute(Sigma, y, m, lab)
    mean, var = fdd.cv_marginals(y, lab)
    assert mean.shape == (n,) and var.shape == (n,)
    _close(mean, bm, 1e-11)
    _close(var, bv, 1e-11)
    _close(fdd.cv_logpdf(y, lab), blp, 1e-11)
    dense = S.Normal(m[:, None], Sigma)
    _close(dense.cv_marginals(y, lab)[0], bm, 1e-11)
    _close(dense.cv_logpdf(y, lab), blp, 1e-11)

    d = rng.uniform(0.5, 2.0, n)
    diag = S.Normal(m[:, None], S.matrix.Diagonal(torch.tensor(d)))
    dm, dv = diag.cv_marginals(y, lab)
    _close(dm, m, 1e-15)
    _close(dv, d, 1e-15)
    _close(diag.cv_logpdf(y, lab), diag.loo_logpdf(y), 1e-15)

    wb = S.GP(0.7 * S.Linear())(x, 0.2)
    assert type(wb.var).__name__ == "Woodbury"
    wm, wv, wlp = cv_brute(0.7 * x @ x.T + 0.2 * np.eye(n), y, np.zeros(n), lab, eps=0.0)
    _close(wb.cv_marginals(y, lab)[0], wm, 1e-10)
    _close(wb.cv_marginals(y, lab)[1], wv, 1e-10)
    _close(wb.cv_logpdf(y, lab), wlp, 1e-10)


def test_host_structured_gradients(host):
    """Diagonal and Woodbury routes: torch-autograd gradients against autograd of the explicit conditioning."""
    S = host
    rng = np.random.default_rng(5)
    n = 25
    x = torch.tensor(rng.standard_normal((n, 2)))
    y = torch.tensor(rng.standard_normal(n))
    lab = _unequal_labels(n, rng, 3)

    def brute(Sigma):
        lp = 0.0
        for l in np.unique(lab):
            I, o = torch.tensor(lab == l), torch.tensor(lab != l)
            W = torch.linalg.solve(Sigma[o][:, o], Sigma[o][:, I])
            mu, cov = W.T @ y[o], Sigma[I][:, I] - Sigma[I][:, o] @ W
            lp = lp + torch.distributions.MultivariateNormal(mu, cov).log_prob(y[I])
        return lp

    for kind in ("woodbury", "diagonal"):
        s = torch.tensor(0.7, dtype=torch.float64, requires_grad=True)
        nz = torch.tensor(0.2, dtype=torch.float64, requires_grad=True)
        if kind == "woodbury":
            got = S.GP(s * S.Linear())(x, nz).cv_logpdf(y, lab)
            want = brute(s * x @ x.T + nz * torch.eye(n, dtype=torch.float64))
        else:
            d = torch.tensor(rng.uniform(0.5, 2.0, n))
            got = S.Normal(S.matrix.Diagonal(s * d + nz, origin=torch.device("cpu"))).cv_logpdf(y, lab)
            want = brute(torch.diag(s * d + nz))
        g1 = torch.autograd.grad(got, (s, nz))
        g2 = torch.autograd.grad(want, (s, nz))
        assert abs(got.item() - want.item()) <= 1e-10 * max(1, abs(want.item()))
        for a, b in zip(g1, g2):
            assert abs(a.item() - b.item()) <= 1e-9 * max(1, abs(b.item())), (kind, g1, g2)


def test_host_identities(host):
    """Singleton folds give leave-one-out, a single fold the prior marginals and ``logpdf``."""
    S = host
    rng = np.random.default_rng(6)
    n = 20
    x = rng.standard_normal((n, 1))
    y = rng.standard_normal(n)
    fdd = S.GP(lambda t: 0.2 * t[..., :1], S.Matern32().stretch(0.8))(x, 0.1)
    for got, want in zip(fdd.cv_marginals(y, rng.permutation(n) * 3 - 7), fdd.loo_marginals(y)):
        _close(got, want, 1e-12)
    _close(fdd.cv_logpdf(y, np.arange(n)), fdd.loo_logpdf(y), 1e-12)
    mean, var = fdd.cv_marginals(y, np.full(n, 4))
    _close(mean, 0.2 * x[:, 0], 1e-12)
    _close(var, 1 + 0.1 + EPS + 0 * var, 1e-12)
    _close(fdd.cv_logpdf(y, np.full(n, 4)), fdd.logpdf(y), 1e-12)


def test_host_labels_shapes_missing_and_errors(host):
    S = host
    rng = np.random.default_rng(4)
    n, k = 24, 3
    x = rng.standard_normal((n, 1))
    fdd = S.GP(S.EQ())(x, 0.1)
    Y = rng.standard_normal((n, k))
    lab = _unequal_labels(n, rng)
    mean, var = fdd.cv_marginals(Y, lab)
    assert mean.shape == (n, k) and var.shape == (n,) and fdd.cv_logpdf(Y, lab).shape == (k,)
    for j in range(k):
        _close(mean[:, j], fdd.cv_marginals(Y[:, j], lab)[0], 1e-14)
    # relabelling (a bijection of labels, float integral labels, a torch tensor) changes nothing
    relab = {v: i for i, v in enumerate(np.unique(lab)[::-1])}
    for other in (np.array([relab[v] for v in lab]) * 5 - 11, lab.astype(float), torch.tensor(lab)):
        _close(fdd.cv_logpdf(Y, other), fdd.cv_logpdf(Y, lab), 1e-13)
    # batched: (B, n, 1) -> (B, n) marginals and (B,) log densities, one set of folds for every member
    xb = rng.standard_normal((2, n, 1))
    yb = rng.standard_normal((2, n, 1))
    fb = S.GP(S.EQ())(xb, 0.1)
    mb, vb = fb.cv_marginals(yb, lab)
    lb = fb.cv_logpdf(yb, lab)
    assert mb.shape == (2, n) and vb.shape == (2, n) and lb.shape == (2,)
    for b in range(2):
        one = S.GP(S.EQ())(xb[b], 0.1)
        _close(mb[b], one.cv_marginals(yb[b], lab)[0], 1e-13)
        _close(lb[b], one.cv_logpdf(yb[b], lab), 1e-13)
    # missing data: the observed sub-problem; a fold that is all missing contributes nothing
    y = Y[:, 0].copy()
    gone = lab == lab[0]
    y[gone] = np.nan
    y[np.flatnonzero(~gone)[:2]] = np.nan
    obs = ~np.isnan(y)
    sub = S.GP(S.EQ())(x[obs], 0.1)
    mean, var = fdd.cv_marginals(y, lab)
    assert np.isnan(mean[~obs]).all() and np.isnan(var[~obs]).all()
    _close(mean[obs], sub.cv_marginals(y[obs], lab[obs])[0], 1e-14)
    _close(var[obs], sub.cv_marginals(y[obs], lab[obs])[1], 1e-14)
    _close(fdd.cv_logpdf(y, lab), sub.cv_logpdf(y[obs], lab[obs]), 1e-14)
    # errors
    for bad in (lab[:-1], lab.reshape(2, -1), lab + 0.5, np.where(lab == lab[0], np.nan, lab), np.array(["a"] * n),
                lab > 0):
        with pytest.raises(ValueError):
            fdd.cv_logpdf(Y, bad)
    # the kernel-matrix marginals come from raw-pointer kernels: a backward through them raises
    l = torch.tensor(1.0, dtype=torch.float64, requires_grad=True)
    mean, _ = S.GP(S.EQ().stretch(l))(torch.tensor(x), 0.1).cv_marginals(torch.tensor(Y[:, 0]), lab)
    with pytest.raises(NotImplementedError, match="cv_marginals"):
        mean.sum().backward()


# ---- 2. values on the GPU -------------------------------------------------------------------------------------------------
@pytest.fixture
def S():
    import stheno_b200 as S

    before = S.B.epsilon, S.B.precision
    yield S
    S.B.epsilon, S.B.precision = before


def _dev(a, dtype=torch.float64):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device="cuda")


def _layout(name, n, rng):
    if name in ("K2", "K5", "K10"):
        return rng.permutation(np.arange(n) % int(name[1:]))
    if name == "blocks64":
        return rng.permutation(n) // 64  # scattered blocks of 64
    if name == "singleton":
        return rng.permutation(n)
    if name == "one":
        return np.zeros(n, int)
    if name == "mixed":  # several padded sizes interleaved in fold order, a singleton among them
        sizes, pattern = [], [60, 140, 90, 1, 130, 200, 50]
        while sum(sizes) < n:
            sizes.append(min(pattern[len(sizes) % len(pattern)], n - sum(sizes)))
        return rng.permutation(np.repeat(np.arange(len(sizes)), sizes))
    if name == "straddle":  # contiguous folds of 100: fold boundaries off every 128-row chunk boundary
        return (np.arange(n) // 100)[::-1].copy()
    raise ValueError(name)


def _check(fdd, Sigma, y, m, lab, bar=1e-10):
    mean_r, var, lp = cv_ref(Sigma, y - m[:, None], lab)
    mean, v = fdd.cv_marginals(y, lab)
    mean, v = np.asarray(torch.as_tensor(mean).cpu()), np.asarray(torch.as_tensor(v).cpu())
    k = y.shape[1]
    return max(_close(mean if k > 1 else mean[:, None], mean_r + m[:, None], bar), _close(v, var, bar),
               _close(np.atleast_1d(np.asarray(torch.as_tensor(fdd.cv_logpdf(y, lab)).cpu())), lp, bar))


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["K2", "K5", "K10", "blocks64", "singleton", "one", "straddle", "mixed"])
@pytest.mark.parametrize("n", [129, 1000, 2500])
def test_values_layouts(S, n, layout):
    rng = np.random.default_rng(n)
    x = rng.standard_normal((n, 3))
    y = rng.standard_normal((n, 2))
    lab = _layout(layout, n, rng)
    f = S.GP(lambda t: 0.3 * t[..., :1], 1.3 * S.EQ().stretch(0.9))
    Sigma = O.kernel_matrix(("scaled", 1.3, ("stretched", 0.9, ("eq",))), x) + 0.05 * np.eye(n)
    # one fold holding every entry inverts Sigma^-1 back to Sigma: its rounding error grows like kappa(Sigma)^2 u, here and
    # in the reference alike
    err = _check(f(x, 0.05), Sigma, y, 0.3 * x[:, 0], lab, 1e-8 if layout == "one" else 1e-10)
    print(f"\n{layout} n={n}: {err:.1e}")


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 17])
def test_values_columns_and_batch(S, k):
    rng = np.random.default_rng(k)
    n = 700
    x = rng.standard_normal((2, n, 2))
    y = rng.standard_normal((2, n, k))
    lab = _layout("K5", n, rng)
    f = S.GP(S.Matern52().stretch(1.1))
    for b in range(2):
        _check(f(x[b], 0.1), O.kernel_matrix(("stretched", 1.1, ("matern52",)), x[b]) + 0.1 * np.eye(n), y[b],
               np.zeros(n), lab)
    if k == 1:
        fdd = f(x, 0.1)
        mean, var = fdd.cv_marginals(y, lab)
        lp = fdd.cv_logpdf(y, lab)
        assert mean.shape == (2, n) and var.shape == (2, n) and lp.shape == (2,)
        for b in range(2):
            mr, vr, lr = cv_ref(O.kernel_matrix(("stretched", 1.1, ("matern52",)), x[b]) + 0.1 * np.eye(n), y[b], lab)
            _close(mean[b], mr[:, 0], 1e-10)
            _close(var[b], vr, 1e-10)
            _close(lp[b], lr[0], 1e-10)


def _model(S, name, n, rng):
    x = rng.standard_normal((n, 3))
    if name == "hetero":
        nv = rng.uniform(0.01, 0.3, n)
        return S.GP(S.EQ().stretch(1.2))(x, nv), O.kernel_matrix(("stretched", 1.2, ("eq",)), x) + np.diag(nv)
    if name == "matern_rq_sum":
        ls = np.array([0.7, 1.3, 2.1])
        k = S.Matern32().stretch(ls) + 0.5 * S.RQ(1.5).stretch(0.8) + 0.2 * S.Linear()
        spec = ("sum", ("sum", ("stretched", ls, ("matern32",)), ("scaled", 0.5, ("stretched", 0.8, ("rq", 1.5)))),
                ("scaled", 0.2, ("linear",)))
        return S.GP(k)(x, 0.1), O.kernel_matrix(spec, x) + 0.1 * np.eye(n)
    if name == "product":
        k = S.EQ().stretch(1.5) * S.Matern52().stretch(2.0)
        spec = ("product", ("stretched", 1.5, ("eq",)), ("stretched", 2.0, ("matern52",)))
        return S.GP(k)(x, 0.05), O.kernel_matrix(spec, x) + 0.05 * np.eye(n)
    if name == "blockdense":
        from stheno_b200.model.observations import combine

        n1 = n // 3
        x1, x2 = x[:n1], x[n1:]
        m = S.Measure()
        f = S.GP(S.EQ().stretch(1.2), measure=m)
        g = S.GP(0.7 * S.Matern52(), measure=m)
        var = m(combine(f(x1, 0.2), (f + g)(x2, 0.1))).var
        assert type(var).__name__ == "BlockDense"
        kf, kh = ("stretched", 1.2, ("eq",)), ("sum", ("stretched", 1.2, ("eq",)), ("scaled", 0.7, ("matern52",)))
        K = O.mo_block_kernel([[kf, kf], [kf, kh]], [x1, x2])
        K[:n1, :n1] += 0.2 * np.eye(n1)
        K[n1:, n1:] += 0.1 * np.eye(n - n1)
        return S.Normal(var), K
    raise ValueError(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hetero", "matern_rq_sum", "product", "blockdense"])
def test_values_models(S, name):
    rng = np.random.default_rng(1000)
    n = 1000
    fdd, Sigma = _model(S, name, n, rng)
    _check(fdd, Sigma, rng.standard_normal((n, 3)), np.zeros(n), _layout("K5", n, rng))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
def test_values_emulated(S, precision):
    S.B.precision = precision
    rng = np.random.default_rng(6000)
    n = 6000
    x = rng.standard_normal((n, 4))
    fdd = S.GP(S.EQ().stretch(1.5))(x, 0.1)
    err = _check(fdd, O.kernel_matrix(("stretched", 1.5, ("eq",)), x) + 0.1 * np.eye(n), rng.standard_normal((n, 1)),
                 np.zeros(n), _layout("K5", n, rng))
    print(f"\n{precision}: max error {err:.2e}")


@pytest.mark.gpu
def test_values_fp32(S):
    """fp32 within ``16 u kappa(Sigma)`` (u = 2^-24) of the fp64 closed form on the fp32-rounded inputs."""
    S.B.epsilon = 1e-6
    rng = np.random.default_rng(300)
    n = 1500
    x = rng.standard_normal((n, 2)).astype(np.float32)
    y = rng.standard_normal((n, 1)).astype(np.float32)
    lab = _layout("K5", n, rng)
    fdd = S.GP(S.EQ().stretch(np.float32(1.1)))(_dev(x, torch.float32), 0.1)
    Sigma = O.kernel_matrix(("stretched", float(np.float32(1.1)), ("eq",)), x.astype(np.float64)) + float(
        np.float32(0.1)) * np.eye(n)
    ev = np.linalg.eigvalsh(Sigma + 1e-6 * np.eye(n))
    bar = 16 * 2.0**-24 * ev[-1] / ev[0]
    mean_r, var, lp = cv_ref(Sigma, y.astype(np.float64), lab, 1e-6)
    mean, v = fdd.cv_marginals(_dev(y, torch.float32), lab)
    assert mean.dtype == torch.float32
    _close(mean.cpu(), mean_r[:, 0], bar)
    _close(v.cpu(), var, bar)
    lpg = fdd.cv_logpdf(_dev(y, torch.float32), lab).item()
    assert abs(lpg - lp[0]) <= bar * max(1.0, abs(lp[0])), (lpg, lp[0], bar)


@pytest.mark.gpu
def test_missing_data(S):
    rng = np.random.default_rng(11)
    n = 700
    x = rng.standard_normal((n, 2))
    y = rng.standard_normal(n)
    lab = _layout("K10", n, rng)
    y[lab == 3] = np.nan  # a fold that is all missing
    y[rng.choice(n, 40, replace=False)] = np.nan
    obs = ~np.isnan(y)
    f = S.GP(0.5 + S.Matern52().stretch(0.9))
    Sigma = O.kernel_matrix(("sum", ("scaled", 0.5, ("one",)), ("stretched", 0.9, ("matern52",))), x[obs]) + 0.1 * np.eye(
        obs.sum())
    mr, vr, lr = cv_ref(Sigma, y[obs, None], lab[obs])
    for yy in (y, _dev(y)):
        fdd = f(x, 0.1)
        mean, var = fdd.cv_marginals(yy, lab)
        mean, var = np.asarray(torch.as_tensor(mean).cpu()), np.asarray(torch.as_tensor(var).cpu())
        assert np.isnan(mean[~obs]).all() and np.isnan(var[~obs]).all()
        _close(mean[obs], mr[:, 0], 1e-10)
        _close(var[obs], vr, 1e-10)
        _close(float(fdd.cv_logpdf(yy, lab)), lr[0], 1e-10)


@pytest.mark.gpu
def test_config2_full_size(S):
    """Config 2: n = 16384, d = 8, EQ().stretch(2), noise 0.1, fp64 "auto", K = 5."""
    rng = np.random.default_rng(2)
    n, d = 16384, 8
    x = rng.standard_normal((n, d))
    y = rng.standard_normal((n, 1))
    lab = _layout("K5", n, rng)
    fdd = S.GP(S.EQ().stretch(2.0))(_dev(x), 0.1)
    mean, var = fdd.cv_marginals(_dev(y), lab)
    lp = fdd.cv_logpdf(_dev(y), lab).item()
    mr, vr, lr = cv_ref(O.kernel_matrix(("stretched", 2.0, ("eq",)), x) + 0.1 * np.eye(n), y, lab)
    print(f"\nconfig 2: mean {_close(mean.cpu(), mr[:, 0], 1e-10):.1e} var {_close(var.cpu(), vr, 1e-10):.1e} "
          f"lp {abs(lp - lr[0]) / abs(lr[0]):.1e}")
    assert abs(lp - lr[0]) <= 1e-10 * abs(lr[0])


# ---- 3. gradients --------------------------------------------------------------------------------------------------------
P0 = {"v1": 1.1, "l1": 0.9, "v2": 0.6, "l2": 1.4, "alpha": 1.7, "lin": 0.2, "noise": 0.12, "mean": 0.4}


def _ref_cov(p, x):
    d = lambda s: ((x[:, None, :] - x[None, :, :]) / s).pow(2).sum(-1)  # noqa: E731
    s = math.sqrt(3.0) * torch.sqrt(torch.clamp_min(d(p["l1"]), 1e-30))
    K = p["v1"] * (1 + s) * torch.exp(-s)
    K = K + p["v2"] * (1 + d(p["l2"]) / (2 * p["alpha"])) ** (-p["alpha"])
    return K + p["lin"] * (x @ x.T)


def ref_cv_logpdf(K, r, lab):
    """``[k]`` fold log densities of ``N(0, K)`` at ``r [n, k]`` in torch, on ``K`` permuted to fold order."""
    perm = torch.as_tensor(np.argsort(lab, kind="stable"), device=K.device)
    K, r = K[perm][:, perm], r[perm]
    sizes = np.unique(lab, return_counts=True)[1]
    L = torch.linalg.cholesky(K)
    C = torch.cholesky_inverse(L)
    alpha = torch.cholesky_solve(r, L)
    lp, o = 0.0, 0
    for s in sizes:
        Lc = torch.linalg.cholesky(C[o : o + s, o : o + s])
        e = torch.cholesky_solve(alpha[o : o + s], Lc)
        lp = lp - 0.5 * s * O.LOG_2_PI + torch.log(torch.diagonal(Lc)).sum() - 0.5 * (alpha[o : o + s] * e).sum(0)
        o += s
    return lp


def _ref_grads(x0, y0, t, w, values, hetero, lab, device="cpu"):
    p = {k: torch.tensor(v, dtype=torch.float64, device=device, requires_grad=True) for k, v in values.items()}
    x, y = x0.to(device).clone().requires_grad_(True), y0.to(device).clone().requires_grad_(True)
    t = t.to(device)
    nz = p["noise"] * (1 + t) if hetero else p["noise"] * torch.ones_like(t)
    K = _ref_cov(p, x) + torch.diag(nz + EPS)
    lp = ref_cv_logpdf(K, y - p["mean"] * x[:, :1], lab)
    (w.to(device) * lp).sum().backward()
    g = {k: v.grad.cpu() for k, v in p.items()}
    g.update(x=x.grad.cpu(), y=y.grad.cpu())
    return lp.detach().cpu(), g


def _gpu_grads(S, x0, y0, t, w, values, hetero, lab):
    p = {k: torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True) for k, v in values.items()}
    x, y = x0.cuda().requires_grad_(True), y0.cuda().requires_grad_(True)
    k = (p["v1"] * S.Matern32().stretch(p["l1"]) + p["v2"] * S.RQ(p["alpha"]).stretch(p["l2"]) + p["lin"] * S.Linear())
    nz = p["noise"] * (1 + t.cuda()) if hetero else p["noise"]
    fdd = S.GP(lambda z: p["mean"] * z[:, :1], k)(x, nz)
    assert type(fdd.var).__name__ == "KernelDense"
    lp = fdd.cv_logpdf(y, lab).reshape(-1)
    assert "_KernelCVBackward" in _graph_nodes(lp)
    (w.cuda() * lp).sum().backward()
    g = {k: v.grad.cpu() for k, v in p.items()}
    g.update(x=x.grad.cpu(), y=y.grad.cpu())
    return lp.detach().cpu(), g


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
@pytest.mark.parametrize("layout,hetero,k", [("K5", False, 1), ("K10", True, 3), ("blocks64", False, 2),
                                             ("straddle", True, 1), ("mixed", True, 2), ("mixed", False, 1)])
def test_gradients(S, layout, hetero, k):
    """Every coefficient, length scale, RQ alpha, the inputs, scalar or vector noise, ``y`` and a mean parameter."""
    n = 1500
    x, y, t, w = _inputs(n, k, n + k)
    lab = _layout(layout, n, np.random.default_rng(k))
    want_lp, want = _ref_grads(x, y, t, w, P0, hetero, lab)
    lp, got = _gpu_grads(S, x, y, t, w, P0, hetero, lab)
    assert ((lp - want_lp).abs() <= 1e-10 * want_lp.abs().clamp_min(1)).all(), (lp, want_lp)
    errs = _grad_errors(got, want)
    print(f"\n{layout} hetero={hetero} k={k}: " + " ".join(f"{a} {e:.1e}" for a, e in errs.items()))
    for name, e in errs.items():
        assert e <= 1e-8, (name, e)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["K5", "mixed"])
def test_gradients_dense_blockdense_route(S, layout):
    from stheno_b200.model.observations import combine

    rng = np.random.default_rng(8)
    n1, n2 = 600, 900
    x1, x2 = torch.tensor(rng.standard_normal((n1, 2))), torch.tensor(rng.standard_normal((n2, 2)))
    y = torch.tensor(rng.standard_normal(n1 + n2))
    lab = _layout(layout, n1 + n2, rng)

    def run(device):
        v = torch.tensor(0.7, dtype=torch.float64, device=device, requires_grad=True)
        l = torch.tensor(1.2, dtype=torch.float64, device=device, requires_grad=True)
        if device == "cuda":
            m = S.Measure()
            f = S.GP(S.EQ().stretch(l), measure=m)
            g = S.GP(v * S.Matern52(), measure=m)
            lp = m(combine(f(x1.cuda(), 0.2), (f + g)(x2.cuda(), 0.1))).cv_logpdf(y.cuda(), lab)
            assert "_DenseCVBackward" in _graph_nodes(lp)
        else:
            X = torch.cat([x1, x2])
            d2 = lambda a, b: (a[:, None, :] - b[None, :, :]).pow(2).sum(-1)  # noqa: E731
            r = torch.sqrt(torch.clamp_min(d2(x2, x2), 1e-30)) * math.sqrt(5.0)
            K = torch.exp(-0.5 * d2(X, X) / l**2) + torch.block_diag(
                0.2 * torch.eye(n1, dtype=torch.float64),
                v * (1 + r + r * r / 3) * torch.exp(-r) + 0.1 * torch.eye(n2, dtype=torch.float64))
            lp = ref_cv_logpdf(K + EPS * torch.eye(n1 + n2, dtype=torch.float64), y[:, None], lab)[0]
        lp.backward()
        return lp.item(), v.grad.item(), l.grad.item()

    got, want = run("cuda"), run("cpu")
    assert abs(got[0] - want[0]) <= 1e-10 * max(1, abs(want[0])), (got, want)
    for a, b in zip(got[1:], want[1:]):
        assert abs(a - b) <= 1e-8 * max(1, abs(b)), (got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("rel_noise", [1e-2, 1e-4, 1e-6, 1e-8])
def test_conditioning_sweep(S, rel_noise):
    """Noise = rel_noise x the variance: the library's gradient errors against torch fp64 autograd on the host, beside the
    error of the same restatement run natively in fp64 on the GPU (cuSOLVER): ``err <= 10 err_native + 1e-10``."""
    values = dict(P0, noise=rel_noise * (P0["v1"] + P0["v2"]))
    x, y, t, w = _inputs(1500, 1, 77)
    lab = _layout("K5", 1500, np.random.default_rng(77))
    _, want = _ref_grads(x, y, t, w, values, False, lab)
    _, got = _gpu_grads(S, x, y, t, w, values, False, lab)
    _, native = _ref_grads(x, y, t, w, values, False, lab, device="cuda")
    e_got, e_nat = _grad_errors(got, want), _grad_errors(native, want)
    print(f"\nnoise/variance {rel_noise:.0e}: library {max(e_got.values()):.1e}, native fp64 {max(e_nat.values()):.1e}")
    assert max(e_got.values()) <= 10 * max(e_nat.values()) + 1e-10, (e_got, e_nat)


# ---- 4. contracts --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_deterministic_and_equal_under_grad(S):
    rng = np.random.default_rng(9)
    n = 2500
    x = _dev(rng.standard_normal((n, 3)))
    y = _dev(rng.standard_normal((n, 2)))
    lab = _layout("blocks64", n, rng)
    l = torch.tensor(1.3, dtype=torch.float64, device="cuda", requires_grad=True)
    nz = torch.tensor(0.1, dtype=torch.float64, device="cuda", requires_grad=True)
    fdd = S.GP(S.EQ().stretch(l))(x, nz)
    a, b = fdd.cv_logpdf(y, lab), fdd.cv_logpdf(y, lab)
    assert torch.equal(a, b)
    m1, v1 = fdd.cv_marginals(y, lab)
    m2, v2 = fdd.cv_marginals(y, lab)
    assert torch.equal(m1, m2) and torch.equal(v1, v2)
    with torch.no_grad():
        c = fdd.cv_logpdf(y, lab)
        m3, v3 = fdd.cv_marginals(y, lab)
    assert a.requires_grad and not c.requires_grad
    assert torch.equal(a.detach(), c) and torch.equal(m1.detach(), m3) and torch.equal(v1.detach(), v3)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_cv_finish_kernel(dtype):
    """``gpk_cv_finish`` against a torch fp64 restatement, on strided inputs, with a NaN entry."""
    from stheno_b200 import ops

    g0 = torch.Generator().manual_seed(1)
    B, k, n = 2, 3, 1000
    sizes = [1, 300, 64, 635]
    off = np.concatenate([[0], np.cumsum(sizes)])
    e, z, r = [torch.randn(B, k, n, generator=g0, dtype=torch.float64) for _ in range(3)]
    v = torch.rand(B, n, generator=g0, dtype=torch.float64) + 0.1
    ldet = torch.randn(B, len(sizes), generator=g0, dtype=torch.float64)
    g = torch.randn(B, k, generator=g0, dtype=torch.float64)
    z[1, 2, 100] = float("nan")
    e, z, r, v, ldet, g = [t.to(dtype) for t in (e, z, r, v, ldet, g)]
    bufs = []
    for t in (e, z):
        buf = torch.zeros(B, 128, 1024, dtype=dtype, device="cuda")
        buf[:, :k, :n] = t.cuda()
        bufs.append(buf[:, :k, :n])
    offsets = torch.tensor(off, device="cuda")
    mean, var, lp = ops.cv_finish(offsets, bufs[0], bufs[1], v.cuda(), ldet.cuda(), r.cuda())
    q, s = ops.cv_finish(offsets, bufs[0], g=g.cuda())
    d = [t.double() for t in (e, z, r, v, ldet, g)]
    want = (d[2] - d[0], d[3], 0.5 * (d[4].sum(1, keepdim=True) - n * O.LOG_2_PI - (d[1] ** 2).sum(-1)),
            d[5].unsqueeze(-1) * d[0], 0.5 * d[5].sum(1, keepdim=True).expand(B, len(sizes)))
    tol = 1e-15 if dtype == torch.float64 else 1e-6
    for got, w in zip((mean, var, lp, q, s), want):
        got, w = got.cpu().double(), w.to(dtype).double()
        assert torch.equal(torch.isnan(got), torch.isnan(w))
        fin = torch.isfinite(w)
        assert ((got[fin] - w[fin]).abs() <= tol * w[fin].abs().clamp_min(1)).all()
    assert torch.isnan(lp[1, 2]) and torch.isfinite(lp[1, :2]).all()
    again = ops.cv_finish(offsets, bufs[0], bufs[1], v.cuda(), ldet.cuda(), r.cuda())[2]
    assert torch.equal(torch.nan_to_num(lp), torch.nan_to_num(again))


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["K10", "blocks64"])
def test_forward_peak_memory(S, layout):
    """Beyond the factor, the forward holds one chunk of identity rows and the fold blocks: never a second ``n_pad^2``."""
    rng = np.random.default_rng(12)
    n = 8192
    x = _dev(rng.standard_normal((n, 4)))
    y = _dev(rng.standard_normal((n, 1)))
    lab = _layout(layout, n, rng)
    fdd = S.GP(S.EQ().stretch(1.5))(x, 0.1)
    fdd.cv_marginals(y, lab)  # warm-up: the emulation scratch is allocated once per stream
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fdd.cv_marginals(y, lab)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    n_pad2 = 8192 * 8192 * 8
    factor = (8192 + 128) * 8192 * 8
    print(f"\n{layout}: peak {peak / 2**20:.0f} MiB above the base, factor {factor / 2**20:.0f} MiB")
    assert peak < factor + 3 * n_pad2 // 4, peak
