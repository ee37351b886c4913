"""Gradients of sparse (``PseudoObs*``) posterior predictions with respect to the test inputs (``autograd._SparsePosteriorMarginals``
/ ``_SubspaceCov``, ``ops.sparse_posterior_marginals_bwd``, ``gpk_sparse_posterior_rows_bwd`` in ``csrc/posterior.cu``).

Nothing that feeds the approximation requires grad, so ``K_z``, the stored ``A`` and ``mu`` are constants.  The reference is
torch fp64 autograd on the host of a dense restatement built from those same matrices: ``K_z + eps I`` and ``A + eps I``
factorised by ``torch.linalg.cholesky``, ``mu``, and the cross kernel written out in torch."""
import contextlib
import math

import pytest
import torch

METHODS = ["vfe", "fitc", "dtc"]
OBS = {"vfe": "PseudoObs", "fitc": "PseudoObsFITC", "dtc": "PseudoObsDTC"}

# Bars.  The forward meets the oracle to MEAN_TOL = 1e-8 of the largest |mean| and VAR_TOL = 1e-9 of the largest prior variance
# (tests/test_sparse_predict.py); here the reference shares K_z, A and mu, so only the solves and the kernel derivative differ.
# The gradient in x*_i is dk(x*_i, z)/dx* contracted with the same solved rows the forward reduces: the mean's gradient with
# L_z^-T h (the forward's dot product), the variance's with L_z^-T v_i and L_S^-T u_i (the forward's squared norms).  Relative
# to the largest gradient entry (at least 1) each keeps its forward bar; 1e-8 covers both.  The acquisition mean + 2 sqrt(var)
# divides the variance's gradient by sqrt(var_i): its bar is 1e-8 / sqrt(min var) (at least 1e-8).
GRAD_TOL = 1e-8
# fp32 (B.epsilon = 1e-6, d = 8 so cond(K_z) stays small): the same contraction with fp32 solves, 1e-4 of the largest entry.
F32_TOL = 1e-4
SQRT5 = math.sqrt(5.0)


@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.Measure, "default", None)
    return s


@contextlib.contextmanager
def precision(mode):
    from stheno_b200 import B

    before = B.precision
    B.precision = mode
    try:
        yield
    finally:
        B.precision = before


def profiled(fn):
    """``fn()`` with the GEMM launch profile on: ``(native fp64 DMMA launches, emulated launches)``."""
    from stheno_b200 import ops

    ops.gemm_profile(True)
    try:
        fn()
        return ops.gemm_profile_read(0)[2], ops.gemm_profile_read(1)[2]
    finally:
        ops.gemm_profile(False)


def _kernel_ref(a, b):
    """``1.2 Matern52(|a - b| / 1.7) + 0.3 EQ(|a - b|)`` ``[n, m]`` in torch (differentiable in ``a``)."""
    d2 = ((a[:, None, :] - b[None, :, :]) ** 2).sum(-1)
    r = torch.sqrt(torch.clamp_min(d2, 1e-300)) / 1.7
    return 1.2 * (1 + SQRT5 * r + 5.0 / 3.0 * r * r) * torch.exp(-SQRT5 * r) + 0.3 * torch.exp(-0.5 * d2)


class Case:
    """A sparse posterior of ``n`` data points through ``m`` inducing points (zero prior mean, prior variance 1.5) and the host
    restatement of its predictions at the test points."""

    def __init__(self, S, method, m, ns, n=2000, d=3, seed=0, dtype=torch.float64):
        g = torch.Generator(device="cuda").manual_seed(seed)
        u = lambda *shape: (torch.rand(*shape, dtype=torch.float64, device="cuda", generator=g) * 6 - 3).to(dtype)  # noqa: E731
        x, z, self.xs0 = u(n, d), u(m, d), u(ns, d)
        y = torch.randn(n, dtype=torch.float64, device="cuda", generator=g).to(dtype)
        noise = (0.05 + 0.1 * torch.rand(n, dtype=torch.float64, device="cuda", generator=g)).to(dtype)
        f = S.GP(1.2 * S.Matern52().stretch(1.7) + 0.3 * S.EQ())
        self.post = f | getattr(S, OBS[method])(f(z), f(x, noise), y)
        from stheno_b200 import matrix as M

        with torch.no_grad():
            self.post(self.xs0[:1]).marginals()  # builds K_z, A, mu and the factors before anything is timed or profiled
            eps = S.B.epsilon
            host = lambda t: t.detach().to("cpu", torch.float64)  # noqa: E731
            Kz = host(M.dense(self.post.mean.K_z)).reshape(m, m)
            A = host(M.dense(self.post.kernel.b.A)).reshape(m, m)
            eye = torch.eye(m, dtype=torch.float64)
            self.Lz = torch.linalg.cholesky(Kz + eps * eye)
            self.LS = torch.linalg.cholesky(A + eps * eye)
            self.h = torch.linalg.solve_triangular(self.Lz, host(self.post.mean.y).reshape(m, 1), upper=False)[:, 0]
            self.z_h = host(z)

    def xs(self):
        return self.xs0.clone().requires_grad_(True)

    def ref(self, xs, want_cov=False):
        """Host ``(mean, var, cov or None)`` at ``xs`` (a leaf on the host) from the shared matrices."""
        R = _kernel_ref(xs, self.z_h)  # [ns, m]
        V = torch.linalg.solve_triangular(self.Lz, R.T, upper=False)
        U = torch.linalg.solve_triangular(self.LS, R.T, upper=False)
        mean = V.T @ self.h
        var = 1.5 - (V * V).sum(0) + (U * U).sum(0)
        cov = _kernel_ref(xs, xs) - V.T @ V + U.T @ U if want_cov else None
        return mean, var, cov


def acq(mean, var):
    return (mean + 2 * var.sqrt()).sum()


LOSSES = {
    "mean": lambda mean, var: mean.sum(),
    "var": lambda mean, var: var.sum(),
    "acq": acq,
}


def ref_grads(c, loss):
    xs = c.xs0.detach().to("cpu", torch.float64).requires_grad_(True)
    mean, var, _ = c.ref(xs)
    LOSSES[loss](mean, var).backward()
    return xs.grad, var.detach()


def check_grad(got, want, var, loss, tol=GRAD_TOL):
    got = got.detach().to("cpu", torch.float64)
    bar = tol * max(1.0, want.abs().max().item())
    if loss == "acq":
        bar /= min(1.0, math.sqrt(var.min().item()))
    err = (got - want).abs().max().item()
    assert err <= bar, (loss, err, bar)


def marginal_grads(c, loss, chunk=None):
    """``d loss / d x*`` through ``marginals()``, or, with ``chunk``, through the autograd function with that chunk."""
    from stheno_b200 import autograd, kernels

    xs = c.xs()
    if chunk is None:
        mean, var = c.post(xs).marginals()
    else:
        post = c.post
        xi = kernels.as_input(xs)
        flat, scales = post.mean.k_zi._flat()
        spec = autograd.SparsePosteriorSpec(flat, kernels.as_input(post.mean.z).scaled(scales), post.mean.K_z.chol(),
                                            post.kernel.b.A.chol(), post.mean._half_y()[0], chunk=chunk)
        prior_v = torch.full((xi.n, 1), 1.5, dtype=xs.dtype, device=xs.device)
        mean, var = autograd.sparse_posterior_marginals(spec, xi.scaled(scales), torch.zeros_like(prior_v), prior_v)
        mean, var = mean[:, 0], var[:, 0]
    LOSSES[loss](mean, var).backward()
    return xs.grad


# ---- marginals against the host restatement -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["auto", "fp64"])
@pytest.mark.parametrize("chunk", [None, 4096, 128])
@pytest.mark.parametrize("method", METHODS)
def test_marginal_gradients(S, method, chunk, mode):
    """300 test points: one chunk (``marginals()``, and the function with chunk 4096), and chunks of 128 with a ragged last
    one of 44 points."""
    with precision(mode):
        c = Case(S, method, 129, 300, seed=len(method) * 10 + (chunk or 1))
        for loss in LOSSES:
            want, var = ref_grads(c, loss)
            check_grad(marginal_grads(c, loss, chunk), want, var, loss)


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_emulated_backward(S, method):
    """m = 1200 (m_pad = 1280), 5000 test points in d = 8 (two chunks, the last ragged): under "auto" the backward's solves and
    products of the 4096-row chunk run on the int8 emulation, under "fp64" on DMMA only; both meet the host reference."""
    for mode in ("auto", "fp64"):
        with precision(mode):
            c = Case(S, method, 1200, 5000, n=6000, d=8, seed=5)
            want, var = ref_grads(c, "acq")
            xs = c.xs()
            mean, v = c.post(xs).marginals()
            loss = acq(mean, v)
            n_dmma, n_oz = profiled(loss.backward)
        assert n_dmma > 0
        assert (n_oz == 0) if mode == "fp64" else (n_oz > 0), (mode, n_oz)
        check_grad(xs.grad, want, var, "acq")


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_fp32(S, monkeypatch, method):
    monkeypatch.setattr(S.B, "epsilon", 1e-6)
    c = Case(S, method, 129, 1000, d=8, seed=31, dtype=torch.float32)
    for loss in LOSSES:
        want, var = ref_grads(c, loss)
        got = marginal_grads(c, loss)
        assert got.dtype == torch.float32
        check_grad(got, want, var, loss, tol=F32_TOL)


# ---- values and routing ---------------------------------------------------------------------------------------------------
def _nodes(t):
    seen, todo, names = set(), [t.grad_fn], []
    while todo:
        fn = todo.pop()
        if fn is None or fn in seen:
            continue
        seen.add(fn)
        names.append(type(fn).__name__)
        todo.extend(f for f, _ in fn.next_functions)
    return names


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_values_bit_identical_and_routed(S, method):
    from stheno_b200 import kernels

    c = Case(S, method, 129, 1000, seed=3)
    with torch.no_grad():
        fdd = c.post(c.xs0)
        m0, v0 = fdd.marginals()
        vd0 = fdd.var_diag
    xs = c.xs()
    fdd = c.post(xs)
    assert kernels._sparse_posterior(c.post.mean, c.post.kernel, fdd.x)
    m1, v1 = fdd.marginals()
    vd1 = c.post(xs).var_diag
    assert torch.equal(m0, m1.detach()) and torch.equal(v0, v1.detach()) and torch.equal(vd0, vd1.detach())
    for t in (m1, v1, vd1):
        assert "_SparsePosteriorMarginalsBackward" in _nodes(t)
        assert "_NoGradientBackward" not in _nodes(t)
    # var_diag alone (no dot product): its gradient is the variance's
    vd1.sum().backward()
    want, _ = ref_grads(c, "var")
    check_grad(xs.grad, want, None, "var")


# ---- full covariance ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["var", "mean_var"])
@pytest.mark.parametrize("method", METHODS)
def test_full_covariance(S, method, entry):
    """``sum(Gc o C)`` (+ ``sum(a o mean)``) with a non-symmetric ``Gc`` at 300 test points."""
    from stheno_b200 import matrix as M

    c = Case(S, method, 129, 300, seed=17)
    g = torch.Generator().manual_seed(1)
    Gc = torch.randn(300, 300, dtype=torch.float64, generator=g)
    a = torch.randn(300, dtype=torch.float64, generator=g)
    xs_h = c.xs0.detach().to("cpu", torch.float64).requires_grad_(True)
    mean, _, cov = c.ref(xs_h, want_cov=True)
    want_mean = entry == "mean_var"
    ((Gc * cov).sum() + ((a * mean).sum() if want_mean else 0.0)).backward()
    xs = c.xs()
    fdd = c.post(xs)
    if want_mean:
        mu, C = fdd.mean_var
        mu = mu[:, 0]
    else:
        mu, C = None, fdd.var
    C = M.dense(C)
    assert "_SubspaceCovBackward" in _nodes(C)
    loss = (Gc.cuda() * C).sum() + ((a.cuda() * mu).sum() if want_mean else 0.0)
    assert abs(loss.item() - ((Gc * cov).sum() + ((a * mean).sum() if want_mean else 0.0)).item()) <= 1e-8 * 300
    loss.backward()
    check_grad(xs.grad, xs_h.grad, None, entry)


# ---- the rows kernel alone ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("form", ["ab", "a", "b"])
def test_rows_kernel(form, dtype):
    """Random buffers of 384 rows with ld 384 > m_pad = 256, c = 300: rows 300 .. 383 are zeroed, the columns past m_pad and
    the rows past c_pad are left alone; NULL ``a`` or ``b`` count as zero (``V`` and ``U`` are then not read)."""
    from stheno_b200 import ops

    c, m_pad, ld, rows = 300, 256, 384, 512
    g = torch.Generator(device="cuda").manual_seed(2)
    r = lambda *s: torch.randn(*s, dtype=torch.float64, device="cuda", generator=g).to(dtype)  # noqa: E731
    V0, U0, h, a, b = r(rows, ld), r(rows, ld), r(m_pad), r(c), r(c)
    a = a if "a" in form else None
    b = b if "b" in form else None
    if b is None:  # not read: garbage must not leak through
        V0[:c, :m_pad] = float("nan")
        U0[:c, :m_pad] = float("nan")
    V, U = V0.clone(), U0.clone()
    fn = ops._fn("gpk_sparse_posterior_rows_bwd", dtype)
    rc = fn(c, m_pad, ops._ptr(V), ops._ptr(U), ld, ops._ptr(h if a is not None else None), ops._ptr(a), ops._ptr(b),
            ops._stream())
    ops.check(rc, "gpk_sparse_posterior_rows_bwd")
    torch.cuda.synchronize()
    V64, U64, h64 = V0.double()[:c, :m_pad], U0.double()[:c, :m_pad], h.double()
    wv = torch.zeros(c, m_pad, dtype=torch.float64, device="cuda")
    wu = torch.zeros_like(wv)
    if a is not None:
        wv += a.double()[:, None] * h64[None, :]
    if b is not None:
        wv -= 2 * b.double()[:, None] * V64
        wu = 2 * b.double()[:, None] * U64
    tol = dict(rtol=1e-14, atol=1e-14) if dtype == torch.float64 else dict(rtol=2e-7, atol=1e-6)
    torch.testing.assert_close(V[:c, :m_pad].double(), wv, **tol)
    torch.testing.assert_close(U[:c, :m_pad].double(), wu, **tol)
    assert (V[c:384, :m_pad] == 0).all() and (U[c:384, :m_pad] == 0).all()
    assert torch.equal(V[:, m_pad:], V0[:, m_pad:]) and torch.equal(U[:, m_pad:], U0[:, m_pad:])
    assert torch.equal(V[384:], V0[384:]) and torch.equal(U[384:], U0[384:])
    # no upstream at all is refused
    assert fn(c, m_pad, ops._ptr(V), ops._ptr(U), ld, ops._ptr(h), None, None, ops._stream()) != 0


# ---- Bayesian optimisation on a sparse posterior --------------------------------------------------------------------------
@pytest.mark.gpu
def test_sparse_bayesian_optimisation_steps(S):
    """``test_posterior_grad.py::test_bayesian_optimisation_steps`` on a ``PseudoObs`` posterior: maximise mu + 2 sigma over x*
    with torch.optim; the first gradient matches central differences of the forward."""
    from stheno_b200 import kernels

    S.B.epsilon = 1e-10
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.rand(400, 2, dtype=torch.float64, device="cuda", generator=g) * 4
    z = torch.rand(30, 2, dtype=torch.float64, device="cuda", generator=g) * 4
    y = torch.sin(x[:, 0]) * torch.cos(x[:, 1])
    f = S.GP(S.EQ().stretch(0.7))
    post = f | S.PseudoObs(f(z), f(x, 0.01), y)

    def acq_of(xs):
        mu, var = post(xs).marginals()
        return (mu + 2 * var.sqrt()).sum()

    xs = (torch.rand(8, 2, dtype=torch.float64, device="cuda", generator=g) * 4).requires_grad_(True)
    assert kernels._sparse_posterior(post.mean, post.kernel, post(xs).x)
    a0 = acq_of(xs)
    a0.backward()
    g0 = xs.grad.clone()
    h = 1e-6
    fd = torch.zeros_like(g0)
    with torch.no_grad():
        for i in range(xs.shape[0]):
            for j in range(xs.shape[1]):
                e = torch.zeros_like(xs)
                e[i, j] = h
                fd[i, j] = (acq_of(xs + e) - acq_of(xs - e)) / (2 * h)
    assert (g0 - fd).abs().max().item() <= 1e-6 * max(1.0, fd.abs().max().item())
    opt = torch.optim.Adam([xs], lr=0.05)
    for _ in range(10):
        opt.zero_grad()
        (-acq_of(xs)).backward()
        opt.step()
    with torch.no_grad():
        assert acq_of(xs).item() > a0.item()


# ---- memory ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_backward_memory_is_bounded(S):
    """n* = 262144, m = 1024 (m_pad = 1024), d = 8.  The composition would hold k(x*, z) for every test point, 2 GiB.  The
    backward needs its two 4096 x m_pad row buffers (64 MiB), one m_pad x m_pad block of copies for the transposed solves, the
    emulation scratch of a 4096-row solve if none is held yet, and a few n*-long vectors and n* x d gradients."""
    from stheno_b200 import _lib, ops

    lib = _lib.load()
    ns, m, d, chunk = 262144, 1024, 8, 4096
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(20000, d, dtype=torch.float64, device="cuda", generator=g)
    z = torch.randn(m, d, dtype=torch.float64, device="cuda", generator=g)
    y = torch.sin(x.sum(-1))
    f = S.GP(S.Matern52().stretch(2.0))
    post = f | S.PseudoObs(f(z), f(x, 0.1), y)
    xs = torch.randn(ns, d, dtype=torch.float64, device="cuda", generator=g).requires_grad_(True)
    mu, var = post(xs).marginals()
    loss = (mu + var).sum()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    oz_before = sum(b.numel() for b in ops._OZ_SCRATCH.values())
    torch.cuda.reset_peak_memory_stats()
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    m_pad = 1024
    oz = max(lib.gpk_trsm_right_oz_ws_bytes(m_pad, chunk, 8) + 1024, 64 << 20) if not oz_before else 0
    bound = 2 * chunk * m_pad * 8 + m_pad * m_pad * 8 + oz + ns * (4 * d + 16) * 8
    assert peak <= bound, (peak, bound)
    assert bound < ns * m_pad * 8 // 4
    assert torch.isfinite(xs.grad).all()
