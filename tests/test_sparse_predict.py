"""Marginals of sparse (``PseudoObs*``) posteriors streamed through ``gpk_sparse_posterior_marginals`` (``csrc/posterior.cu``).

``marginals()``, ``marginal_credible_bounds()`` and ``var_diag`` of a ``PosteriorMean`` / ``PosteriorKernel + SubspaceKernel``
pair of one problem evaluate the K1 rows ``k(x*, z)`` once per chunk of test points, solve a copy against ``L_z`` and another
against the factor of the stored ``A + eps I``, and reduce both in one pass.  Checked here against the oracle, against the
composition every other route still runs (``PosteriorMean.dev`` and the ``SumKernel`` element-wise evaluation, called
directly on the same objects), chunk by chunk, emulated, in fp32, for bounded device memory, at config 4's full size, and
for the routes that keep the composition."""
import contextlib
import os

import numpy as np
import pytest
import torch

from oracle import gp_oracle as O

METHODS = ["vfe", "fitc", "dtc"]
OBS = {"vfe": "PseudoObs", "fitc": "PseudoObsFITC", "dtc": "PseudoObsDTC"}
SPEC = ("sum", ("scaled", 1.2, ("stretched", 1.7, ("matern52",))), ("scaled", 0.3, ("eq",)))

# Bars against the oracle (fp64).  The posterior mean is a smooth function of ``mu``, which the streamed ELBO meets to
# rtol 1e-8 / atol 1e-10 (tests/test_sparse_accumulate.py): the same bar, relative to the largest |mean|.  Each variance term
# (``|L_z^-1 k|^2``, ``|L_S^-1 k|^2``) lies in [0, k(x*, x*)]; perturbing K_z and A by one rounding and refactorising moves the
# variance of these problems (d = 3, m <= 300, cond(K_z) <= 3e5) by at most 6e-12, so 1e-9 of the largest prior variance leaves
# more than two orders of magnitude for the tensor-core solves.  Both bars are far inside those of
# tests/test_model.py::test_sparse_vs_oracle (1e-6 / 1e-5).
MEAN_TOL = 1e-8
VAR_TOL = 1e-9
# Against the composition: the same factors and the same K1 rows, so only the order of the sums differs.
SAME_TOL = 1e-12


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


def host(v):
    return (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)).astype(np.float64).reshape(-1)


class Case:
    """A sparse posterior of ``n`` data points through ``m`` inducing points, its test points ``xs`` and the oracle's
    marginals there (diagonal of ``O.sparse_posterior``'s variance, with the prior means and inducing noise it leaves out)."""

    def __init__(self, S, method, m, ns, variant="plain", n=2000, d=3, seed=0, dtype=np.float64, eps=1e-12):
        rng = np.random.default_rng(seed)
        x, z, y = rng.uniform(-3, 3, (n, d)), rng.uniform(-3, 3, (m, d)), rng.standard_normal(n)
        noise = 0.05 + rng.uniform(0, 0.1, n)
        xs = rng.uniform(-3, 3, (ns, d))
        kernel, spec = 1.2 * S.Matern52().stretch(1.7) + 0.3 * S.EQ(), SPEC
        mean_fn = noise_z = None
        if variant == "prior_mean":
            mean_fn = lambda a: 0.5 * a.sum(-1) + 1.0  # noqa: E731
        elif variant == "noise_z":
            noise_z = 0.01 + rng.uniform(0, 0.05, m)
        elif variant == "delta":
            kernel = S.EQ().stretch(1.3) + 0.1 * S.Delta()
            spec = ("sum", ("stretched", 1.3, ("eq",)), ("scaled", 0.1, ("delta",)))
            xs[: min(ns, m) : 2] = z[: min(ns, m) : 2]  # test points on inducing points: Delta meets coincident pairs
        elif variant == "linear":
            kernel = S.EQ().stretch(1.5) + 0.5 * S.Matern32() * S.Linear().stretch(4.0)
            spec = ("sum", ("stretched", 1.5, ("eq",)), ("scaled", 0.5, ("product", ("matern32",), ("stretched", 4.0, ("linear",)))))
        elif variant == "xs_is_z":
            xs = z
        x, z, y, noise, xs = (a.astype(dtype) for a in (x, z, y, noise, xs))
        if noise_z is not None:
            noise_z = noise_z.astype(dtype)
        t = lambda a: torch.as_tensor(a, device="cuda")  # noqa: E731
        self.xs_np = xs.astype(np.float64)
        if mean_fn is None:
            f = S.GP(kernel)
        else:
            f = S.GP(lambda a: 0.5 * a.sum(-1, keepdim=True) + 1.0, kernel)
        self.f = f
        zd = t(z)
        u = f(zd) if noise_z is None else f(zd, t(noise_z))
        self.obs = getattr(S, OBS[method])(u, f(t(x), t(noise)), t(y))
        self.post = f | self.obs
        self.xs = t(xs)
        # the oracle, on the inputs the device saw
        x64, z64, y64, n64 = (a.astype(np.float64) for a in (x, z, y, noise))
        mx = mz = ms = None
        if mean_fn is not None:
            mx, mz, ms = mean_fn(x64), mean_fn(z64), mean_fn(self.xs_np)
        nz = None if noise_z is None else noise_z.astype(np.float64)
        c = O.sparse_compute(spec, z64, x64, n64, y64, method, noise_z=nz, mean_x=mx, mean_z=mz, eps=eps)
        Kzs = O.kernel_matrix(spec, z64, self.xs_np)
        mz_col = np.zeros((m, 1)) if mz is None else mz[:, None]
        self.mean_ref = O.iqf(c["K_z"], Kzs, c["mu"] - mz_col, eps=eps)[:, 0] + (0.0 if ms is None else ms)
        self.prior_var = O.kernel_elwise(spec, self.xs_np)[:, 0]
        self.var_ref = self.prior_var - O.iqf_diag(c["K_z"], Kzs, eps=eps) + O.iqf_diag(c["A"], Kzs, eps=eps)

    def routed(self, x=None):
        from stheno_b200 import kernels

        return kernels._sparse_posterior(self.post.mean, self.post.kernel, self.fdd().x if x is None else x)

    def fdd(self, xs=None):
        return self.post(self.xs if xs is None else xs)

    def composition(self):
        """Today's composition at ``xs``: ``PosteriorMean.dev`` and the ``SumKernel`` element-wise evaluation, the variances
        clamped at zero as ``marginals()`` clamps them."""
        from stheno_b200 import kernels

        xi = kernels.as_input(self.xs)
        with torch.no_grad():
            return self.post.mean.dev(xi), torch.clamp_min(kernels._elwise_any(self.post.kernel, xi, None, True), 0.0)

    def check_oracle(self, mean, var, mean_tol=MEAN_TOL, var_tol=VAR_TOL):
        mean, var = host(mean), host(var)
        m_scale = max(1.0, np.abs(self.mean_ref).max())
        v_scale = np.abs(self.prior_var).max()
        err_m = np.abs(mean - self.mean_ref).max() / m_scale
        err_v = np.abs(var - self.var_ref).max() / v_scale
        assert err_m <= mean_tol and err_v <= var_tol, (err_m, err_v)


def check_same(new, old, v_scale, tol=SAME_TOL):
    """``new`` against ``old`` (mean, variance): max |difference| relative to the largest |mean| (at least 1) and to
    ``v_scale``, the largest prior variance (which bounds each variance term)."""
    (m1, v1), (m0, v0) = new, old
    m1, v1, m0, v0 = map(host, (m1, v1, m0, v0))
    err_m = np.abs(m1 - m0).max() / max(1.0, np.abs(m0).max())
    err_v = np.abs(v1 - v0).max() / v_scale
    assert err_m <= tol and err_v <= tol, (err_m, err_v)


# ---- against the oracle and against the composition ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ns", [1, 127, 128, 129, 5000])
@pytest.mark.parametrize("m", [1, 37, 129, 300])
@pytest.mark.parametrize("method", METHODS)
def test_marginals_against_oracle_and_composition(S, method, m, ns):
    c = Case(S, method, m, ns, seed=m * 10 + ns)
    assert c.routed()
    mean, var = c.fdd().marginals()
    c.check_oracle(mean, var)
    check_same((mean, var), c.composition(), c.prior_var.max())


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["prior_mean", "noise_z", "delta", "linear", "xs_is_z"])
@pytest.mark.parametrize("method", METHODS)
def test_model_variants(S, method, variant):
    c = Case(S, method, 129, 300, variant=variant, seed=7)
    assert c.routed()
    fdd = c.fdd()
    mean, var = fdd.marginals()
    c.check_oracle(mean, var)
    check_same((mean, var), c.composition(), c.prior_var.max())
    # var_diag (variances only: no dot product, not clamped) and the credible bounds take the same route
    vd = c.fdd().var_diag
    assert np.array_equal(np.maximum(host(vd), 0.0), host(var))
    m2, lo, hi = c.fdd().marginal_credible_bounds()
    assert np.array_equal(host(m2), host(mean))
    np.testing.assert_allclose(host(hi) - host(m2), 1.96 * np.sqrt(host(var)), rtol=1e-12)


# ---- the ops call directly -----------------------------------------------------------------------------------------------
def _direct(c, xs, chunk, want_dot=True):
    from stheno_b200 import kernels, ops

    mean = c.post.mean
    flat, scales = mean.k_zi._flat()
    xi, zi = kernels.as_input(xs), mean.z
    return ops.sparse_posterior_marginals(flat, xi.scaled(scales), zi.scaled(scales), mean.K_z.chol(),
                                          c.post.kernel.b.A.chol(), mean._half_y()[0], want_dot=want_dot, chunk=chunk)


def bits(t):
    return t.view(torch.int64 if t.dtype == torch.float64 else torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("ns", [129, 385, 1000])
def test_ragged_chunks_bit_identical(S, ns):
    """Chunks of 128 test points, the last one ragged (385 = 3 x 128 + 1: a last chunk of one row), give the same bits as one
    chunk; without the dot product the variance terms are the same bits too."""
    c = Case(S, "vfe", 300, ns, seed=ns)
    with torch.no_grad():
        one = _direct(c, c.xs, chunk=4096)
        many = _direct(c, c.xs, chunk=128)
        nodot = _direct(c, c.xs, chunk=128, want_dot=False)
    assert nodot[0] is None
    for a, b in zip(one, many):
        assert torch.equal(bits(a), bits(b))
    for a, b in zip(one[1:], nodot[1:]):
        assert torch.equal(bits(a), bits(b))


# ---- emulated solves ------------------------------------------------------------------------------------------------------
def predicted_oz_solve_launches(lib, m_pad, c_pad, slices=8):
    """Emulated GEMMs of one recursive right solve of ``c_pad`` rows against an ``m_pad`` factor (``trsm_right_rec``)."""

    def solve(n):
        if n <= 128:
            return 0
        h = (n // 128 // 2) * 128
        return solve(h) + (1 if lib.gpk_gemm_nt_oz_ws_bytes(c_pad, n - h, h, slices) else 0) + solve(n - h)

    return solve(m_pad)


@pytest.mark.gpu
def test_emulated_solves(S):
    """m = 1200 (m_pad = 1280) and 5000 test points: the first chunk's two solves (4096 rows) have a 4096 x 640 x 640 product,
    which runs on the int8 emulation under "auto" and "int8x8" (8 slices, the posterior's policy) and on DMMA under "fp64".
    In d = 8: 1200 inducing points in d = 3 give cond(K_z) = 3e7, and one rounding of K_z and A then moves the variance by
    1.7e-9, beyond the bar whatever the solves do; in d = 8 cond(K_z) = 67 and that sensitivity is 5e-15."""
    from stheno_b200 import _lib

    lib = _lib.load()
    ns, m = 5000, 1200
    want = 2 * sum(predicted_oz_solve_launches(lib, 1280, c_pad) for c_pad in (4096, 1024))
    assert want >= 2
    out = {}
    for mode in ("auto", "int8x8", "fp64"):
        with precision(mode):
            c = Case(S, "vfe", m, ns, n=6000, d=8, seed=5)
            c.fdd(c.xs[:1]).marginals()  # the factors and L_z^-1 (mu - m_z) before the profiled call
            res = {}
            n_dmma, n_oz = profiled(lambda: res.update(mv=c.fdd().marginals()))
        assert n_oz == (0 if mode == "fp64" else want), (mode, n_oz, want)
        assert n_dmma > 0
        c.check_oracle(*res["mv"])
        out[mode] = res["mv"]
    for mode in ("auto", "int8x8"):
        check_same(out[mode], out["fp64"], c.prior_var.max(), tol=VAR_TOL)


# ---- fp32 -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_fp32(S, monkeypatch, method):
    """fp32 inputs with ``B.epsilon = 1e-6`` against the fp64 oracle on the fp32-rounded inputs: 1e-3 of the largest |mean|
    and of the largest prior variance (the bar form of tests/test_sparse_accumulate.py::test_fp32_streamed)."""
    monkeypatch.setattr(S.B, "epsilon", 1e-6)
    c = Case(S, method, 129, 1000, seed=31, dtype=np.float32, eps=1e-6)
    assert c.routed()
    mean, var = c.fdd().marginals()
    assert mean.dtype == torch.float32 and var.dtype == torch.float32
    c.check_oracle(mean, var, mean_tol=1e-3, var_tol=1e-3)


# ---- memory ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_memory_is_bounded(S):
    """m = 2048, n* = 2^20: the composition holds two n* x m_pad fp64 row buffers at once, 2 * 2^20 * 2048 * 8 B = 32 GiB (not
    run here).  The streamed call needs its workspace (two 4096 x 2048 buffers, 128 MiB), the emulation scratch of a 4096-row
    solve, and a few vectors of n* elements (prior terms, the three outputs, the sums) plus the stretched copy of x*."""
    from stheno_b200 import _lib, ops

    lib = _lib.load()
    ns, m, d = 2**20, 2048, 8
    rng = np.random.default_rng(8)
    x, z, y = rng.standard_normal((20000, d)), rng.standard_normal((m, d)), rng.standard_normal(20000)
    f = S.GP(S.Matern52().stretch(2.0))
    t = lambda a: torch.as_tensor(a, device="cuda")  # noqa: E731
    post = f | S.PseudoObs(f(t(z)), f(t(x), 0.1), t(y))
    xs = torch.randn(ns, d, dtype=torch.float64, device="cuda")
    with torch.no_grad():
        post(xs[:1]).marginals()
        fdd = post(xs)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        oz_before = sum(b.numel() for b in ops._OZ_SCRATCH.values())
        mean, var = fdd.marginals()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    m_pad, chunk = 2048, 4096
    ws = lib.gpk_sparse_posterior_ws_elems(chunk, m_pad) * 8
    oz = max(lib.gpk_trsm_right_oz_ws_bytes(m_pad, chunk, 8) + 1024, 64 << 20) if not oz_before else 0
    bound = ws + oz + ns * (d + 16) * 8
    old = 2 * ns * m_pad * 8
    assert peak <= bound, (peak, bound)
    assert bound < old // 40
    assert mean.shape == (ns,) and torch.isfinite(mean).all() and (var > 0).all()


# ---- routes that keep the composition -------------------------------------------------------------------------------------
@pytest.fixture(params=["cpu", pytest.param("gpu", marks=pytest.mark.gpu)])
def SB(request, monkeypatch):
    """The package on the GPU, or on the CPU with the torch stand-in backend: the routes below never reach the streamed call,
    so the routing is checked without a GPU too."""
    import stheno_b200 as s

    if request.param == "cpu":
        from tests import _cpu_backend

        _cpu_backend.install(monkeypatch)
    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.Measure, "default", None)
    return s


def check_composition(post, xs):
    """``post(xs)`` is not routed to the streamed call, and its marginals are those of the composition, bit for bit."""
    from stheno_b200 import kernels

    fdd = post(xs)
    assert not kernels._sparse_posterior(post.mean, post.kernel, fdd.x)
    mean, var = fdd.marginals()
    with torch.no_grad():
        xi = kernels.as_input(xs)
        m0, v0 = post.mean.dev(xi), kernels._elwise_any(post.kernel, xi, None, True)
    assert np.array_equal(host(mean), host(m0)) and np.array_equal(host(var), host(torch.clamp_min(v0, 0.0)))


def _batched_case(s):
    rng = np.random.default_rng(3)
    x, z, y = rng.uniform(-3, 3, (200, 3)), rng.uniform(-3, 3, (37, 3)), rng.standard_normal(200)
    f = s.GP(s.EQ().stretch(1.5))
    return f | s.PseudoObs(f(z), f(x, 0.1), y), rng.uniform(-3, 3, (2, 50, 3))


def test_batched_test_points_keep_the_composition(monkeypatch):
    """Batched test points of an unbatched sparse posterior, on the CPU stand-in: not routed, the composition's values."""
    import stheno_b200 as s
    from tests import _cpu_backend

    _cpu_backend.install(monkeypatch)
    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.Measure, "default", None)
    check_composition(*_batched_case(s))


@pytest.mark.gpu
def test_batched_test_points_are_not_routed(S):
    from stheno_b200 import kernels

    post, xs = _batched_case(S)
    assert not kernels._sparse_posterior(post.mean, post.kernel, post(xs).x)


def test_multi_output_inducing_points_keep_the_composition(SB):
    # as tests/test_model.py::test_combine_and_multi_fdd_observations
    rng = np.random.default_rng(30)
    m = SB.Measure()
    f1 = SB.GP(lambda t: t, SB.EQ(), measure=m)
    f2 = SB.GP(2.0 * SB.Matern32(), measure=m)
    x1, x2 = rng.standard_normal((4, 1)), rng.standard_normal((3, 1))
    y1, y2 = rng.standard_normal(4), rng.standard_normal(3)
    obs = SB.PseudoObs((f1(x1), f2(x2)), (f1(x1, 0.1), y1), (f2(x2, 0.2), y2))
    check_composition(f1 | obs, rng.standard_normal((6, 1)))


def test_cross_kernel_that_does_not_flatten_keeps_the_composition(SB):
    rng = np.random.default_rng(6)
    x, z, y = rng.uniform(0, 4, (300, 1)), np.linspace(0, 4, 20)[:, None], rng.standard_normal(300)
    f = SB.GP(SB.EQ().periodic(2.0))
    check_composition(f | SB.PseudoObs(f(z), f(x, 0.1), y), rng.uniform(0, 4, (40, 1)))


@pytest.mark.gpu
def test_grad_mode_keeps_the_composition_and_refuses_backward(S):
    """A kernel variance that requires grad: the values match the no-grad (streamed) ones and ``backward()`` raises."""
    from stheno_b200 import kernels

    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(200, 2, dtype=torch.float64, device="cuda", generator=g)
    z = torch.randn(30, 2, dtype=torch.float64, device="cuda", generator=g)
    xs = torch.randn(64, 2, dtype=torch.float64, device="cuda", generator=g)
    y = torch.sin(x[:, 0])

    def build(grad):
        v = torch.tensor(1.3, dtype=torch.float64, device="cuda", requires_grad=grad)
        f = S.GP(v * S.Matern52().stretch(1.5))
        post = f | S.PseudoObs(f(z), f(x, 0.1), y)
        fdd = post(xs)
        return kernels._sparse_posterior(post.mean, post.kernel, fdd.x), fdd.marginals()

    with torch.no_grad():
        routed, want = build(False)
    assert routed
    routed, got = build(True)
    assert not routed
    for a, b in zip(got, want):
        assert torch.allclose(a.detach(), b, rtol=1e-9, atol=1e-12)
    with pytest.raises(NotImplementedError):
        (got[0].sum() + got[1].sum()).backward()


# ---- config 4 at full size ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_config4_full_size(S):
    """BASELINE config 4 (n = 262144, m = 4096, d = 8, Matern52().stretch(2), noise 0.1, VFE): train without grad, predict at
    262144 points.  At 512 seeded indices: the composition evaluated at just those points to 1e-11 (the same factors; the
    solves of 4096-row chunks and of 512 rows split their products differently between the int8 emulation and DMMA), and the
    oracle built from ``sparse_compute_chunked``'s ``mu`` and ``A`` and ``K_z`` to 1e-9 of the largest |mean| and of the prior
    variance 1 (the bar of test_full_size_parity.py::test_c4_full_size_vs_oracle's ``mu``)."""
    try:
        import threadpoolctl

        threadpoolctl.threadpool_limits(limits=os.cpu_count() or 1)
    except Exception:
        pass
    from stheno_b200 import kernels

    rng = np.random.default_rng(4)
    n, m, d, ns = 262144, 4096, 8, 262144
    x, y = rng.standard_normal((n, d)), rng.standard_normal(n)
    z = np.random.default_rng(44).standard_normal((m, d))
    xs = np.random.default_rng(45).standard_normal((ns, d))
    idx = np.sort(np.random.default_rng(46).choice(ns, 512, replace=False))
    t = lambda a: torch.as_tensor(a, device="cuda")  # noqa: E731
    f = S.GP(S.Matern52().stretch(2.0))
    with torch.no_grad():
        post = f | S.PseudoObs(f(t(z)), f(t(x), 0.1), t(y))
        fdd = post(t(xs))
        assert kernels._sparse_posterior(post.mean, post.kernel, fdd.x)
        mean, var = fdd.marginals()
        xi = kernels.as_input(t(xs[idx]))
        m0, v0 = post.mean.dev(xi), torch.clamp_min(kernels._elwise_any(post.kernel, xi, None, True), 0.0)
    mean, var = host(mean), host(var)
    check_same((mean[idx], var[idx]), (m0, v0), 1.0, tol=1e-11)
    spec = ("stretched", 2.0, ("matern52",))
    c = O.sparse_compute_chunked(spec, z, x, 0.1, y, "vfe", chunk=16384, workers=min(16, max(1, (os.cpu_count() or 1) // 4)))
    Kzs = O.kernel_matrix(spec, z, xs[idx])
    mean_ref = O.iqf(c["K_z"], Kzs, c["mu"])[:, 0]
    var_ref = 1.0 - O.iqf_diag(c["K_z"], Kzs) + O.iqf_diag(c["A"], Kzs)
    err_m = np.abs(mean[idx] - mean_ref).max() / max(1.0, np.abs(mean_ref).max())
    err_v = np.abs(var[idx] - var_ref).max()
    assert err_m <= 1e-9 and err_v <= 1e-9, (err_m, err_v)
