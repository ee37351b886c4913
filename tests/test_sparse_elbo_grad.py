"""Analytic, streamed gradient of the sparse ELBO (``PseudoObs*.elbo`` under grad; ``autograd.sparse_elbo``,
``ops.sparse_elbo_bwd``, ``gpk_sparse_rows_bwd``) against torch autograd through ``generic_grad.sparse_compute_torch``.

Notation (``observations.py:279-336``): ``L = chol(K_z + eps I)``, ``W = L^-1 K_zx`` with columns ``w_i``, ``q_i = |w_i|^2``,
``kappa_i`` = the noise for VFE / DTC and ``noise_i + kd_i - q_i`` for FITC, ``A = I + W diag(1/kappa) W^T``, ``s = A^-1 p``.
Per data point, ``u_i = A^-1 w_i``, ``r_i = ybar_i - s.w_i``, ``g_i = dE/dw_i``; ``H = sum_i g_i w_i^T``; then
``dE/dK_zx[:, i] = L^-T g_i`` and ``dE/dK_z = -1/2 L^-T H L^-1``.

The CPU test restates that chunked algorithm in torch (below) and checks it on this machine; the GPU tests run the library."""
import gc
import math

import numpy as np
import pytest
import torch

from stheno_b200.generic_grad import kernel_diag_torch, kernel_torch, sparse_compute_torch

METHODS = ["vfe", "fitc", "dtc"]


# ---- torch restatement of the chunked backward (host) --------------------------------------------------------------------
def chunked_elbo_grad(method, k_z, k_zx, k_x, z, x, kn, nz, ybar, eps, chunk, params):
    """Gradients of the ELBO w.r.t. ``params`` by the chunked algorithm of ``ops.sparse_elbo_bwd`` / ``autograd._SparseElbo``:
    the per-point step of ``gpk_sparse_rows_bwd``, ``H`` accumulated chunk by chunk, and the kernel matrices' vector-Jacobian
    products (what the K1-backward kernels contract) through torch."""
    n, m = x.shape[0], z.shape[0]
    eye = torch.eye(m, dtype=z.dtype)
    out = [torch.zeros_like(p) for p in params]

    def vjp(t, g):
        gs = torch.autograd.grad(t, params, g, retain_graph=True, allow_unused=True)
        for o, gi in zip(out, gs):
            if gi is not None:
                o += gi

    Kz = kernel_torch(k_z, z, z) + (torch.diag(nz) if nz is not None else 0.0)
    with torch.no_grad():
        L = torch.linalg.cholesky(Kz + eps * eye)
        A, p = eye.clone(), torch.zeros(m, dtype=z.dtype)
        for a in range(0, n, chunk):  # the forward, chunk by chunk
            W = torch.linalg.solve_triangular(L, kernel_torch(k_zx, z, x[a:a + chunk]), upper=False)
            kap = kn[a:a + chunk]
            if method == "fitc":
                kap = kap + kernel_diag_torch(k_x, x[a:a + chunk]) - (W * W).sum(0)
            A += (W / kap) @ W.T
            p += (W / kap) @ ybar[a:a + chunk]
        Ainv = torch.linalg.inv(A + eps * eye)
        s = Ainv @ p
        Li = torch.linalg.inv(L)
    H = torch.zeros(m, m, dtype=z.dtype)
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        Kc = kernel_torch(k_zx, z, x[a:b])
        kd = kernel_diag_torch(k_x, x[a:b]) if method != "dtc" else None
        with torch.no_grad():
            W = Li @ Kc
            U = Ainv @ W
            q = (W * W).sum(0)
            sig, yb = kn[a:b].detach(), ybar[a:b].detach()
            kap = sig + kd.detach() - q if method == "fitc" else sig
            r = yb - s @ W
            gk = (r * r + (W * U).sum(0) - kap) / (2 * kap ** 2)
            if method == "vfe":
                g_sig, g_kd, g_q = gk + (kd.detach() - q) / (2 * sig ** 2), -0.5 / sig, 0.5 / sig
            elif method == "fitc":
                g_sig, g_kd, g_q = gk, gk, -gk
            else:
                g_sig, g_kd, g_q = gk, None, torch.zeros_like(gk)
            G = (-U + s[:, None] * r) / kap + 2 * g_q * W
            H += G @ W.T
            g_Kc = Li.T @ G
        vjp(Kc, g_Kc)
        vjp(kn[a:b], g_sig)
        vjp(ybar[a:b], -r / kap)
        if kd is not None:
            vjp(kd, g_kd)
    vjp(Kz, -0.5 * Li.T @ H @ Li)
    return out


def _host_problem(method, n, m, d, seed):
    g = torch.Generator().manual_seed(seed)
    dt = torch.float64
    var = torch.tensor(1.3, dtype=dt, requires_grad=True)
    ell = torch.tensor(0.9, dtype=dt, requires_grad=True)
    c2 = torch.tensor(0.4, dtype=dt, requires_grad=True)
    x = torch.randn(n, d, dtype=dt, generator=g).requires_grad_()
    z = torch.randn(m, d, dtype=dt, generator=g).requires_grad_()
    kn = (0.05 + 0.1 * torch.rand(n, dtype=dt, generator=g)).requires_grad_()
    nz = (1e-3 + 1e-3 * torch.rand(m, dtype=dt, generator=g)).requires_grad_()
    y = torch.randn(n, dtype=dt, generator=g).requires_grad_()
    import stheno_b200 as S

    k = var * S.Matern52().stretch(ell) + c2 * S.EQ()
    return k, [var, ell, c2, x, z, kn, nz, y]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("chunk", [64, 30, 23])
def test_chunked_algorithm_matches_autograd_on_host(method, chunk):
    """1, 2 and 3 (ragged) chunks of 64 points against torch autograd through ``sparse_compute_torch``, fp64 on the CPU."""
    k, params = _host_problem(method, 64, 9, 2, 5)
    var, ell, c2, x, z, kn, nz, y = params
    eps = 1e-12
    elbo = sparse_compute_torch(method, k, k, k, z, x, kn, nz, y[:, None], torch.zeros(9, 1, dtype=x.dtype), eps)[3]
    want = torch.autograd.grad(elbo, params)
    got = chunked_elbo_grad(method, k, k, k, z, x, kn, nz, y, eps, chunk, params)
    for name, g_, w in zip(("var", "ell", "c2", "x", "z", "kn", "nz", "y"), got, want):
        err = float((g_ - w).abs().max()) / max(1.0, float(w.abs().max()))
        assert err <= 1e-10, (method, chunk, name, err)


# ---- the GPU --------------------------------------------------------------------------------------------------------------
@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.Measure, "default", None)
    return s


def _kernel(S, kind, T, d):
    """The kernel of case ``kind`` built from tensors ``T(v)`` that require grad."""
    if kind == "m52_eq":
        return T(1.2) * S.Matern52().stretch(T(1.7)) + T(0.3) * S.EQ()
    if kind == "eq_ard":
        return T(1.1) * S.EQ().stretch(T([0.8 + 0.3 * i for i in range(d)]))
    if kind == "m12":
        return T(0.9) * S.Matern12().stretch(T(1.4))
    if kind == "m32":
        return T(1.3) * S.Matern32().stretch(T(1.1))
    if kind == "rq":
        return T(1.0) * S.RQ(1.5).stretch(T(1.2))
    if kind == "linear":
        return T(0.8) * S.EQ().stretch(T(1.6)) * (T(0.5) * S.Linear())
    if kind == "delta":
        return T(1.2) * S.EQ().stretch(T(1.3)) + T(0.05) * S.Delta()
    raise ValueError(kind)


def _problem(S, method, n, m, d, *, kind="m52_eq", dtype=torch.float64, seed=0, noise="vector", nz="diag", interdomain=False):
    """``(elbo_fn, ref_fn, params)``: the library's ELBO and the ``sparse_compute_torch`` reference as functions of fresh models
    over the same leaf tensors ``params`` (every coefficient and length scale, x, z, the noise, y, the inducing noise and a mean
    parameter)."""
    g = torch.Generator().manual_seed(seed)
    dev = "cuda"
    params = []

    def T(v):
        t = torch.tensor(v, dtype=dtype, device=dev, requires_grad=True)
        params.append(t)
        return t

    def leaf(t):
        t = t.to(device=dev, dtype=dtype).requires_grad_()
        params.append(t)
        return t

    x = leaf(torch.randn(n, d, dtype=torch.float64, generator=g) / math.sqrt(d))
    z = leaf(torch.randn(m, d, dtype=torch.float64, generator=g) / math.sqrt(d))
    y = leaf(torch.sin(3 * x.detach().cpu().double().sum(-1)) + 0.3 * torch.randn(n, dtype=torch.float64, generator=g))
    sig = leaf(0.05 + 0.1 * torch.rand(n, dtype=torch.float64, generator=g)) if noise == "vector" else T(0.2)
    nzv = {"diag": lambda: leaf(1e-3 + 1e-3 * torch.rand(m, dtype=torch.float64, generator=g)), "scalar": lambda: T(1e-2),
           None: lambda: None}[nz]()
    b = T(0.3)
    k = _kernel(S, kind, T, d)
    kh = T(0.4) * S.Matern32().stretch(T(0.7)) if interdomain else None
    cls = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[method]

    def build():
        gp = S.GP(lambda t: b * t.sum(-1), k)
        f = gp + S.GP(kh, measure=gp.measure) if interdomain else gp
        return gp, f, cls(gp(z, nzv), f(x, sig), y)

    def elbo_fn():
        gp, f, obs = build()
        return obs.elbo(f.measure)

    def ref_fn():
        gp, f, obs = build()
        meas = f.measure
        kn = sig.expand(n) if sig.dim() == 0 else sig
        nzd = None if nzv is None else (nzv.expand(m) if nzv.dim() == 0 else nzv)
        ybar = y[:, None] - b * x.sum(-1, keepdim=True)
        return sparse_compute_torch(method, meas.kernels[gp], meas.kernels[gp, f], meas.kernels[f], z, x, kn, nzd, ybar,
                                    torch.zeros(m, 1, dtype=dtype, device=dev), S.B.epsilon)[3]

    return elbo_fn, ref_fn, params


def _grad(e, params):
    """``d e / d params``, zeros for the parameters ``e`` does not use (DTC does not read ``k_x``)."""
    gs = torch.autograd.grad(e, params, allow_unused=True)
    return [torch.zeros_like(p) if g_ is None else g_ for p, g_ in zip(params, gs)]


def _errors(got, want):
    return [float((a - w).abs().max()) / max(1.0, float(w.abs().max())) for a, w in zip(got, want)]


def _check_parity(S, method, n, m, d, bar=1e-8, **kw):
    elbo_fn, ref_fn, params = _problem(S, method, n, m, d, **kw)
    ref = ref_fn()
    want = _grad(ref, params)
    e = elbo_fn()
    assert e.requires_grad
    got = _grad(e, params)
    assert abs(float(e) - float(ref)) <= 1e-10 * max(1.0, abs(float(ref))), (float(e), float(ref))
    errs = _errors(got, want)
    print(f"\n{method} n={n} m={m} d={d} {kw}: max gradient error {max(errs):.2e}")
    assert max(errs) <= bar, errs
    return e, errs


SHAPES = {"1x1": (1, 1, 1, None), "200x7": (200, 7, 2, None), "700x37_c96": (700, 37, 3, 96),
          "700x37_c250": (700, 37, 3, 250), "3000x300": (3000, 300, 8, None)}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
@pytest.mark.parametrize("method", METHODS)
def test_gradients_match_autograd(S, monkeypatch, method, precision, shape):
    n, m, d, chunk = SHAPES[shape]
    monkeypatch.setattr(S.B, "precision", precision)
    if chunk:
        monkeypatch.setattr(S.B, "sparse_chunk", chunk)
    _check_parity(S, method, n, m, d, seed=n + m)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
@pytest.mark.parametrize("method", METHODS)
def test_gradients_emulated_shape(S, monkeypatch, method, precision):
    """n = 20000, m = 1100 (m_pad 1152) at chunk 16384: under "auto" / "int8x8" the solves and GEMMs of the backward (and the
    factor of K_z) run on the int8-slice emulation; two chunks, the second ragged."""
    monkeypatch.setattr(S.B, "precision", precision)
    _check_parity(S, method, 20000, 1100, 2, seed=3)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["eq_ard", "m12", "m32", "rq", "linear", "delta"])
@pytest.mark.parametrize("method", METHODS)
def test_gradients_kernels(S, method, kind):
    _check_parity(S, method, 500, 40, 3, kind=kind, seed=11)


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_gradients_scalar_noises_and_interdomain(S, method):
    """A scalar observation noise and a scalar inducing noise that require grad; then ``f = g + h`` observed through
    ``u = g(z)``, so that ``k_z``, ``k_zx`` and ``k_x`` differ, with no inducing noise."""
    _check_parity(S, method, 600, 30, 2, noise="scalar", nz="scalar", seed=21)
    _check_parity(S, method, 600, 30, 2, nz=None, interdomain=True, seed=22)


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_two_chunks_at_scale(S, method):
    _check_parity(S, method, 32768, 1024, 8, seed=7)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("method", METHODS)
def test_value_under_grad_equals_no_grad(S, monkeypatch, method, dtype):
    """The ELBO under grad is the no-grad ELBO bit for bit: the forward runs the no-grad launches, and every K_z here is
    factored with 8 slices either way (no scalar inducing noise of 1e-3 of the variance at m_pad >= 2048)."""
    if dtype == torch.float32:
        monkeypatch.setattr(S.B, "epsilon", 1e-6)
    for n, m, chunk in ((700, 37, 250), (20000, 2100, 16384)):
        monkeypatch.setattr(S.B, "sparse_chunk", chunk)
        elbo_fn, _, _ = _problem(S, method, n, m, 3, dtype=dtype, seed=m)
        e = elbo_fn()
        with torch.no_grad():
            e0 = elbo_fn()
        assert e.requires_grad and not e0.requires_grad
        assert torch.equal(e.detach(), e0), (n, m, float(e), float(e0))


#: fp32 bar: err <= C32 2^-24 kappa max(1, max |want|), kappa = the condition number of K_z + eps I (eps = 1e-6), as for the
#: fp32 log-pdf gradients (tests/test_logpdf_grad_paths.py).  DESIGN.md section 4 records the measured ratios.
C32 = 16.0


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_fp32_gradients(S, monkeypatch, method):
    monkeypatch.setattr(S.B, "epsilon", 1e-6)
    monkeypatch.setattr(S.B, "sparse_chunk", 400)
    n, m, d = 1000, 60, 3
    f32_fn, _, p32 = _problem(S, method, n, m, d, dtype=torch.float32, seed=9)
    _, ref_fn, p64 = _problem(S, method, n, m, d, dtype=torch.float64, seed=9)
    with torch.no_grad():  # the reference sees the fp32-rounded inputs and parameters
        for a, b in zip(p64, p32):
            a.copy_(b.double())
    e = f32_fn()
    got = torch.autograd.grad(e, p32)
    assert e.dtype == torch.float32 and all(g_.dtype == torch.float32 for g_ in got)
    ref = ref_fn()
    want = torch.autograd.grad(ref, p64)
    with torch.no_grad():  # p64: x, z, y, noise, inducing noise, mean parameter, then the kernel's
        k = _kernel(S, "m52_eq", lambda v: torch.tensor(v, dtype=torch.float64, device="cuda"), d)
        z = p64[1]
        Kz = kernel_torch(k, z, z) + torch.diag(p64[4]) + 1e-6 * torch.eye(m, dtype=torch.float64, device="cuda")
        ev = torch.linalg.eigvalsh(Kz)
        kappa = float(ev[-1] / ev[0])
    u = 2.0 ** -24
    errs = _errors([g_.double() for g_ in got], want)
    print(f"\n{method}: kappa {kappa:.3e} elbo rel {abs(float(e) - float(ref)) / abs(float(ref)):.2e} "
          + " ".join(f"{r / (u * kappa):.2e}" for r in errs))
    assert max(errs) <= C32 * u * kappa, (kappa, errs)
    assert abs(float(e) - float(ref)) <= 1e-4 * abs(float(ref))


@pytest.mark.gpu
def test_only_some_inputs_require_grad(S):
    """Only the noise, or only z, requires grad: the backward forms only what reaches them, and those gradients still match."""
    rng = np.random.default_rng(4)
    n, m, d = 900, 50, 2
    x = torch.tensor(rng.standard_normal((n, d)), device="cuda")
    z0 = torch.tensor(rng.standard_normal((m, d)), device="cuda")
    y = torch.tensor(rng.standard_normal(n), device="cuda")
    k = 1.2 * S.Matern52().stretch(0.8)
    for which in ("noise", "z"):
        sig = torch.tensor(0.1, device="cuda", dtype=torch.float64, requires_grad=which == "noise")
        z = z0.clone().requires_grad_(which == "z")
        t = sig if which == "noise" else z
        for method in METHODS:
            cls = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[method]
            f = S.GP(k)
            (got,) = torch.autograd.grad(cls(f(z), f(x, sig), y).elbo(f.measure), [t])
            ref = sparse_compute_torch(method, k, k, k, z, x, sig.expand(n), None, y[:, None],
                                       torch.zeros(m, 1, dtype=x.dtype, device="cuda"), S.B.epsilon)[3]
            (want,) = torch.autograd.grad(ref, [t])
            assert _errors([got], [want])[0] <= 1e-8, (which, method)


@pytest.mark.gpu
def test_batched_problem_keeps_the_generic_route(S):
    """A batched problem under grad is not streamed: it returns exactly what ``sparse_compute_torch`` returns."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(3, 80, 2, dtype=torch.float64, generator=g).cuda()
    z = torch.randn(3, 9, 2, dtype=torch.float64, generator=g).cuda()
    y = torch.randn(3, 80, 1, dtype=torch.float64, generator=g).cuda()
    ell = torch.tensor(1.3, dtype=torch.float64, device="cuda", requires_grad=True)
    k = S.EQ().stretch(ell)
    f = S.GP(k)
    e = S.PseudoObs(f(z), f(x, 0.2), y).elbo(f.measure)
    want = sparse_compute_torch("vfe", k, k, k, z, x, torch.full((3, 80), 0.2, dtype=torch.float64, device="cuda"), None, y,
                                torch.zeros(3, 9, 1, dtype=torch.float64, device="cuda"), S.B.epsilon)[3]
    assert torch.equal(e.detach(), want.detach())
    (ge,) = torch.autograd.grad(e.sum(), [ell])
    (gw,) = torch.autograd.grad(want.sum(), [ell])
    assert torch.equal(ge, gw)


@pytest.mark.gpu
@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("method", METHODS)
def test_mean_parameter_alone(S, method, batched):
    """Only a constant mean's parameter requires grad: the ELBO takes a gradient route (the analytic one unbatched, the torch
    restatement batched) and its gradient is the whole of ``dE/dc``, not just the part that ``y - m(x)`` carries."""
    g = torch.Generator().manual_seed(12)
    bs = (3,) if batched else ()
    x, z, y = (torch.randn(bs + s, dtype=torch.float64, generator=g).cuda() for s in ((80, 2), (9, 2), (80, 1)))
    c = torch.tensor(0.7, dtype=torch.float64, device="cuda", requires_grad=True)
    k = 1.1 * S.EQ().stretch(1.3)
    cls = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[method]
    f = S.GP(c * S.OneMean(), k)
    e = cls(f(z), f(x, 0.2), y).elbo(f.measure)
    ones = torch.ones(bs + (9, 1), dtype=torch.float64, device="cuda")
    want = sparse_compute_torch(method, k, k, k, z, x, torch.full(bs + (80,), 0.2, dtype=torch.float64, device="cuda"), None,
                                y - c, c * ones, S.B.epsilon)[3]
    (ge,) = torch.autograd.grad(e.sum(), [c])
    (gw,) = torch.autograd.grad(want.sum(), [c])
    assert _errors([ge], [gw])[0] <= 1e-8, (float(ge), float(gw))


@pytest.mark.gpu
def test_elbo_is_not_replaced_by_a_later_prediction(S):
    """The ELBO returned under grad stays the stored one when ``mu`` is asked for later (which takes the generic route)."""
    rng = np.random.default_rng(6)
    x, z, y = (torch.tensor(rng.standard_normal(s), device="cuda") for s in ((300, 2), (20, 2), (300,)))
    ell = torch.tensor(0.9, dtype=torch.float64, device="cuda", requires_grad=True)
    f = S.GP(S.EQ().stretch(ell))
    obs = S.PseudoObs(f(z), f(x, 0.1), y)
    e = obs.elbo(f.measure)
    mean = (f | obs)(x[:4]).mean
    assert obs.elbo(f.measure) is e and mean.requires_grad


# ---- config 4 -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_config4_memory_and_finite_differences(S):
    """BASELINE config 4 (n = 262144, m = 4096, d = 8, Matern52, fp64) under grad: the loss and every gradient in
    O(chunk m_pad + m_pad^2) memory, and the analytic directional derivative along 3 random directions in (variance, length
    scale, noise, z) against central differences of the streamed ELBO at two step sizes."""
    from stheno_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(4)
    n, m, d = 262144, 4096, 8
    x = torch.randn(n, d, device="cuda", dtype=torch.float64, generator=g)
    y = torch.randn(n, device="cuda", dtype=torch.float64, generator=g)
    z0 = torch.randn(m, d, device="cuda", dtype=torch.float64, generator=g)
    p0 = torch.tensor([1.0, 2.0, 0.1], dtype=torch.float64, device="cuda")

    def elbo(p, z):
        f = S.GP(p[0] * S.Matern52().stretch(p[1]))
        return S.PseudoObs(f(z), f(x, p[2]), y).elbo(f.measure)

    with torch.no_grad():
        elbo(p0, z0)  # warm the emulation scratch and the kernels
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    p = p0.clone().requires_grad_()
    z = z0.clone().requires_grad_()
    e = elbo(p, z)
    gp, gz = torch.autograd.grad(e, [p, z])
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    c_pad, m_pad = ops.round_up(S.B.sparse_chunk), ops.round_up(m)
    bound = 8 * (6 * c_pad * m_pad + 8 * m_pad * m_pad) + 64 * n * d
    print(f"\nconfig 4: elbo {float(e):.10e}, peak {peak / 2**20:.0f} MiB above the pre-call level (bound {bound / 2**20:.0f} MiB)")
    assert torch.isfinite(gp).all() and torch.isfinite(gz).all()
    assert peak <= bound, (peak, bound)
    gen = torch.Generator(device="cuda").manual_seed(5)
    for k in range(3):
        dp = torch.randn(3, device="cuda", dtype=torch.float64, generator=gen) * p0
        dz = torch.randn(m, d, device="cuda", dtype=torch.float64, generator=gen)
        ana = float((gp * dp).sum() + (gz * dz).sum())
        fds = []
        with torch.no_grad():
            for h in (1e-4, 1e-5):
                fds.append(float(elbo(p0 + h * dp, z0 + h * dz) - elbo(p0 - h * dp, z0 - h * dz)) / (2 * h))
        print(f"direction {k}: analytic {ana:.12e} fd(1e-4) {fds[0]:.12e} fd(1e-5) {fds[1]:.12e} "
              f"rel {abs(fds[0] - ana) / abs(ana):.2e} {abs(fds[1] - ana) / abs(ana):.2e} fd spread "
              f"{abs(fds[0] - fds[1]) / abs(ana):.2e}")
        assert min(abs(fd - ana) for fd in fds) <= 1e-6 * abs(ana), (k, ana, fds)
