"""``Normal.sample / entropy / kl`` and ``matrix.logdet / iqf / iqf_diag / ratio`` on every covariance type (``Diagonal``,
``Dense``, ``KernelDense``, ``BlockDense``, ``Woodbury``) against NumPy fp64 references built from ``oracle.gp_oracle``.

* Sampling is replayed exactly: the generator state is saved before ``sample`` and the same ``eps`` is drawn again, so
  ``s - mean`` is checked element by element against ``L eps`` -- with ``L`` the factor the product read, under the error
  bound of the GEMM path that ran (asserted on the in-situ launch profile), and end to end against the NumPy factor.
* ``entropy``, ``kl``, ``iqf_diag(a, b, c)`` with ``c != b`` and ``ratio`` at batch 1 and 3, in fp64 (native and emulated)
  and fp32; ``Woodbury`` against its dense matrix at ranks that pad to 128 and 256, including a missing-data submatrix.
* Missing data in device-resident observations (the asynchronous NaN flag, then ``submatrix``).
* Functions whose values come from raw-pointer kernels keep their values under grad mode and refuse a backward.

Every GPU case is marked ``gpu``; the guard test that also runs on the torch-CPU stand-in of the ops is not."""
import contextlib

import numpy as np
import pytest
import torch

from oracle import gp_oracle as O

U64, U32 = 2.0**-53, 2.0**-24
F64, F32 = torch.float64, torch.float32
#: emulated fp64 product with 8 int8 slices: |error| <= TOL8 rowmax(A) colmax(B) sqrt(K) (tests/test_gemm_paths.py)
TOL8 = 5e-15
#: Elements of ``s - mean`` sampled from the 7-slice factor that ``auto`` gives a well-conditioned ``KernelDense`` (EQ,
#: n = 2500, noise 0.1 of the variance) against ``L_ref eps``, relative to ``|L_ref| |eps|``: measured 4.4e-12 on an H100
#: 80GB HBM3 (700 W), against 1.1e-13 with 8 slices and 9.0e-14 native (factor elements: 4.2e-13, 1.1e-14 and 8.8e-15 of
#: max |L_ref|).  The bar leaves a factor of 2.3.
GAP_7_SLICES = 1e-11

gpu = pytest.mark.gpu


@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.B, "precision", "auto")
    monkeypatch.setattr(s.Measure, "default", None)
    return s


def _eps(dtype):
    return 1e-12 if dtype == F64 else 1e-6


@contextlib.contextmanager
def _setup(S, dtype, precision="auto"):
    S.B.epsilon, S.B.precision = _eps(dtype), precision
    yield


def _dev(a, dtype=F64):
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda").to(dtype)


def _host(t):
    """fp64 NumPy copy of a result (tensors, or arrays when the result's origin is NumPy)."""
    if isinstance(t, torch.Tensor):
        return t.detach().double().cpu().numpy()
    return np.asarray(t, np.float64)


def _rounded(a, dtype):
    """``a`` as the device holds it, in fp64."""
    return np.asarray(a, np.float32).astype(np.float64) if dtype == F32 else np.asarray(a, np.float64)


# ---- covariance types ---------------------------------------------------------------------------------------------
KF = ("stretched", 1.3, ("eq",))


def make_var(S, kind, n, batch, dtype, rng):
    """``(device matrix, dense fp64 reference [*bs, n, n], jitter the device adds before factorising)``."""
    bs = (batch,) if batch > 1 else ()
    eps = _eps(dtype)
    if kind == "diag":
        d = _rounded(rng.uniform(0.5, 1.5, bs + (n,)), dtype)
        K = np.zeros(bs + (n, n))
        K[..., np.arange(n), np.arange(n)] = d
        return S.matrix.Diagonal(_dev(d, dtype)), K, 0.0
    if kind == "dense":
        G = rng.standard_normal(bs + (n, n))
        K = _rounded(G @ np.swapaxes(G, -1, -2) / n + 0.5 * np.eye(n), dtype)
        return S.matrix.Dense(_dev(K, dtype)), K, eps
    if kind == "kernel":
        x = _rounded(rng.standard_normal(bs + (n, 2)), dtype)
        var = S.GP(S.EQ().stretch(1.3))(_dev(x, dtype), 0.1).var
        assert type(var).__name__ == "KernelDense"
        K = O.kernel_matrix(KF, x) + 0.1 * np.eye(n)
        return var, K, eps
    if kind == "woodbury":
        x = _rounded(rng.standard_normal(bs + (n, 3)), dtype)
        var = S.GP(0.7 * S.Linear())(_dev(x, dtype), 0.3).var
        assert type(var).__name__ == "Woodbury"
        return var, 0.7 * x @ np.swapaxes(x, -1, -2) + 0.3 * np.eye(n), 0.0
    if kind == "block":
        assert batch == 1
        var, K, _ = make_block(S, n, dtype, rng)
        return var, K, eps
    raise ValueError(kind)


def make_block(S, n, dtype, rng):
    """The joint of ``f(x1, 0.2)``, ``(f + 2 g)(x2, vector noise)``, ``g(x3)`` with blocks of 37, n - 42 and 5 points
    (as in tests/test_model.py::test_block_joint_with_unequal_blocks_and_mixed_noise): ``(var, dense reference, fdds)``."""
    from stheno_b200.model.observations import combine

    sizes = (37, n - 42, 5)
    xs = [_rounded(rng.standard_normal((k, 2)), dtype) for k in sizes]
    nv = _rounded(rng.uniform(0.1, 0.3, sizes[1]), dtype)
    m = S.Measure()
    f = S.GP(S.EQ().stretch(1.2), measure=m)
    g = S.GP(0.7 * S.Matern52(), measure=m)
    h = f + 2.0 * g
    fdds = (f(_dev(xs[0], dtype), 0.2), h(_dev(xs[1], dtype), _dev(nv, dtype)), g(_dev(xs[2], dtype)))
    kf, kg = ("stretched", 1.2, ("eq",)), ("scaled", 0.7, ("matern52",))
    kh, khg = ("sum", kf, ("scaled", 4.0, kg)), ("scaled", 2.0, kg)
    K = O.mo_block_kernel([[kf, kf, ("zero",)], [kf, kh, khg], [("zero",), khg, kg]], xs)
    K[:37, :37] += 0.2 * np.eye(37)
    K[37 : n - 5, 37 : n - 5] += np.diag(nv)
    var = m(combine(*fdds)).var
    assert type(var).__name__ == "BlockDense"
    return var, K, (m, fdds)


# ---- 1. sampling, replayed exactly ----------------------------------------------------------------------------------
def _replay(state, shape, dtype):
    g = torch.Generator(device="cuda")
    g.set_state(state)
    return torch.randn(shape, dtype=dtype, device="cuda", generator=g)


def _profiled(ops, fn):
    """``(result, launches of the fp64 DMMA GEMM, launches of the emulation)`` of ``fn()``."""
    ops.gemm_profile(True)
    try:
        out = fn()
        n_v3, n_oz = ops.gemm_profile_read(0)[2], ops.gemm_profile_read(1)[2]
    finally:
        ops.gemm_profile(False)
    return out, n_v3, n_oz


def _assert_path(path, n_v3, n_oz):
    if path in ("v2", "tf32x3"):  # v2 and the fp32 kernels are not profiled
        assert (n_v3, n_oz) == (0, 0), (path, n_v3, n_oz)
    elif path == "v3":
        assert (n_v3, n_oz) == (1, 0), (path, n_v3, n_oz)
    else:
        assert n_v3 == 0 and n_oz >= 1, (path, n_v3, n_oz)


def product_bound(path, L, eps, K):
    """Elementwise bound on ``|fl(L eps) - L eps|`` for the GEMM path that ran (``K`` = the padded reduction length)."""
    absprod = np.abs(L) @ np.abs(eps)
    if path in ("v2", "v3"):
        return 2 * K * U64 * absprod + 4 * U64 * absprod
    if path == "emulated":
        return TOL8 * np.abs(L).max(-1)[..., :, None] * np.abs(eps).max(-2)[..., None, :] * np.sqrt(K) + 4 * U64 * absprod
    # 3xTF32 with fp32 accumulation: the standard bound of an fp32 sum of K products.  The 6e-6 max(|A| |B|) that
    # tests/test_gpu_primitives.py measures on zero-mean operands does not hold here: with the mostly positive rows of a
    # kernel factor at K = 2560 the error reached 1.0e-5 max(|L| |eps|) and, element by element, 2.1e-5 |L| |eps| (H100),
    # 14x inside this bound.
    return 2 * K * U32 * absprod


#: (path, n, num, batch, dtype, B.precision): the sampling product ``(L eps)^T = eps^T L^T`` is a GEMM with M = round_up(num),
#: N = K = n_pad; it is emulated for batch 1 under "auto" once M N K >= 1.5e9.
SAMPLE_CASES = [
    ("v2", 1, 1, 1, F64, "auto"),
    ("v2", 127, 130, 1, F64, "fp64"),
    ("v2", 128, 1, 1, F64, "auto"),
    ("v2", 129, 130, 1, F64, "auto"),
    ("v3", 700, 130, 1, F64, "fp64"),
    ("v3", 700, 1, 1, F64, "auto"),
    ("v3", 2500, 1, 1, F64, "fp64"),
    ("emulated", 2500, 300, 1, F64, "auto"),
    ("v2", 129, 130, 3, F64, "auto"),
    ("v3", 700, 130, 3, F64, "auto"),
    ("tf32x3", 1, 1, 1, F32, "auto"),
    ("tf32x3", 127, 130, 1, F32, "auto"),
    ("tf32x3", 700, 1, 3, F32, "auto"),
    ("tf32x3", 2500, 130, 1, F32, "auto"),
]


def _sample_case_id(c):
    return f"{c[0]}-n{c[1]}-num{c[2]}-b{c[3]}-{'f64' if c[4] == F64 else 'f32'}-{c[5]}"


def _check_product(path, ch, s, mean, eps, dtype):
    """``s - mean`` against ``L_dev eps`` in fp64, ``L_dev`` the factor the product read."""
    L = _host(ch.L())
    e = _host(eps).reshape(L.shape[:1] + eps.shape[-2:])
    P = L @ e
    got = (_host(s) - mean).reshape(P.shape)
    u = U64 if dtype == F64 else U32
    bound = product_bound(path, L, e, ch.n_pad) + 2 * u * (np.abs(P) + np.abs(mean).reshape(-1, P.shape[-2], 1))
    err = np.abs(got - P) / bound
    assert err.max() <= 1.0, (path, err.max())
    return L, e


@gpu
@pytest.mark.parametrize("case", SAMPLE_CASES, ids=_sample_case_id)
def test_sample_kernel_dense_replayed(S, case):
    """``KernelDense`` samples: the product on the path the shape selects, then end to end against NumPy's factor."""
    from stheno_b200 import ops

    path, n, num, batch, dtype, precision = case
    rng = np.random.default_rng(n + num + batch)
    with _setup(S, dtype, precision):
        var, K, jit = make_var(S, "kernel", n, batch, dtype, rng)
        mean = _rounded(rng.standard_normal(var.shape[:-1] + (1,)), dtype)
        nrm = S.Normal(_dev(mean, dtype), var)
        ch = var.chol()  # factorised outside the profiled window: only the sampling product is profiled
        g = torch.Generator(device="cuda").manual_seed(7)
        state = g.get_state()
        (_, s), n_v3, n_oz = _profiled(ops, lambda: nrm.sample(g, num))
        _assert_path(path, n_v3, n_oz)
        assert s.shape == var.shape[:-1] + (num,) and s.dtype == dtype
        eps = _replay(state, (ch.batch, n, num), dtype)
        _, e = _check_product(path, ch, s, mean.reshape(-1, n, 1), eps, dtype)
    if dtype == F64 and not (path == "emulated"):
        # end to end: every factor here is native fp64 or 8-slice, well inside 1e-10 of |L_ref| |eps|
        L_ref = O.chol_eps(K, jit).reshape(-1, n, n)
        ref = L_ref @ e
        got = (_host(s) - mean).reshape(ref.shape)
        assert (np.abs(got - ref) <= 1e-10 * (np.abs(L_ref) @ np.abs(e))).all()


@gpu
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
def test_sample_end_to_end_emulated_factor(S, precision, capsys):
    """n = 2500, num = 300 against ``L_ref = cholesky(K + noise + eps I)``.  Under ``auto`` this well-conditioned
    ``KernelDense`` is factorised with 7 int8 slices: its elements stay within ``GAP_7_SLICES`` (measured, written into
    DESIGN.md); with 8 slices or native fp64 the bar is 1e-10."""
    n, num = 2500, 300
    rng = np.random.default_rng(2500)
    with _setup(S, F64, precision):
        var, K, jit = make_var(S, "kernel", n, 1, F64, rng)
        nrm = S.Normal(var)
        g = torch.Generator(device="cuda").manual_seed(3)
        state = g.get_state()
        _, s = nrm.sample(g, num)
        eps = _host(_replay(state, (n, num), F64))
        L_dev = _host(var.chol().L())[0]
    L_ref = O.chol_eps(K, jit)
    scale = np.abs(L_ref) @ np.abs(eps)
    gap = float((np.abs(_host(s) - L_ref @ eps) / scale).max())
    gap_L = float(np.abs(L_dev - L_ref).max() / np.abs(L_ref).max())
    with capsys.disabled():
        print(f"\n[sample end to end, {precision}] max |s - L_ref eps| / (|L_ref| |eps|) = {gap:.3e}; "
              f"max |L_dev - L_ref| / max |L_ref| = {gap_L:.3e}")
    assert gap <= (GAP_7_SLICES if precision == "auto" else 1e-10), gap


@gpu
@pytest.mark.parametrize("kind", ["diag", "dense", "kernel_noise", "woodbury", "block"])
def test_sample_covariance_types(S, kind):
    """One case per covariance type, end to end against NumPy (and the product against the factor it read, where that
    factor is cached on the matrix)."""
    from stheno_b200 import ops

    rng = np.random.default_rng(11)
    num = 130
    g = torch.Generator(device="cuda").manual_seed(5)
    state = g.get_state()
    ch = None
    if kind == "block":
        n = 182
        var, K, (m, fdds) = make_block(S, n, F64, rng)
        (_, *parts), n_v3, n_oz = _profiled(ops, lambda: m.sample(g, num, *fdds))
        assert [p.shape for p in parts] == [(37, num), (140, num), (5, num)]
        s, mean, path = torch.cat(parts, dim=0), np.zeros((n, 1)), "v2"
    else:
        n, batch = {"diag": (129, 3), "dense": (700, 1), "kernel_noise": (129, 1), "woodbury": (300, 1)}[kind]
        var, K, jit = make_var(S, kind.replace("_noise", ""), n, batch, F64, rng)
        mean = rng.standard_normal(var.shape[:-1] + (1,))
        nrm = S.Normal(_dev(mean), var)
        path = "v3" if kind == "dense" else "v2"
        if kind == "dense":
            ch = var.chol()
        if kind == "kernel_noise":  # sample(noise=) adds to the symbolic matrix: a new KernelDense, factorised here
            (_, s), n_v3, n_oz = _profiled(ops, lambda: nrm.sample(g, num, noise=0.05))
            K = K + 0.05 * np.eye(n)
        else:
            (_, s), n_v3, n_oz = _profiled(ops, lambda: nrm.sample(g, num))
    _assert_path(path, n_v3, n_oz)
    if kind == "diag":  # sqrt(d) eps: one rounding in the root, one in the product, one in the mean
        eps = _host(_replay(state, var.shape[:-1] + (num,), F64))
        P = np.sqrt(np.diagonal(K, axis1=-2, axis2=-1))[..., None] * eps
        assert (np.abs(_host(s) - mean - P) <= 4 * U64 * (np.abs(P) + np.abs(mean))).all()
        return
    eps = _replay(state, (1, n, num), F64)
    if ch is not None:
        _check_product(path, ch, s, mean.reshape(-1, n, 1), eps, F64)
    e = _host(eps)[0]
    L_ref = O.chol_eps(K, 1e-12)
    ref = L_ref @ e
    assert (np.abs(_host(s).reshape(n, num) - mean.reshape(n, 1) - ref) <= 1e-10 * (np.abs(L_ref) @ np.abs(e))).all()


@gpu
@pytest.mark.parametrize("n", [700, 2500])
@pytest.mark.parametrize("order", ["logpdf_first", "sample_first"])
def test_sampling_shares_the_cached_factor(S, order, n):
    """``L_lower_`` zeroes the upper triangle of the CACHED factor in place: log-pdfs before and after a sample on the
    same FDD agree to 1e-12, and a posterior conditioned on that FDD still matches the oracle."""
    rng = np.random.default_rng(n)
    x, xs = rng.standard_normal((n, 2)), rng.standard_normal((50, 2))
    y = rng.standard_normal(n)
    f = S.GP(S.EQ().stretch(1.3))
    fd = f(_dev(x), 0.1)
    g = torch.Generator(device="cuda").manual_seed(1)
    ref = float(O.fdd_logpdf(KF, x, 0.1, y))
    if order == "logpdf_first":
        lp1 = float(fd.logpdf(_dev(y)))
        fd.sample(g, 3)
    else:
        fd.sample(g, 3)
        lp1 = float(fd.logpdf(_dev(y)))
    assert fd.var._chol is not None and fd.var._chol._upper_zeroed
    lp2 = float(fd.logpdf(_dev(y)))
    assert abs(lp2 - lp1) <= 1e-12 * abs(lp1), (lp1, lp2)
    assert abs(lp1 - ref) <= 1e-10 * abs(ref), (lp1, ref)
    post = f | (fd, _dev(y))
    mref, vref = O.posterior(KF, x, 0.1, y, xs)
    np.testing.assert_allclose(_host(post(_dev(xs)).mean), mref, rtol=1e-8, atol=1e-9)
    np.testing.assert_allclose(_host(S.B.dense(post(_dev(xs)).var)), vref, rtol=1e-7, atol=1e-8)


# ---- 2. entropy, kl, logdet, iqf_diag, ratio ------------------------------------------------------------------------
KINDS = ["diag", "dense", "kernel", "woodbury", "block"]
#: (B.precision, dtype, batch, n)
ALGEBRA_CASES = (
    [("auto", F64, 1, n) for n in (1, 127, 128, 129, 700, 2500)]
    + [("fp64", F64, 3, n) for n in (129, 700)]
    + [("fp64", F64, 1, 2500)]
    + [("auto", F32, 1, 700), ("auto", F32, 3, 129)]
)


def _case_id(c):
    return f"{c[0]}-{'f64' if c[1] == F64 else 'f32'}-b{c[2]}-n{c[3]}"


def _cond(*Ks):
    return max(float(np.linalg.cond(K).max()) for K in Ks)


def _tol(dtype, n, *Ks):
    """Relative bar on a sum of terms.  fp64: 1e-10.  fp32: a backward-stable Cholesky of ``K`` in fp32 is the exact
    factor of ``K + dK`` with ``|dK| <= c n u_32 |L| |L^T|``; each of logdet, ``x^T K^-1 x`` and ``tr(B^-1 A)`` then moves
    by at most about ``n u_32 cond(K)`` times its own magnitude (first order: ``tr(K^-1 dK)``, ``x^T K^-1 dK K^-1 x``), and
    so does rounding ``K`` itself to fp32.  The bar is ``n u_32 max cond`` relative to the sum of the terms' magnitudes."""
    return 1e-10 if dtype == F64 else max(n * U32 * _cond(*Ks), 10 * U32)


@gpu
@pytest.mark.parametrize("case", ALGEBRA_CASES, ids=_case_id)
@pytest.mark.parametrize("kind", KINDS)
def test_entropy_kl_iqf_ratio(S, kind, case):
    precision, dtype, batch, n = case
    if kind == "block" and (batch > 1 or n < 43):
        pytest.skip("the three-block joint is unbatched and has at least 43 points")
    rng = np.random.default_rng(n * 7 + batch)
    bs = (batch,) if batch > 1 else ()
    with _setup(S, dtype, precision):
        var, K, jit = make_var(S, kind, n, batch, dtype, rng)
        mp = _rounded(rng.standard_normal(bs + (n, 1)), dtype)
        p = S.Normal(_dev(mp, dtype), var)
        # the Diagonal / Dense partners: ratio's diag(a) / b.diag branch and its solve branch
        dq = _rounded(rng.uniform(0.5, 2.0, bs + (n,)), dtype)
        Kd = np.zeros(bs + (n, n))
        Kd[..., np.arange(n), np.arange(n)] = dq
        G = rng.standard_normal(bs + (n, n))
        Kq = _rounded(G @ np.swapaxes(G, -1, -2) / n + np.eye(n), dtype)
        mq = _rounded(rng.standard_normal(bs + (n, 1)), dtype)
        q_diag = S.Normal(_dev(mq, dtype), S.matrix.Diagonal(_dev(dq, dtype)))
        q_dense = S.Normal(_dev(mq, dtype), S.matrix.Dense(_dev(Kq, dtype)))
        e = S.B.epsilon
        checks = [
            ("kl(p, p)", lambda: p.kl(p), O.kl_terms(mp, K, mp, K, jit, jit), (K,)),
            ("kl(p, q_diag)", lambda: p.kl(q_diag), O.kl_terms(mp, K, mq, Kd, jit, 0.0), (K, Kd)),
            ("kl(q_diag, p)", lambda: q_diag.kl(p), O.kl_terms(mq, Kd, mp, K, 0.0, jit), (K, Kd)),
            ("kl(p, q_dense)", lambda: p.kl(q_dense), O.kl_terms(mp, K, mq, Kq, jit, e), (K, Kq)),
            ("kl(q_dense, p)", lambda: q_dense.kl(p), O.kl_terms(mq, Kq, mp, K, e, jit), (K, Kq)),
        ]
        for name, fn, terms, Ks in checks:
            got = _host(fn())
            ref = sum(terms) / 2
            scale = sum(np.abs(t) for t in terms) / 2
            err = np.abs(got - ref) / scale
            assert err.max() <= _tol(dtype, n, *Ks), (name, got, ref, err.max())
        got = _host(p.entropy())
        ld = O.logdet(K, jit)
        err = np.abs(got - O.entropy(K, jit)) / (np.abs(ld) + n * (O.LOG_2_PI + 1))
        assert err.max() <= _tol(dtype, n, K), ("entropy", err.max())
        got = _host(S.matrix.ratio(var, q_dense.var))
        ref = O.ratio(K, Kq, e)
        assert (np.abs(got - ref) / np.abs(ref)).max() <= _tol(dtype, n, K, Kq)
        # iqf_diag(a, b, c), c != b, 130 columns; bar relative to sqrt(b^T a^-1 b c^T a^-1 c) (Cauchy-Schwarz)
        b = _rounded(rng.standard_normal(bs + (n, 130)), dtype)
        c = _rounded(rng.standard_normal(bs + (n, 130)), dtype)
        got = _host(S.matrix.iqf_diag(var, _dev(b, dtype), _dev(c, dtype)))
        ref = O.iqf_diag(K, b, c, eps=jit)
        scale = np.sqrt(O.iqf_diag(K, b, eps=jit) * O.iqf_diag(K, c, eps=jit))
        assert got.shape == ref.shape
        assert (np.abs(got - ref) / scale).max() <= _tol(dtype, n, K)


# ---- 3. Woodbury against its dense matrix ---------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("batched", [False, True], ids=["single", "batched_left"])
@pytest.mark.parametrize("n", [50, 97, 1000])
@pytest.mark.parametrize("r", [3, 130])
def test_woodbury_against_dense(S, r, n, batched, dtype):
    """The Schur complement ``I + U^T D^-1 U`` is a GEMM with K = round_up(n, 32): at n = 50 in fp32 that is the FFMA
    kernel, at n = 1000 in fp64 the v3 kernel; r = 130 pads the complement to 256.  ``left`` batched over 3 with one
    diagonal for all; then the missing-data submatrix."""
    rng = np.random.default_rng(r * n)
    bs = (3,) if batched else ()
    M = S.matrix
    d = _rounded(rng.uniform(0.2, 0.6, n), dtype)
    U = _rounded(0.5 * rng.standard_normal(bs + (n, r)), dtype)
    K = U @ np.swapaxes(U, -1, -2) + np.diag(d)
    b = _rounded(rng.standard_normal(bs + (n, 5)), dtype)
    c = _rounded(rng.standard_normal(bs + (n, 5)), dtype)
    y = _rounded(rng.standard_normal(bs + (n, 1)), dtype)
    with _setup(S, dtype):
        W = M.Woodbury(M.Diagonal(_dev(d, dtype)), M.LowRank(_dev(U, dtype)))
        tol = _tol(dtype, n, K)
        ld = O.logdet(K, 0.0)
        assert (np.abs(_host(M.logdet(W)) - ld) <= tol * (np.abs(ld) + n)).all()
        scale_bc = np.sqrt(np.abs(O.iqf(K, b, eps=0.0)).max() * np.abs(O.iqf(K, c, eps=0.0)).max())
        assert (np.abs(_host(M.iqf(W, _dev(b, dtype), _dev(c, dtype))) - O.iqf(K, b, c, eps=0.0)) <= tol * scale_bc).all()
        qd = O.iqf_diag(K, b, eps=0.0)
        assert (np.abs(_host(M.iqf_diag(W, _dev(b, dtype))) - qd) <= tol * qd).all()
        qbc = O.iqf_diag(K, b, c, eps=0.0)
        got = _host(M.iqf_diag(W, _dev(b, dtype), _dev(c, dtype)))
        assert (np.abs(got - qbc) <= tol * np.sqrt(qd * O.iqf_diag(K, c, eps=0.0))).all()
        lp = _host(S.Normal(W).logpdf(_dev(y, dtype)))
        ref = O.normal_logpdf(None, K, y, eps=0.0)
        assert (np.abs(lp - ref) <= tol * (np.abs(ld) + n * O.LOG_2_PI + O.iqf_diag(K, y, eps=0.0)[..., 0])).all()
        keep = np.ones(n, bool)
        keep[[0, n // 2, n - 1]] = False
        sub = M.submatrix(W, torch.as_tensor(keep, device="cuda"))
        Ks = K[..., keep, :][..., :, keep]
        lds = O.logdet(Ks, 0.0)
        assert (np.abs(_host(M.logdet(sub)) - lds) <= tol * (np.abs(lds) + n)).all()
        qs = O.iqf_diag(Ks, b[..., keep, :], eps=0.0)
        assert (np.abs(_host(M.iqf_diag(sub, _dev(b[..., keep, :], dtype))) - qs) <= tol * qs).all()


# ---- 4. missing data on device-resident observations ----------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("kind", ["kernel", "woodbury", "diag"])
def test_missing_device_observations(S, kind, dtype):
    """NaNs in a CUDA ``y`` at rows 0, 127, 128 and n - 1: the device flag sends the log-pdf to ``submatrix``; evaluated
    twice in a row so that the flag ring is reused."""
    n = 300
    rng = np.random.default_rng(3)
    with _setup(S, dtype):
        var, K, jit = make_var(S, kind, n, 1, dtype, rng)
        mean = _rounded(rng.standard_normal((n, 1)), dtype)
        nrm = S.Normal(_dev(mean, dtype), var)
        y = _rounded(rng.standard_normal(n), dtype)
        y[[0, 127, 128, n - 1]] = np.nan
        keep = ~np.isnan(y)
        Kk = K[np.ix_(keep, keep)]
        ref = float(O.normal_logpdf(mean, K, y, eps=jit))
        tol = _tol(dtype, n, Kk)
        scale = abs(O.logdet(Kk, jit)) + n * O.LOG_2_PI + float(O.iqf_diag(Kk, y[keep, None] - mean[keep], eps=jit)[0])
        for _ in range(2):
            got = float(nrm.logpdf(_dev(y, dtype)))
            assert np.isfinite(got) and abs(got - ref) <= tol * scale, (got, ref)


# ---- 5. raw-pointer matrix functions refuse a backward --------------------------------------------------------------
def _ell_fdd(S, n, dtype=F64):
    dev = S._util._device_fn()
    rng = np.random.default_rng(0)
    x = torch.as_tensor(rng.standard_normal((n, 2)), dtype=dtype, device=dev)
    ell = torch.tensor(1.3, dtype=dtype, device=dev, requires_grad=True)
    return S.GP(S.EQ().stretch(ell))(x, 0.1), ell


def _refused(value, reference):
    """Same value as without grad mode, a graph, and a backward that raises."""
    assert value.requires_grad
    torch.testing.assert_close(value.detach(), reference, rtol=1e-14, atol=0)
    with pytest.raises(NotImplementedError):
        value.sum().backward()


def test_entropy_refuses_gradient_cpu(cpu_backend, monkeypatch):
    import stheno_b200 as S

    monkeypatch.setattr(S.B, "epsilon", 1e-12)
    fd, _ = _ell_fdd(S, 40)
    e = fd.entropy()
    with torch.no_grad():
        e0 = _ell_fdd(S, 40)[0].entropy()
    _refused(e, e0)


@gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_entropy_refuses_gradient(S, dtype):
    with _setup(S, dtype):
        fd, _ = _ell_fdd(S, 300, dtype)
        e = fd.entropy()
        with torch.no_grad():
            e0 = _ell_fdd(S, 300, dtype)[0].entropy()
        _refused(e, e0)


@gpu
@pytest.mark.parametrize("order", ["pq", "qp"])
def test_kl_refuses_gradient(S, order):
    """``ratio`` densifies the kernel matrix through a differentiable K1 and then solves a copy of it in place: its graph
    said ``d ratio / dA = I``.  Both argument orders now refuse the backward."""
    rng = np.random.default_rng(1)
    n = 200
    G = rng.standard_normal((n, n))
    q = S.Normal(_dev(rng.standard_normal((n, 1))), S.matrix.Dense(_dev(G @ G.T / n + np.eye(n))),
                 origin=torch.device("cuda"))

    def kl():
        p = _ell_fdd(S, n)[0]
        return p.kl(q) if order == "pq" else q.kl(p)

    value = kl()
    with torch.no_grad():
        ref = kl()
    _refused(value, ref)


@gpu
def test_iqf_diag_refuses_gradient_of_rhs(S):
    """A right-hand side that requires grad is copied into the solve's buffer: autograd saw ``|d|^2``, not ``|L^-1 d|^2``."""
    rng = np.random.default_rng(2)
    n = 200
    G = rng.standard_normal((n, n))
    var = S.matrix.Dense(_dev(G @ G.T / n + np.eye(n)))
    d = _dev(rng.standard_normal((n, 3))).requires_grad_()
    value = S.matrix.iqf_diag(var, d)
    with torch.no_grad():
        ref = S.matrix.iqf_diag(var, d)
    _refused(value, ref)
    value = S.matrix.iqf_diag(var, d, 2 * d)
    with torch.no_grad():
        ref = S.matrix.iqf_diag(var, d, 2 * d)
    _refused(value, ref)


@gpu
def test_woodbury_entropy_refuses_gradient(S):
    """``logdet`` of a Woodbury matrix adds the raw-pointer Schur-complement log-det to a differentiable ``sum log d``:
    the graph held half of the gradient."""
    rng = np.random.default_rng(4)
    n, r = 300, 5
    U = _dev(0.5 * rng.standard_normal((n, r))).requires_grad_()
    d = _dev(rng.uniform(0.2, 0.6, n)).requires_grad_()

    def entropy():
        return S.Normal(S.matrix.Woodbury(S.matrix.Diagonal(d), S.matrix.LowRank(U)), origin=d.device).entropy()

    value = entropy()
    with torch.no_grad():
        ref = entropy()
    _refused(value, ref)
