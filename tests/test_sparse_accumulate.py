"""The streamed sparse accumulation (``gpk_sparse_accumulate``, ``csrc/sparse.cu``) stage by stage and end to end.

One ``SparseAccumulator.add`` is read back from its workspace (``Wc [c_pad][m_pad]``, ``WcT [m_pad][c_pad]``, ``q``, ``rs``,
``ybs``) and every stage is checked against its own reference, built from what the device produced in the stage before it
(the factor ``ch.L()``, the device ``Wc``, ``q`` and ``WcT``), so that one stage's error never hides another's:
  Wc      forward and backward error of ``solve_triangular(L, K_zx)``; zero padding
  q       extended-precision row sums of the device ``Wc^2``
  rs, ybs ``1 / sqrt(kn')`` in extended precision (``kn'`` holds ``corr`` for FITC) to a few ulp; zero padding
  WcT     ``T(Wc[i][j] * rs[i])`` bit for bit
  A       ``A_in + WcT WcT^T`` on the lower 128-tiles within ``c_pad u |W||W|^T`` (plus the slicing bound where the product is
          emulated); the tiles above the block diagonal keep a sentinel and the padding stays identity / zero, bit for bit
  prod    ``prod_in + WcT ybs``; ``prod[m:]`` exactly 0
  scalars extended-precision sums; the trace part exactly 0 for FITC and DTC
at tile edges, multi-tile ``A``, and the shapes where the fp64 SYRK / the solve's largest GEMM run on the int8 emulation
(predicted from the library's size queries and checked on the launch profile).  Then several chunks, a stale workspace,
run-to-run reproducibility, ``PseudoObs*`` against the oracle (prior mean, Delta term with shared points, a Linear product,
the materialised route), fp32 inputs, and one chunk large enough for ``c_pad / 32`` to pass the 65535 grid limit."""
import contextlib
import math

import numpy as np
import pytest
import scipy.linalg as sla
import torch

from oracle import gp_oracle as O

pytestmark = pytest.mark.gpu

U = {torch.float64: 2.0**-53, torch.float32: 2.0**-24}
U64 = 2.0**-53
NP = {torch.float64: np.float64, torch.float32: np.float32}
TOL_OZ8 = 5e-15  # 8-slice emulation bound relative to rowmax(A) colmax(B) sqrt(K) (tests/test_gemm_paths.py)
COEF = 1.3  # the stage tests' kernel: COEF * exp(-|x - z|^2 / 2) on pre-stretched inputs
METHODS = ["vfe", "fitc", "dtc"]
DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    from stheno_b200 import ops

    return ops


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


def profiled(ops, fn):
    """``fn()`` with the GEMM launch profile on: ``(native fp64 DMMA launches, emulated launches)``."""
    ops.gemm_profile(True)
    try:
        fn()
        return ops.gemm_profile_read(0)[2], ops.gemm_profile_read(1)[2]
    finally:
        ops.gemm_profile(False)


def round_up(v):
    return (v + 127) // 128 * 128


# ---- stage-by-stage checks of one add -----------------------------------------------------------------------------------
class Problem:
    """``m`` inducing points and the data of one or more chunks on the device in ``dtype``, with their host copies in fp64
    (the device values, so the references see exactly what the kernels saw)."""

    def __init__(self, ops, dtype, m, n, method, seed):
        rng = np.random.default_rng(seed)
        d = 2
        self.dtype, self.m, self.method = dtype, m, method
        dev = lambda a: torch.as_tensor(a, device="cuda", dtype=dtype)
        self.zd, self.xd = dev(rng.uniform(-2, 2, (m, d))), dev(rng.uniform(-2, 2, (n, d)))
        self.knd = dev(0.05 + rng.uniform(0, 0.1, n))
        self.ybd = dev(rng.standard_normal(n))
        self.kdd = None if method == "dtc" else dev(np.full(n, COEF))
        host = lambda t: None if t is None else t.double().cpu().numpy()
        self.z, self.x, self.kn, self.yb, self.kd = map(host, (self.zd, self.xd, self.knd, self.ybd, self.kdd))
        self.flat = ops.FlatKernel([(COEF, [("eq", 0)])], 1)
        # K_z + 0.3 I: a well-conditioned factor (the accumulation takes any padded lower factor)
        self.ch = ops.chol_from_kernel(self.flat, self.zd[None, None], noise_scalar=0.3)
        assert not self.ch.info.any()
        self.L = self.ch.L()[0].double().cpu().numpy()
        self.m_pad = self.ch.n_pad

    def accumulator(self, ops, chunk=16384):
        return ops.SparseAccumulator(self.flat, self.zd[None, None], self.ch, self.method, chunk=chunk)

    def add(self, acc, a, b):
        acc.add(self.xd[a:b][None, None], None if self.kdd is None else self.kdd[a:b], self.knd[a:b], self.ybd[a:b])

    def kzx(self, a, b):
        d2 = ((self.z[:, None, :] - self.x[None, a:b, :]) ** 2).sum(-1)
        return COEF * np.exp(-0.5 * d2)


def seed_state(acc, rng):
    """Random ``A_in`` on the leading m x m block of the lower tiles (identity / zero padding as the accumulator starts it),
    a sentinel on the tiles above the block diagonal, random ``prod_in[:m]`` and ``scalars_in`` with a zero trace part."""
    m, m_pad, dt = acc.m, acc.m_pad, acc.A.dtype
    A = torch.eye(m_pad, dtype=torch.float64)
    A[:m, :m] = torch.as_tensor(rng.uniform(-1, 1, (m, m)))
    t = torch.arange(m_pad) // 128
    A[t[None, :] > t[:, None]] = -7.25e3
    acc.A.copy_(A.to(dt)[None])
    acc.prod.zero_()
    acc.prod[:m] = torch.as_tensor(rng.standard_normal(m), dtype=dt)
    acc.scalars.copy_(torch.tensor([0.75, -0.5, 0.0], dtype=dt))


def bits(t):
    return t.view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def check_add(P, acc, a, b, emulated):
    """Add points ``a:b`` to ``acc`` and check every stage.  ``emulated``: the SYRK runs on the int8 emulation."""
    dt, u, T = P.dtype, U[P.dtype], NP[P.dtype]
    m, m_pad, c = P.m, P.m_pad, b - a
    c_pad = round_up(c)
    A_in, prod_in, s_in = acc.A[0].clone(), acc.prod.clone(), acc.scalars.double().cpu().numpy()
    P.add(acc, a, b)
    torch.cuda.synchronize()
    ws = acc.ws
    o = 0
    Wc_d = ws[o : o + c_pad * m_pad].view(c_pad, m_pad); o += c_pad * m_pad
    WcT_d = ws[o : o + m_pad * c_pad].view(m_pad, c_pad); o += m_pad * c_pad
    q_d, rs_d, ybs_d = ws[o : o + c_pad], ws[o + c_pad : o + 2 * c_pad], ws[o + 2 * c_pad : o + 3 * c_pad]
    Wc, WcT = Wc_d.cpu().numpy(), WcT_d.cpu().numpy()
    q, rs, ybs = q_d.cpu().numpy(), rs_d.cpu().numpy(), ybs_d.cpu().numpy()

    # Wc = (L^-1 K_zx)^T, zero padding
    assert not Wc[c:].any() and not Wc[:, m:].any()
    X, Bt = Wc[:c, :m].astype(np.float64), P.kzx(a, b).T
    want = sla.solve_triangular(P.L, Bt.T, lower=True).T
    assert np.abs(X - want).max() <= 100 * m_pad * u * np.abs(want).max()
    rows = sorted({r % c for r in (0, 1, 127, 128, c // 2, c - 1)})
    Xl, Bl, Ll = X[rows].astype(np.longdouble), Bt[rows].astype(np.longdouble), P.L.astype(np.longdouble)
    r = np.abs(Xl @ Ll.T - Bl).max(-1)
    assert (r / ((np.abs(Xl) @ np.abs(Ll.T)).max(-1) + np.abs(Bl).max(-1))).max() <= 4 * m_pad * u

    # q = |w_i|^2 of the device Wc (m_pad fused multiply-adds in T)
    kn = P.kn[a:b]
    if P.method != "dtc":
        Wl = Wc[:c].astype(np.longdouble)
        q_ref = (Wl * Wl).sum(1)
        assert (np.abs(q[:c] - q_ref) <= (m_pad + 2) * u * q_ref + 1e-300).all()
        corr = P.kd[a:b] - q[:c].astype(np.float64)  # the device's double arithmetic, operation for operation
        if P.method == "fitc":
            kn = kn + corr

    # rs = 1 / sqrt(kn'), ybs = ybar rs, zero padding
    k_l = kn.astype(np.longdouble)
    rs_ref = 1 / np.sqrt(k_l)
    ybs_ref = P.yb[a:b].astype(np.longdouble) * rs_ref
    assert (np.abs(rs[:c] - rs_ref) <= 4 * u * rs_ref).all()
    assert (np.abs(ybs[:c] - ybs_ref) <= (4 * u + 8 * U64) * np.abs(ybs_ref)).all()
    assert not rs[c:].any() and not ybs[c:].any()

    # WcT[j][i] = T(Wc[i][j] rs[i]): one rounding in T
    I = np.int64 if T is np.float64 else np.int32
    assert np.array_equal(np.ascontiguousarray((Wc * rs[:, None]).astype(T).T).view(I), WcT.view(I))

    # A: lower tiles, sampled rows, residual in extended precision
    A = acc.A[0]
    t = torch.arange(m_pad, device="cuda") // 128
    upper = t[None, :] > t[:, None]
    assert torch.equal(bits(A[upper]), bits(A_in[upper]))
    lower = ~upper
    pad = torch.zeros(m_pad, m_pad, dtype=torch.bool, device="cuda")
    pad[m:, :] = pad[:, m:] = True
    assert torch.equal(bits(A[pad & lower]), bits(A_in[pad & lower]))
    An, A_inn = A.double().cpu().numpy(), A_in.double().cpu().numpy()
    Wt = WcT[:m].astype(np.longdouble)
    rowmax = np.abs(WcT[:m].astype(np.float64)).max(1)
    for i in sorted({r_ % m for r_ in (0, 1, 127, 128, 129, m // 2, m - 2, m - 1)}):
        j1 = min(m, (i // 128 + 1) * 128)
        dots = Wt[:j1] @ Wt[i]
        ref = A_inn[i, :j1] + dots
        absd = np.abs(Wt[:j1]) @ np.abs(Wt[i])
        bound = (c_pad + 8) * u * absd + 4 * u * (np.abs(ref) + np.abs(A_inn[i, :j1]))
        if emulated:
            bound = bound + TOL_OZ8 * rowmax[i] * rowmax[:j1] * math.sqrt(c_pad)
        err = np.abs(An[i, :j1] - ref)
        assert (err <= bound).all(), (i, float((err / bound).max()))

    # prod += WcT ybs
    prod = acc.prod.double().cpu().numpy()
    assert not prod[m:].any()
    yl = ybs.astype(np.longdouble)
    pin = prod_in[:m].double().cpu().numpy()
    p_ref = pin + Wt @ yl
    p_bound = (c_pad + 4) * U64 * (np.abs(Wt) @ np.abs(yl)) + 2 * u * (np.abs(p_ref) + np.abs(pin))
    assert (np.abs(prod[:m] - p_ref) <= p_bound).all()

    # scalars: sum log(2 pi kn'), sum ybar^2 / kn', trace part
    s = acc.scalars.double().cpu().numpy()
    yl2 = P.yb[a:b].astype(np.longdouble) ** 2
    terms = [np.log(2 * np.pi * k_l), yl2 / k_l]
    extra = [4 * U64 * c, 0.0]  # the absolute error of each log term (its argument is rounded)
    if P.method == "vfe":
        terms.append((P.kd[a:b].astype(np.longdouble) - q[:c].astype(np.longdouble)) / k_l)
        extra.append(0.0)
    for j, (tj, ej) in enumerate(zip(terms, extra)):
        ref = s_in[j] + float(tj.sum())
        bound = (c + 8) * U64 * float(np.abs(tj).sum()) + ej + 2 * u * (abs(ref) + abs(s_in[j]))
        assert abs(s[j] - ref) <= bound, (j, s[j], ref, bound)
    if P.method != "vfe":
        assert s[2] == 0.0


def predicted_oz_launches(lib, m_pad, c_pad, slices=8):
    """Emulated GEMM launches of one fp64 add, from the library's size queries: the SYRK (one launch per K pass of at most
    65536) and the GEMMs of the recursive right solve of c_pad rows (the recursion of ``trsm_right_rec``)."""
    syrk = (-(-c_pad // 65536)) if lib.gpk_gemm_nt_oz_ws_bytes(m_pad, m_pad, c_pad, slices) else 0

    def solve(n):
        if n <= 128:
            return 0
        h = (n // 128 // 2) * 128
        return solve(h) + (1 if lib.gpk_gemm_nt_oz_ws_bytes(c_pad, n - h, h, slices) else 0) + solve(n - h)

    return syrk, solve(m_pad)


#: (m, c, emulated SYRK, emulated GEMMs in the solve) of an fp64 add under the default precision
SHAPES = [
    (1, 1, False, 0),
    (37, 128, False, 0),
    (128, 127, False, 0),
    (129, 129, False, 0),
    (300, 1000, False, 0),  # multi-tile A
    (640, 4000, True, 0),  # 640^2 4096 >= 1.5e9
    (256, 70000, True, 0),  # K = 70016 > 65536: two exact passes
    (1000, 16384, True, 1),  # and the solve's 16384 x 512 x 512 GEMM
]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("m,c,em_syrk,em_solve", SHAPES)
def test_one_add_stage_by_stage(ops, m, c, em_syrk, em_solve, dtype, method):
    P = Problem(ops, dtype, m, c, method, seed=m * 7 + c)
    acc = P.accumulator(ops)
    seed_state(acc, np.random.default_rng(1))
    m_pad, c_pad = P.m_pad, round_up(c)
    syrk, solve = predicted_oz_launches(acc.lib, m_pad, c_pad)
    assert (syrk > 0, solve) == (em_syrk, em_solve)
    n_dmma, n_oz = profiled(ops, lambda: check_add(P, acc, 0, c, emulated=em_syrk and dtype == torch.float64))
    assert n_oz == (syrk + solve if dtype == torch.float64 else 0), (n_oz, syrk, solve)


@pytest.mark.parametrize("m,c", [(mm, cc) for mm, cc, em, _ in SHAPES if em])
def test_emulated_shapes_on_fp64_tensor_cores(ops, m, c):
    """The shapes above that emulate, with ``B.precision = "fp64"``: the SYRK runs on DMMA and meets the same bounds."""
    P = Problem(ops, torch.float64, m, c, "vfe", seed=m + c)
    acc = P.accumulator(ops)
    seed_state(acc, np.random.default_rng(2))
    with precision("fp64"):
        n_dmma, n_oz = profiled(ops, lambda: check_add(P, acc, 0, c, emulated=False))
    assert n_oz == 0 and n_dmma >= 1, (n_dmma, n_oz)


# ---- across chunks ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("sizes", [(1000, 700, 1), (300, 1000, 128)])
def test_chunks_stage_by_stage(ops, sizes, method, dtype):
    """Several adds on one accumulator, the last of 1 or of exactly 128 points: each add checked as above on the workspace
    the earlier (larger) chunk left behind."""
    m = 300
    P = Problem(ops, dtype, m, sum(sizes), method, seed=sum(sizes))
    acc = P.accumulator(ops)
    seed_state(acc, np.random.default_rng(3))
    a = 0
    for c in sizes:
        check_add(P, acc, a, a + c, emulated=False)
        a += c


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("method", METHODS)
def test_stale_workspace(ops, method, dtype):
    """A workspace grown by a larger chunk and filled with NaN gives, bit for bit, what a fresh one gives (chunks of at most
    256 points, so the comparison does not depend on how the per-chunk sums are ordered)."""
    sizes = (200, 1, 128, 77)
    P = Problem(ops, dtype, 300, sum(sizes), method, seed=11)
    runs = []
    for stale in (True, False):
        acc = P.accumulator(ops)
        if stale:
            acc._workspace(4000).fill_(float("nan"))
        a = 0
        for c in sizes:
            P.add(acc, a, a + c)
            a += c
        runs.append((acc.A.clone(), acc.prod.clone(), acc.scalars.clone()))
        assert not torch.isnan(acc.A).any()
    for x, y in zip(*runs):
        assert torch.equal(bits(x), bits(y))


# ---- reproducibility ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("method", METHODS)
def test_adds_are_reproducible(ops, method, dtype):
    """The same adds twice (chunks of many 256-point blocks): A, prod and the ELBO sums are bit-identical."""
    sizes = (65536, 30000, 4097)
    P = Problem(ops, dtype, 129, sum(sizes), method, seed=12)
    runs = []
    for _ in range(3):
        acc = P.accumulator(ops)
        a = 0
        for c in sizes:
            P.add(acc, a, a + c)
            a += c
        runs.append((acc.A.clone(), acc.prod.clone(), acc.scalars.clone()))
    for run in runs[1:]:
        for x, y in zip(runs[0], run):
            assert torch.equal(bits(x), bits(y))


def _elbo_problem(rng, n, m, d=3):
    x, z, y = rng.uniform(-3, 3, (n, d)), rng.uniform(-3, 3, (m, d)), rng.standard_normal(n)
    noise = 0.05 + rng.uniform(0, 0.1, n)
    return x, z, y, noise


SPEC = ("sum", ("scaled", 1.2, ("stretched", 1.7, ("matern52",))), ("scaled", 0.3, ("eq",)))


def _kernel(S):
    return 1.2 * S.Matern52().stretch(1.7) + 0.3 * S.EQ()


OBS = {"vfe": "PseudoObs", "fitc": "PseudoObsFITC", "dtc": "PseudoObsDTC"}


@pytest.mark.parametrize("method", METHODS)
def test_elbo_is_reproducible(S, monkeypatch, method):
    monkeypatch.setattr(S.B, "sparse_chunk", 20000)
    x, z, y, noise = _elbo_problem(np.random.default_rng(13), 50000, 200)
    e = []
    for _ in range(3):
        f = S.GP(_kernel(S))
        e.append(float(getattr(S, OBS[method])(f(z), f(x, noise), y).elbo(f.measure)))
    assert e[0] == e[1] == e[2], e


# ---- end to end against the oracle ---------------------------------------------------------------------------------------
def _check_oracle(S, obs, f, want, elbo_rtol=1e-10):
    assert abs(float(obs.elbo(f.measure)) - want["elbo"]) <= elbo_rtol * abs(want["elbo"])
    np.testing.assert_allclose(S.B.to_numpy(obs.mu(f.measure)).reshape(-1), want["mu"].reshape(-1), rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(S.B.to_numpy(S.B.dense(obs.A(f.measure))).reshape(want["A"].shape), want["A"], rtol=1e-8,
                               atol=1e-9)


@pytest.mark.parametrize("chunk", [1000, 2047, None])
@pytest.mark.parametrize("m", [129, 300])
@pytest.mark.parametrize("method", METHODS)
def test_pseudo_obs_against_oracle(S, monkeypatch, method, m, chunk):
    n = 6000
    monkeypatch.setattr(S.B, "sparse_chunk", chunk or n)
    x, z, y, noise = _elbo_problem(np.random.default_rng(m + (chunk or 0)), n, m)
    f = S.GP(_kernel(S))
    obs = getattr(S, OBS[method])(f(z), f(x, noise), y)
    _check_oracle(S, obs, f, O.sparse_compute(SPEC, z, x, noise, y, method))


@pytest.mark.parametrize("method", METHODS)
def test_pseudo_obs_prior_mean(S, monkeypatch, method):
    monkeypatch.setattr(S.B, "sparse_chunk", 2047)
    x, z, y, noise = _elbo_problem(np.random.default_rng(21), 6000, 300)
    f = S.GP(lambda t: 0.5 * t.sum(-1, keepdim=True) + 1.0, _kernel(S))
    obs = getattr(S, OBS[method])(f(z), f(x, noise), y)
    mean = lambda a: 0.5 * a.sum(-1) + 1.0
    _check_oracle(S, obs, f, O.sparse_compute(SPEC, z, x, noise, y, method, mean_x=mean(x), mean_z=mean(z)))


@pytest.mark.parametrize("method", METHODS)
def test_pseudo_obs_delta_with_shared_points(S, monkeypatch, method):
    """A Delta term and inducing points that are data points: the cross kernel meets coincident pairs."""
    monkeypatch.setattr(S.B, "sparse_chunk", 1000)
    rng = np.random.default_rng(22)
    x, _, y, noise = _elbo_problem(rng, 6000, 1)
    z = x[rng.choice(6000, 300, replace=False)]
    f = S.GP(S.EQ().stretch(1.3) + 0.1 * S.Delta())
    spec = ("sum", ("stretched", 1.3, ("eq",)), ("scaled", 0.1, ("delta",)))
    obs = getattr(S, OBS[method])(f(z), f(x, noise), y)
    _check_oracle(S, obs, f, O.sparse_compute(spec, z, x, noise, y, method))


@pytest.mark.parametrize("method", METHODS)
def test_pseudo_obs_linear_product(S, monkeypatch, method):
    """A composite with a Linear factor (the generic K1 kernel rather than the stationary fast path)."""
    monkeypatch.setattr(S.B, "sparse_chunk", 2047)
    x, z, y, noise = _elbo_problem(np.random.default_rng(23), 6000, 129)
    f = S.GP(S.EQ().stretch(1.5) + 0.5 * S.Matern32() * S.Linear().stretch(4.0))
    spec = ("sum", ("stretched", 1.5, ("eq",)), ("scaled", 0.5, ("product", ("matern32",), ("stretched", 4.0, ("linear",)))))
    obs = getattr(S, OBS[method])(f(z), f(x, noise), y)
    _check_oracle(S, obs, f, O.sparse_compute(spec, z, x, noise, y, method))


@pytest.mark.parametrize("method", METHODS)
def test_materialised_route_against_oracle(S, method):
    """A leading batch dimension of 1 takes the materialised route; it agrees with the oracle too."""
    x, z, y, noise = _elbo_problem(np.random.default_rng(24), 6000, 300)
    f = S.GP(_kernel(S))
    obs = getattr(S, OBS[method])(f(z[None]), f(x[None], noise[None]), y[None, :, None])
    want = O.sparse_compute(SPEC, z, x, noise, y, method)
    e = S.B.to_numpy(obs.elbo(f.measure))
    assert e.shape == (1,) and abs(float(e[0]) - want["elbo"]) <= 1e-10 * abs(want["elbo"])
    np.testing.assert_allclose(S.B.to_numpy(obs.mu(f.measure)).reshape(-1), want["mu"].reshape(-1), rtol=1e-8, atol=1e-10)


# ---- fp32 ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
def test_fp32_streamed(S, monkeypatch, method):
    """fp32 inputs with ``B.epsilon = 1e-6`` against the fp64 oracle on the fp32-rounded inputs (ELBO to 1e-4 relative), and
    the streamed result against the materialised one."""
    monkeypatch.setattr(S.B, "epsilon", 1e-6)
    monkeypatch.setattr(S.B, "sparse_chunk", 2047)
    x, z, y, noise = _elbo_problem(np.random.default_rng(31), 6000, 129)
    x, z, y, noise = (a.astype(np.float32) for a in (x, z, y, noise))
    f = S.GP(_kernel(S))
    t = lambda a: torch.as_tensor(a, device=DEV)
    obs = getattr(S, OBS[method])(f(t(z)), f(t(x), t(noise)), t(y))
    e = obs.elbo(f.measure)
    assert e.dtype == torch.float32
    want = O.sparse_compute(SPEC, z.astype(np.float64), x.astype(np.float64), noise.astype(np.float64),
                            y.astype(np.float64), method, eps=1e-6)
    assert abs(float(e) - want["elbo"]) <= 1e-4 * abs(want["elbo"])
    mu = S.B.to_numpy(obs.mu(f.measure)).reshape(-1).astype(np.float64)
    scale = np.abs(want["mu"]).max()
    assert np.abs(mu - want["mu"].reshape(-1)).max() <= 1e-3 * scale
    f2 = S.GP(_kernel(S))
    mat = getattr(S, OBS[method])(f2(t(z)[None]), f2(t(x)[None], t(noise)[None]), t(y)[None, :, None])
    e2 = float(S.B.to_numpy(mat.elbo(f2.measure))[0])
    assert abs(float(e) - e2) <= 1e-4 * abs(want["elbo"])
    mu2 = S.B.to_numpy(mat.mu(f2.measure)).reshape(-1).astype(np.float64)
    assert np.abs(mu - mu2).max() <= 1e-3 * scale


# ---- one large chunk ----------------------------------------------------------------------------------------------------
def test_one_chunk_past_the_grid_limit(S, monkeypatch):
    """2,097,025 points in one chunk: c_pad = 2^21, c_pad / 32 = 65536 row tiles of the scaled transpose."""
    n = 2_097_025
    monkeypatch.setattr(S.B, "sparse_chunk", n)
    rng = np.random.default_rng(41)
    x, z, y = rng.uniform(0, 100, (n, 1)), np.array([[20.0], [50.0], [80.0]]), rng.standard_normal(n)
    noise = 0.5
    f = S.GP(S.EQ().stretch(10.0))
    obs = S.PseudoObs(f(z), f(x, noise), y)
    want = O.sparse_compute(("stretched", 10.0, ("eq",)), z, x, noise, y, "vfe")
    assert abs(float(obs.elbo(f.measure)) - want["elbo"]) <= 1e-10 * abs(want["elbo"])
    np.testing.assert_allclose(S.B.to_numpy(obs.mu(f.measure)).reshape(-1), want["mu"].reshape(-1), rtol=1e-8, atol=1e-10)


@pytest.mark.parametrize("rows,cols", [(2**21 + 1, 3), (3, 2**21 + 1)])
def test_transpose_long_dimension(ops, rows, cols):
    src = torch.randn(1, rows, cols, device="cuda", dtype=torch.float64)
    out = ops.transpose(src, rows, cols)
    assert torch.equal(bits(out[0]), bits(src[0].T.contiguous()))
