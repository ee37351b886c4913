"""Full posterior covariances against fp64 references, on every product path and at the benchmarked size.

The dense ``m x m`` (or ``mx x my``) result of a posterior is ``prior - V_x V_y^T`` with ``V = k(x*, z) L^-T``: one solve of
all test points (``Chol.solve_rows_``) and one ``gemm_nt`` over ``K = n_pad``.  Each case here

* asserts the path it claims: every solve and product is wrapped and its launches read from the in-situ GEMM profile
  (kind 0 = the fp64 DMMA v3 kernel, kind 1 = the int8-slice emulation; the v2 kernels are not profiled), and an fp32
  product is proven to have run on the 3xTF32 wgmma kernel by a probe of the same shape (:func:`tc32_probe`);
* compares element by element with the oracle (``oracle/gp_oracle.py``) or a NumPy fp64 restatement, relative to
  ``sqrt(prior_ii prior_jj)``;
* checks internal consistency: ``var`` is bit-symmetric, ``mean_var`` gives the ``var`` and ``mean`` of the separate routes bit
  for bit, and ``diag(var)`` meets the chunked marginals route (``gpk_posterior_marginals`` / the streamed sparse marginals).

Routes: exact ``var`` (lower product, beta = 1, mirrored) and ``mean_var`` (``PosteriorKernel._cov_lower``); cross-covariances
between different inputs or processes (non-lower product, no mirror); sparse ``var`` (the exact part plus ``SubspaceKernel``'s
plain product, solved against ``A``'s factor); multi-output posteriors (``BlockDense`` joint factor, dense cross rows); a
factorisation workspace filled with NaN / huge stale values; config 2's posterior at n = 16384, m = 4096.
"""
import os

import numpy as np
import pytest
import torch

from oracle import gp_oracle as O
from tests.test_gpu_primitives import tc32_probe

pytestmark = pytest.mark.gpu

DEV = "cuda"
U32 = 2.0**-24
#: fp64 bar against the oracle, relative to sqrt(prior_ii prior_jj) (means: to max(1, max |mean|))
TOL = 1e-10
#: fp64 bar between two device routes over the same factor (the full covariance's diagonal vs the chunked marginals), relative
#: to the prior variance
SAME_TOL = 1e-12
#: fp32 bar: C32 2^-24 kappa(K_x + noise + eps I), as in tests/test_logpdf_grad_paths.py, relative as above.  Measured on
#: an H100 (80GB HBM3, 700 W power limit), worst error over var, mean and var_diag in units of 2^-24 kappa: 0.062 (exact,
#: batch 1, kappa 4.1e2), 0.042 (exact, batch 4, kappa 2.3e2), 0.058 (multi-output, N = 2537, batch 2, kappa 5.2e4).  A wrong
#: tile or a lost beta term gives O(1) relative errors, ~1e3 times the bar.
C32 = 16.0
PRECISIONS = ["auto", "int8x8", "fp64"]
SLICES = {"auto": 8, "int8x8": 8, "fp64": 0}


@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.B, "precision", "auto")
    monkeypatch.setattr(s.Measure, "default", None)
    return s


def t(a, dtype=torch.float64):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device=DEV)


def host(v):
    return v.detach().double().cpu().numpy()


def dense(a):
    from stheno_b200 import matrix

    return matrix.dense(a)


def _threads():
    try:
        import threadpoolctl

        threadpoolctl.threadpool_limits(limits=os.cpu_count() or 1)
    except Exception:
        pass


# ---------------------------------------------------------------------------------------------------------------------
# launch paths
# ---------------------------------------------------------------------------------------------------------------------
class Launches:
    """What the wrapped solves, products and factorisations ran since :meth:`clear`."""

    def __init__(self):
        self.gemm, self.solve, self.potrf = [], [], []

    def clear(self):
        self.gemm.clear()
        self.solve.clear()
        self.potrf.clear()


@pytest.fixture
def paths(monkeypatch):
    """Wraps ``ops.gemm_nt``, ``ops.Chol.solve_rows_`` and ``ops._potrf``: each call is run with the GEMM profile on and
    recorded with its shape and launch counts; an fp32 product also records which kernel a probe of its shape runs on."""
    from stheno_b200 import ops

    rec = Launches()
    real_gemm, real_solve, real_potrf = ops.gemm_nt, ops.Chol.solve_rows_, ops._potrf

    def profiled(fn):
        ops.gemm_profile(True)
        try:
            out = fn()
            return out, ops.gemm_profile_read(0)[2], ops.gemm_profile_read(1)[2]
        finally:
            ops.gemm_profile(False)

    def gemm(A, Bm, C=None, *, alpha=1.0, beta=0.0, lower=False):
        out, v3, oz = profiled(lambda: real_gemm(A, Bm, C, alpha=alpha, beta=beta, lower=lower))
        call = dict(M=A.shape[1], N=Bm.shape[1], K=A.shape[2], batch=A.shape[0], dtype=A.dtype, alpha=alpha,
                    beta=beta if C is not None else 0.0, lower=lower, v3=v3, oz=oz)
        if A.dtype == torch.float32:
            call["kernel"] = tc32_probe(ops, call["M"], call["N"], call["K"], call["batch"], lower, gemm=real_gemm)
        rec.gemm.append(call)
        return out

    def solve(self, Bt):
        out, _, oz = profiled(lambda: real_solve(self, Bt))
        rec.solve.append(dict(n_pad=self.n_pad, rows=Bt.shape[1], batch=self.batch, dtype=self.dtype, oz=oz))
        return out

    def potrf(W, n, n_pad, extra, k, well_conditioned=False):
        out, _, oz = profiled(lambda: real_potrf(W, n, n_pad, extra, k, well_conditioned))
        rec.potrf.append(dict(n_pad=n_pad, batch=W.shape[0], dtype=W.dtype, oz=oz))
        return out

    monkeypatch.setattr(ops, "gemm_nt", gemm)
    monkeypatch.setattr(ops.Chol, "solve_rows_", solve)
    monkeypatch.setattr(ops, "_potrf", potrf)
    return rec


def gemm_path(call):
    """The kernel a recorded product ran on."""
    if call["dtype"] == torch.float32:
        return call["kernel"]
    if call["oz"]:
        return "emulated" if call["v3"] == 0 else f"mixed {call}"
    return {0: "v2", 1: "v3"}.get(call["v3"], f"several v3 launches {call}")


def gemm_expected(call, precision):
    """The kernel the library's size rules choose for a product: the emulation for a single fp64 problem whose size query is
    non-zero under ``precision``'s slice count, else v3 for K >= 512 (K % 32 == 0), else v2; fp32: 3xTF32."""
    from stheno_b200 import _lib

    if call["dtype"] == torch.float32:
        return "tc32"
    s = SLICES[precision]
    if s and call["batch"] == 1 and _lib.load().gpk_gemm_nt_oz_ws_bytes(call["M"], call["N"], call["K"], s) > 0:
        return "emulated"
    return "v3" if call["K"] >= 512 and call["K"] % 32 == 0 else "v2"


def solve_emulated(call, precision):
    from stheno_b200 import _lib

    s = SLICES[precision] if call["dtype"] == torch.float64 else 0
    return bool(s and call["batch"] == 1 and _lib.load().gpk_trsm_right_oz_ws_bytes(call["n_pad"], call["rows"], s) > 0)


def check_products(rec, precision, want):
    """Every recorded product ran where the size rules send it, and the products are ``want``: a list of
    ``(M, N, K, lower, beta)`` (alpha -1 where beta is 1).  Returns the paths taken."""
    got = [(c["M"], c["N"], c["K"], c["lower"], c["beta"]) for c in rec.gemm]
    assert got == want, (got, want)
    taken = []
    for c in rec.gemm:
        assert c["alpha"] == (-1.0 if c["beta"] == 1.0 else 1.0), c
        assert gemm_path(c) == gemm_expected(c, precision), (c, precision)
        taken.append(gemm_path(c))
    return taken


def check_solves(rec, precision, rows, n_pads):
    """The recorded solves are of ``rows`` padded rows against factors of ``n_pads``, each emulated exactly when the size
    query says so.  Returns whether each was emulated."""
    assert [(c["rows"], c["n_pad"]) for c in rec.solve] == [(rows, n) for n in n_pads], rec.solve
    out = []
    for c in rec.solve:
        emu = solve_emulated(c, precision)
        assert (c["oz"] > 0) == emu, (c, precision)
        out.append(emu)
    return out


def check_factor(rec, n_pad, batch, dt):
    """One factorisation of ``n_pad`` was recorded, emulated exactly for a single fp64 problem of ``n_pad >= 2048`` ("auto")."""
    assert [(c["n_pad"], c["batch"]) for c in rec.potrf] == [(n_pad, batch)], rec.potrf
    emulated = rec.potrf[0]["oz"] > 0
    assert emulated == (dt == "fp64" and batch == 1 and n_pad >= 2048), rec.potrf
    return emulated


def pad(n):
    return (int(n) + 127) // 128 * 128


def rel_err(got, want, scale):
    return float(np.max(np.abs(np.asarray(got, np.float64) - want) / scale))


def kappa(K):
    ev = np.linalg.eigvalsh(K)
    return float(ev[-1] / ev[0])


# ---------------------------------------------------------------------------------------------------------------------
# exact var, mean_var and marginal_credible_bounds
# ---------------------------------------------------------------------------------------------------------------------
EQS, M52S = ("stretched", 1.1, ("eq",)), ("stretched", 0.8, ("matern52",))
SPEC = ("sum", ("scaled", 1.3, EQS), ("scaled", 0.4, M52S))
D = 3

#: name -> (n, m, batch, dtype, variant).  Paths under "auto" (size rules of gpk.h, each asserted per call):
#:   n = 300:  K = 384 < 512, product on v2; solves native (n_pad 384)
#:   n = 2500: K = 2560, product on v3 for m <= 129 (M = N < 256 or M N K < 1.5e9); m = 1000 (1024^2 2560 = 2.7e9): emulated
#:             product and emulated solve (1024 rows x 1280 x 1280 >= 1.5e9)
#:   emulated: n = 6000, m = 1100 (1152^2 6016 = 8e9): emulated solve and emulated lower product
#:   batch2:   DMMA only (the emulation serves single problems)
CASES = {f"n{n}_m{m}": (n, m, 1, "fp64", "plain") for n in (300, 2500) for m in (1, 127, 129, 1000)}
CASES.update({
    "emulated": (6000, 1100, 1, "fp64", "plain"),
    "batch2": (2500, 300, 2, "fp64", "plain"),
    "mean_hetero": (1500, 257, 1, "fp64", "mean_hetero"),
    "fp32_b1": (700, 300, 1, "fp32", "plain"),
    "fp32_b4": (300, 129, 4, "fp32", "mean_hetero"),
})
FP64_CASES = [c for c, v in CASES.items() if v[3] == "fp64"]
FP32_CASES = [c for c, v in CASES.items() if v[3] == "fp32"]
CLAIMS_AUTO = {"n300_m1000": (["v2", "v2"], [False]), "n2500_m129": (["v3", "v3"], [False]),
               "n2500_m1000": (["emulated", "emulated"], [True]), "emulated": (["emulated", "emulated"], [True]),
               "batch2": (["v3", "v3"], [False]), "fp32_b1": (["tc32", "tc32"], [False]),
               "fp32_b4": (["tc32", "tc32"], [False])}


def _mean_fn(a):
    return 0.3 * a.sum(-1) + 0.5


_EXACT = {}


def exact_problem(case):
    """Inputs (as the device sees them) and the oracle's posterior for every batch element (cached per case)."""
    if case in _EXACT:
        return _EXACT[case]
    n, m, B, dt, variant = CASES[case]
    rng = np.random.default_rng(list(CASES).index(case))
    npdt = np.float32 if dt == "fp32" else np.float64
    x = rng.uniform(-4, 4, (B, n, D)).astype(npdt).astype(np.float64)
    xs = rng.uniform(-4, 4, (B, m, D)).astype(npdt).astype(np.float64)
    y = rng.standard_normal((B, n)).astype(npdt).astype(np.float64)
    if variant == "mean_hetero":
        noise = (0.05 + 0.1 * rng.uniform(size=(B, n))).astype(npdt).astype(np.float64)
    else:
        noise = np.full((B, n), 0.1)
    eps = 1e-6 if dt == "fp32" else 1e-12
    out = {"x": x, "xs": xs, "y": y, "noise": noise, "eps": eps, "mean": [], "var": [], "kappa": 0.0}
    for b in range(B):
        mx = ms = None
        if variant == "mean_hetero":
            mx, ms = _mean_fn(x[b]), _mean_fn(xs[b])
        mean, var = O.posterior(SPEC, x[b], noise[b], y[b], xs[b], mean_x=mx, mean_xs=ms, eps=eps)
        out["mean"].append(mean[:, 0])
        out["var"].append(var)
        if dt == "fp32":
            out["kappa"] = max(out["kappa"], kappa(O.kernel_matrix(SPEC, x[b]) + np.diag(noise[b]) + eps * np.eye(n)))
    out["prior"] = O.kernel_elwise(SPEC, xs[0])[:, 0]  # stationary: the same at every point and batch
    _EXACT[case] = out
    return out


def exact_posterior(S, case):
    """``(post, xs)`` on the device for ``case``."""
    n, m, B, dt, variant = CASES[case]
    p = exact_problem(case)
    tdt = torch.float32 if dt == "fp32" else torch.float64
    S.B.epsilon = p["eps"]
    kern = 1.3 * S.EQ().stretch(1.1) + 0.4 * S.Matern52().stretch(0.8)
    f = S.GP(lambda a: 0.3 * a.sum(-1, keepdim=True) + 0.5, kern) if variant == "mean_hetero" else S.GP(kern)
    sl = (lambda a: a[0]) if B == 1 else (lambda a: a)
    x, xs = t(sl(p["x"]), tdt), t(sl(p["xs"]), tdt)
    y = t(sl(p["y"][..., None]), tdt)
    noise = t(sl(p["noise"]), tdt) if variant == "mean_hetero" else 0.1
    return f | (f(x, noise), y), xs


def exact_bounds(case):
    """``(bar against the oracle, bar between device routes)``."""
    p = exact_problem(case)
    if CASES[case][3] == "fp32":
        tol = C32 * U32 * p["kappa"]
        return tol, tol
    return TOL, SAME_TOL


def run_exact(S, paths, case, precision):
    n, m, B, dt, _ = CASES[case]
    p = exact_problem(case)
    S.B.precision = precision
    post, xs = exact_posterior(S, case)
    tol, same_tol = exact_bounds(case)
    mean = post(xs).mean  # factorises K_x (and solves for the mean)
    shp = (B, m) if B > 1 else (m,)

    paths.clear()
    var = dense(post(xs).var)
    taken = check_products(paths, precision, [(pad(m), pad(m), pad(n), True, 1.0)])
    solved = check_solves(paths, precision, pad(m), [pad(n)])
    paths.clear()
    mu, var_mv = post(xs).mean_var
    var_mv = dense(var_mv)
    taken += check_products(paths, precision, [(pad(m), pad(m), pad(n), True, 1.0)])
    if precision == "auto" and case in CLAIMS_AUTO:
        assert (taken, solved) == CLAIMS_AUTO[case], (case, taken, solved)

    # internal consistency
    assert var.shape == (B, m, m) if B > 1 else var.shape == (m, m)
    assert torch.equal(var, var.transpose(-1, -2)), "var is not bit-symmetric"
    assert torch.equal(var_mv, var), "mean_var's covariance differs from var's"
    assert torch.equal(mu, mean), "mean_var's mean differs from mean"
    mm, mv = post(xs).marginals()
    cm, lo, hi = post(xs).marginal_credible_bounds()
    prior = p["prior"][0]
    diag = torch.diagonal(var, dim1=-2, dim2=-1).clamp_min(0.0)
    d_err = (diag.double() - mv.double().reshape(diag.shape)).abs().max().item() / prior
    assert d_err <= same_tol, (case, precision, d_err)
    m_scale = max(1.0, max(np.abs(mb).max() for mb in p["mean"]))
    mm_err = (mm.double().reshape(shp) - mean.double().reshape(shp)).abs().max().item() / m_scale
    assert mm_err <= same_tol, (case, precision, mm_err)
    assert torch.equal(cm, mm)

    # against the oracle
    var_h, mean_h = host(var).reshape(B, m, m), host(mean).reshape(B, m)
    lo_h, hi_h = host(lo).reshape(B, m), host(hi).reshape(B, m)
    worst = 0.0
    for b in range(B):
        v_err = rel_err(var_h[b], p["var"][b], prior)  # stationary prior: sqrt(p_ii p_jj) = prior
        mu_err = rel_err(mean_h[b], p["mean"][b], m_scale)
        assert v_err <= tol, (case, precision, b, v_err, tol)
        assert mu_err <= tol, (case, precision, b, mu_err, tol)
        sd = 1.96 * np.sqrt(np.maximum(np.diag(p["var"][b]), 0.0))
        # |sqrt(a) - sqrt(b)| <= sqrt(|a - b|)
        b_tol = tol * m_scale + 1.96 * np.sqrt(tol * prior)
        assert np.abs(lo_h[b] - (p["mean"][b] - sd)).max() <= b_tol
        assert np.abs(hi_h[b] - (p["mean"][b] + sd)).max() <= b_tol
        worst = max(worst, v_err / tol, mu_err / tol)
    print(f"\n{case} {precision}: products {taken} solve emulated {solved}; worst error / bar {worst:.2e}, "
          f"diag vs marginals {d_err:.1e}" + (f", kappa {p['kappa']:.2e}" if dt == "fp32" else ""))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", FP64_CASES)
def test_exact_covariance(S, paths, case, precision):
    """``var``, ``mean_var`` and ``marginal_credible_bounds`` of an exact posterior, fp64, under every precision mode."""
    run_exact(S, paths, case, precision)


@pytest.mark.parametrize("case", FP32_CASES)
def test_exact_covariance_fp32(S, paths, case):
    """The same in fp32 (eps 1e-6): both products run on the 3xTF32 wgmma kernel."""
    run_exact(S, paths, case, "auto")


# ---------------------------------------------------------------------------------------------------------------------
# cross-covariances between different inputs or processes
# ---------------------------------------------------------------------------------------------------------------------
#: size -> (n, mx, my).  "emulated": the non-lower product is 1152 x 1536 x 2560 = 4.5e9 (>= 1.5e9) under "auto"
CROSS = {"native": (2500, 300, 517), "emulated": (2500, 1100, 1500)}
#: each process in the independent (a, b): f = 1.5 a + b, u1 = a, u2 = 0.5 a + b; so k_fi = 1.5 a_i EQ + b_i M52
CROSS_COEF = {"f": (1.5, 1.0), "u1": (1.0, 0.0), "u2": (0.5, 1.0)}


def _lin(ca, cb):
    return ("sum", ("scaled", ca, EQS), ("scaled", cb, M52S))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("size", list(CROSS))
def test_cross_covariances(S, paths, size, precision):
    """A measure of two independent processes a (EQ) and b (Matern52) with u1 = a, u2 = 0.5 a + b and f = u1 + u2 observed.
    ``post(f)(xa, xb)``, ``post(u2)(xa, xb)``, ``post[u1, u2](xa, xb)`` and ``post[u1, u2](xa)``: non-lower products with
    beta = 1, no mirror, against ``k_ij(xa, xb) - (L^-1 k_fi(x, xa))^T (L^-1 k_fj(x, xb))``."""
    n, mx, my = CROSS[size]
    rng = np.random.default_rng(31 + mx)
    x, xa, xb = (rng.uniform(-4, 4, (k, D)) for k in (n, mx, my))
    y = rng.standard_normal(n)
    S.B.precision = precision
    meas = S.Measure()
    a = S.GP(S.EQ().stretch(1.1), measure=meas)
    b = S.GP(S.Matern52().stretch(0.8), measure=meas)
    u1, u2 = a, 0.5 * a + b
    f = u1 + u2
    post = meas | (f(t(x), 0.1), t(y))
    xa_d, xb_d = t(xa), t(xb)
    post(f)(xa_d).mean  # factorise K_x

    L = O.chol_eps(O.kernel_matrix(_lin(2.25, 1.0), x) + 0.1 * np.eye(n))
    cases = [("f", "f", "xb"), ("u2", "u2", "xb"), ("u1", "u2", "xb"), ("u1", "u2", "xa")]
    procs = {"f": f, "u1": u1, "u2": u2}
    worst = 0.0
    for pi, pj, second in cases:
        x2, x2_d, m2 = (xb, xb_d, my) if second == "xb" else (xa, xa_d, mx)
        paths.clear()
        C = host(dense(post.kernels[procs[pi], procs[pj]](xa_d, x2_d)))
        taken = check_products(paths, precision, [(pad(mx), pad(m2), pad(n), False, 1.0)])
        if precision == "auto":
            assert taken == (["emulated"] if size == "emulated" else ["v3"]), (pi, pj, second, taken)
        (ai, bi), (aj, bj) = CROSS_COEF[pi], CROSS_COEF[pj]
        Vi = O._tri(L, O.kernel_matrix(_lin(1.5 * ai, bi), x, xa))
        Vj = O._tri(L, O.kernel_matrix(_lin(1.5 * aj, bj), x, x2))
        want = O.kernel_matrix(_lin(*_prior_coef(pi, pj)), xa, x2) - Vi.T @ Vj
        pa = O.kernel_elwise(_lin(*_prior_coef(pi, pi)), xa)[:, 0]
        pb = O.kernel_elwise(_lin(*_prior_coef(pj, pj)), x2)[:, 0]
        err = rel_err(C, want, np.sqrt(pa[:, None] * pb[None, :]))
        assert err <= TOL, (pi, pj, second, precision, err)
        worst = max(worst, err / TOL)
    print(f"\ncross {size} {precision}: worst error / bar {worst:.2e}")


def _prior_coef(pi, pj):
    """Coefficients of (EQ, M52) in the prior cross-kernel of two processes."""
    (ai, bi), (aj, bj) = CROSS_COEF[pi], CROSS_COEF[pj]
    return ai * aj, bi * bj


# ---------------------------------------------------------------------------------------------------------------------
# sparse var
# ---------------------------------------------------------------------------------------------------------------------
METHODS = ["vfe", "fitc", "dtc"]
OBS = {"vfe": "PseudoObs", "fitc": "PseudoObsFITC", "dtc": "PseudoObsDTC"}
SPARSE_SPEC = ("sum", ("scaled", 1.2, ("stretched", 1.7, ("matern52",))), ("scaled", 0.3, ("eq",)))
#: inducing points -> test points.  m = 1100: m_pad = 1152 splits 512 / 640 in the solve, so the solve's product is emulated
#: from 1.5e9 / (512 x 640) = 4578 rows on: 4600 test points (4608 rows) are the fewest that put it there
SPARSE = {129: 300, 1100: 4600}


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("m", list(SPARSE))
def test_sparse_covariance(S, paths, m, method):
    """``var`` of a sparse posterior (``PosteriorKernel + SubspaceKernel``) against ``oracle.sparse_posterior``; its diagonal
    against the streamed sparse marginals.  Inducing noise keeps ``K_z`` conditioned (cond <= ~2e5) at m = 1100."""
    ns = SPARSE[m]
    n = 2000
    rng = np.random.default_rng(7 + m)
    x, z, xs = rng.uniform(-3, 3, (n, D)), rng.uniform(-3, 3, (m, D)), rng.uniform(-3, 3, (ns, D))
    y = rng.standard_normal(n)
    noise = 0.05 + 0.1 * rng.uniform(size=n)
    noise_z = 0.01 + 0.02 * rng.uniform(size=m)
    f = S.GP(1.2 * S.Matern52().stretch(1.7) + 0.3 * S.EQ())
    obs = getattr(S, OBS[method])(f(t(z), t(noise_z)), f(t(x), t(noise)), t(y))
    post = f | obs
    xs_d = t(xs)
    mean = host(post(xs_d).mean)[:, 0]  # computes K_z, A and mu

    paths.clear()
    var = dense(post(xs_d).var)
    taken = check_products(paths, "auto", [(pad(ns), pad(ns), pad(m), True, 1.0), (pad(ns), pad(ns), pad(m), False, 0.0)])
    solved = check_solves(paths, "auto", pad(ns), [pad(m), pad(m)])
    if m == 1100:
        assert (taken, solved) == (["emulated", "emulated"], [True, True]), (taken, solved)
    _, mv = post(xs_d).marginals()

    mean_ref, var_ref = O.sparse_posterior(SPARSE_SPEC, z, x, noise, y, xs, method, noise_z=noise_z)
    prior = O.kernel_elwise(SPARSE_SPEC, xs)[:, 0]
    scale = np.sqrt(prior[:, None] * prior[None, :])
    var_h = host(var)
    err = rel_err(var_h, var_ref, scale)
    m_err = rel_err(mean, mean_ref[:, 0], max(1.0, np.abs(mean_ref).max()))
    asym = rel_err(var_h, var_h.T, scale)
    d_err = rel_err(np.maximum(np.diag(var_h), 0.0), host(mv), prior)
    print(f"\nsparse {method} m={m}: products {taken} solves emulated {solved}; var {err:.2e} mean {m_err:.2e} "
          f"asymmetry {asym:.1e} diag vs streamed marginals {d_err:.1e}")
    assert err <= TOL, err
    assert m_err <= TOL, m_err
    assert asym <= SAME_TOL, asym  # the exact part is mirrored; the subspace part is a plain A A^T product
    assert d_err <= SAME_TOL, d_err


# ---------------------------------------------------------------------------------------------------------------------
# multi-output posteriors
# ---------------------------------------------------------------------------------------------------------------------
#: block sizes; neither set is made of multiples of 128, so diagonal 128-tiles of the joint straddle blocks.  "large":
#: N = 2537, n_pad = 2560 >= 2048 -- the joint factor's trailing updates are emulated for a single fp64 problem
MO = {"small": [100, 157, 128, 1], "large": [1000, 1537]}
MO_D = 2
MO_EQ, MO_M32 = ("stretched", 0.9, ("eq",)), ("stretched", 1.6, ("matern32",))
MO_DELTA = [0.3, 0.0, 0.2, 0.1]


def _mo_spec(H, i, j):
    return ("sum", ("sum", ("scaled", float(H[i, 0] * H[j, 0]), MO_EQ), ("scaled", float(H[i, 1] * H[j, 1]), MO_M32)),
            ("scaled", MO_DELTA[i] * MO_DELTA[j], ("delta",)))


_MO = {}


def mo_problem(sizes, batch, dt):
    key = (sizes, batch, dt)
    if key in _MO:
        return _MO[key]
    ns = MO[sizes]
    p = len(ns)
    rng = np.random.default_rng(len(ns) * 10 + batch)
    npdt = np.float32 if dt == "fp32" else np.float64
    r = lambda *s: rng.uniform(-3, 3, s).astype(npdt).astype(np.float64)  # noqa: E731
    H = rng.standard_normal((p, 2))
    xs_in = [r(batch, k, MO_D) for k in ns]
    ys = [rng.standard_normal((batch, k)).astype(npdt).astype(np.float64) for k in ns]
    # mixed noise: a scalar for even blocks, a vector for odd ones
    noises = [0.05 * (i + 1) if i % 2 == 0 else (0.02 + 0.05 * rng.uniform(size=(batch, k))).astype(npdt).astype(np.float64)
              for i, k in enumerate(ns)]
    xt = r(batch, 300, MO_D)
    eps = 1e-6 if dt == "fp32" else 1e-12
    specs = [[_mo_spec(H, i, j) for j in range(p)] for i in range(p)]
    out = {"H": H, "x": xs_in, "y": ys, "noise": noises, "xt": xt, "eps": eps, "mean": [], "var": [], "kappa": 0.0}
    for b in range(batch):
        K = O.mo_block_kernel(specs, [xi[b] for xi in xs_in])
        K += np.diag(np.concatenate([np.full(k, nz) if np.ndim(nz) == 0 else nz[b] for k, nz in zip(ns, noises)]))
        L = O.chol_eps(K, eps)
        Kc = np.vstack([O.kernel_matrix(_mo_spec(H, i, 0), xs_in[i][b], xt[b]) for i in range(p)])
        V = O._tri(L, Kc)
        out["mean"].append((V.T @ O._tri(L, np.concatenate([yi[b] for yi in ys])[:, None]))[:, 0])
        out["var"].append(O.kernel_matrix(specs[0][0], xt[b]) - V.T @ V)
        if dt == "fp32":
            out["kappa"] = max(out["kappa"], kappa(K + eps * np.eye(K.shape[0])))
    out["prior"] = float(O.kernel_elwise(specs[0][0], xt[0][:1])[0, 0])
    _MO[key] = out
    return out


def mo_posterior(S, sizes, batch, dt):
    """``(measure, f_0, [(fdd_i, y_i)], test inputs)`` on the device."""
    p = mo_problem(sizes, batch, dt)
    tdt = torch.float32 if dt == "fp32" else torch.float64
    sl = (lambda a: a[0]) if batch == 1 else (lambda a: a)
    S.B.epsilon = p["eps"]
    meas = S.Measure()
    a = S.GP(S.EQ().stretch(0.9), measure=meas)
    b = S.GP(S.Matern32().stretch(1.6), measure=meas)
    e = S.GP(S.Delta(), measure=meas)
    H = p["H"]
    fs = []
    for i in range(len(MO[sizes])):
        fi = float(H[i, 0]) * a + float(H[i, 1]) * b
        fs.append(fi + MO_DELTA[i] * e if MO_DELTA[i] else fi)
    pairs = []
    for i, fi in enumerate(fs):
        nz = p["noise"][i]
        nz = nz if np.ndim(nz) == 0 else t(sl(nz), tdt)
        pairs.append((fi(t(sl(p["x"][i]), tdt), nz), t(sl(p["y"][i][..., None]), tdt)))
    return meas, fs[0], pairs, t(sl(p["xt"]), tdt)


@pytest.mark.parametrize("dt", ["fp64", "fp32"])
@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("sizes", list(MO))
def test_multi_output_posterior(S, paths, sizes, batch, dt):
    """Processes f_i = H_i1 a + H_i2 b (+ c_i e, e a Delta process) observed at blocks of different sizes with mixed noise;
    ``mean``, ``var_diag`` and ``var`` of the posterior of f_0 at new points against a NumPy joint (``mo_block_kernel`` +
    ``chol_eps``).  The joint is a ``BlockDense`` factorised in place; the cross rows take the dense + transpose route."""
    p = mo_problem(sizes, batch, dt)
    meas, f0, pairs, xt = mo_posterior(S, sizes, batch, dt)
    post = meas | tuple(pairs)
    paths.clear()
    fdd = post(f0)(xt)
    mean = host(fdd.mean).reshape(batch, -1)
    N = sum(MO[sizes])
    emulated_factor = check_factor(paths, pad(N), batch, dt)
    paths.clear()
    var = dense(post(f0)(xt).var)
    check_products(paths, "auto", [(pad(300), pad(300), pad(N), True, 1.0)])
    vd = host(post(f0)(xt).var_diag).reshape(batch, -1)
    assert torch.equal(var, var.transpose(-1, -2))

    if dt == "fp32":
        tol = same_tol = C32 * U32 * p["kappa"]
    else:
        tol, same_tol = TOL, SAME_TOL
    var_h = host(var).reshape(batch, 300, 300)
    prior = p["prior"]
    m_scale = max(1.0, max(np.abs(mb).max() for mb in p["mean"]))
    worst = 0.0
    for bi in range(batch):
        errs = (rel_err(mean[bi], p["mean"][bi], m_scale), rel_err(var_h[bi], p["var"][bi], prior),
                rel_err(vd[bi], np.diag(p["var"][bi]), prior))
        assert max(errs) <= tol, (sizes, batch, dt, bi, errs, tol)
        assert rel_err(np.diag(var_h[bi]), vd[bi], prior) <= same_tol
        worst = max(worst, max(errs) / tol)
    print(f"\nmulti-output {sizes} batch {batch} {dt}: factor emulated {emulated_factor}; worst error / bar {worst:.2e}"
          + (f", kappa {p['kappa']:.2e}" if dt == "fp32" else ""))


# ---------------------------------------------------------------------------------------------------------------------
# stale memory in the factorisation workspace
# ---------------------------------------------------------------------------------------------------------------------
STALE = [float("nan"), 1e300]


def _poisoned_workspace(monkeypatch, fill):
    """Make every factorisation workspace start out as ``fill`` in its matrix part (what a recycled allocation may hold):
    whatever the factorisation does not write stays ``fill``."""
    from stheno_b200 import ops

    real = ops._new_workspace

    def poisoned(B, n, k, device, dtype, rhs_t):
        W, n_pad, extra = real(B, n, k, device, dtype, rhs_t)
        W[:, :n_pad].fill_(fill)
        return W, n_pad, extra

    monkeypatch.setattr(ops, "_new_workspace", poisoned)


@pytest.mark.parametrize("sizes", list(MO))
def test_multi_output_factor_ignores_stale_workspace(S, monkeypatch, sizes):
    """The joint of a multi-output posterior is written block by block into the padded workspace, lower blocks only.  With
    the workspace pre-filled with NaN or 1e300 the posterior mean, covariance and the joint log-pdf are finite and bit-identical
    to those from a zero-filled workspace."""
    outs = {}
    for fill in [0.0] + STALE:
        with monkeypatch.context() as mp:
            _poisoned_workspace(mp, fill)
            meas, f0, pairs, xt = mo_posterior(S, sizes, 1, "fp64")
            post = meas | tuple(pairs)
            fdd = post(f0)(xt)
            outs[fill] = (fdd.mean, dense(fdd.var), torch.as_tensor(meas.logpdf(*pairs)))
    for fill in STALE:
        for got, want in zip(outs[fill], outs[0.0]):
            assert got.isfinite().all(), (sizes, fill)
            assert torch.equal(got, want), (sizes, fill)


@pytest.mark.parametrize("route", ["kernel", "dense"])
def test_single_output_factor_ignores_stale_workspace(S, monkeypatch, route):
    """Control for the multi-output case: ``chol_from_kernel`` (K1 writes whole diagonal tiles) and ``chol_from_dense`` (the
    padded copy) at n = 2537, with the factor, log-det, fused right-hand side and a solve through ``L_padded`` compared."""
    from stheno_b200 import ops

    rng = np.random.default_rng(3)
    n = 2537
    x = rng.uniform(-3, 3, (n, MO_D))
    xg = t(x / 0.9)[None, None]
    flat = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    rhs = t(rng.standard_normal((1, 1, n)))
    rows = t(rng.standard_normal((1, 256, pad(n))))
    rows[:, :, n:] = 0.0
    K = ops.kernel_matrix(flat, xg, noise_scalar=0.1)
    outs = {}
    for fill in [0.0] + STALE:
        with monkeypatch.context() as mp:
            _poisoned_workspace(mp, fill)
            if route == "kernel":
                ch = ops.chol_from_kernel(flat, xg, noise_scalar=0.1, jitter=1e-12, rhs_t=rhs, full_precision=True)
            else:
                ch = ops.chol_from_dense(K, jitter=1e-12, rhs_t=rhs)
            outs[fill] = (ch.L(), ch.logdet, ch.rhs_half().clone(), ch.solve_rows_(rows.clone()))
    for fill in STALE:
        for got, want in zip(outs[fill], outs[0.0]):
            assert got.isfinite().all(), (route, fill)
            assert torch.equal(got, want), (route, fill)


# ---------------------------------------------------------------------------------------------------------------------
# the benchmarked size: config 2's posterior_solve leg (n = 16384, d = 8, m = 4096, "auto")
# ---------------------------------------------------------------------------------------------------------------------
BENCH_SPEC = ("sum", ("stretched", 2.0, ("eq",)), ("scaled", 0.1, ("delta",)))
BENCH_ROWS = np.arange(7, 4096, 16)  # 256 full rows spread over the matrix
BENCH_BLOCK = (slice(1024, 1280), slice(3072, 3328))  # one 256 x 256 block far below the diagonal


@pytest.fixture(scope="module")
def bench_ref():
    """bench.py's inputs (seed 2, test points seed 22) and ONE host factorisation of n = 16384."""
    _threads()
    rng = np.random.default_rng(2)
    n, d, m = 16384, 8, 4096
    x = rng.standard_normal((n, d))
    y = rng.standard_normal(n)
    xs = np.random.default_rng(22).standard_normal((m, d))
    L = O.chol_eps(O.kernel_matrix(BENCH_SPEC, x))
    V = O._tri(L, O.kernel_matrix(BENCH_SPEC, x, xs))  # [n, m]
    mean = (V.T @ O._tri(L, y[:, None]))[:, 0]
    del L
    # Delta between the distinct test points of xs[rows] and xs is 1 exactly on the shared ones: the same-object identity
    rows = O.kernel_matrix(BENCH_SPEC, xs[BENCH_ROWS], xs) - V[:, BENCH_ROWS].T @ V
    r, c = BENCH_BLOCK
    block = O.kernel_matrix(BENCH_SPEC, xs[r], xs[c]) - V[:, r].T @ V[:, c]
    return {"x": x, "y": y, "xs": xs, "mean": mean, "rows": rows, "block": block}


def test_benchmarked_size(S, paths, bench_ref):
    """``mean_var`` at bench.py's posterior_solve inputs: one emulated solve of 4096 rows against n_pad = 16384 and one emulated
    lower product (4096 x 4096 x 16384), mirrored.  ``var`` is bit-symmetric, its diagonal and the mean meet ``marginals()``,
    and 256 full rows and a 256 x 256 block meet the oracle."""
    f = S.GP(S.EQ().stretch(2.0) + 0.1 * S.Delta())
    post = f | (f(t(bench_ref["x"])), t(bench_ref["y"]))
    xs = t(bench_ref["xs"])
    post(xs[:1]).mean  # factorise K_x
    paths.clear()
    mu, var = post(xs).mean_var
    var = dense(var)
    taken = check_products(paths, "auto", [(4096, 4096, 16384, True, 1.0)])
    solved = check_solves(paths, "auto", 4096, [16384])
    assert (taken, solved) == (["emulated"], [True])
    mm, mv = post(xs).marginals()
    prior = 1.1
    assert torch.equal(var, var.T)
    d_err = (torch.diagonal(var).clamp_min(0.0) - mv).abs().max().item() / prior
    mu = host(mu)[:, 0]
    m_scale = max(1.0, np.abs(bench_ref["mean"]).max())
    mm_err = np.abs(host(mm) - mu).max() / m_scale
    var_h = host(var)
    r, c = BENCH_BLOCK
    errs = (rel_err(var_h[BENCH_ROWS], bench_ref["rows"], prior), rel_err(var_h[r, c], bench_ref["block"], prior),
            rel_err(mu, bench_ref["mean"], m_scale))
    print(f"\nbenchmarked size: rows {errs[0]:.2e} block {errs[1]:.2e} mean {errs[2]:.2e}; diag vs marginals {d_err:.1e}, "
          f"mean vs marginals {mm_err:.1e}")
    assert d_err <= SAME_TOL and mm_err <= SAME_TOL, (d_err, mm_err)
    assert max(errs) <= TOL, errs
