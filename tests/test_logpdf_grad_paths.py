"""Gradients of ``logpdf`` where the analytic backward (``autograd._alpha_and_G``) runs its large solve and product on the
int8-slice emulation, on per-batch views, with several columns and in fp32 -- against torch fp64 autograd on the host
CPU through a dense restatement of each model (kernel, ``+ (noise + eps) I``, ``cholesky``, ``solve_triangular``), which
shares no code with libgpk, the emulation or cuSOLVER.

The backward forms ``K^-1 = L^-T L^-1`` from one solve of the ``n_pad x n_pad`` identity and one lower-tile product,
adds ``1/2 sum_c g_c alpha_c alpha_c^T`` through a ``round_up(k, 16)``-wide product and runs batches one at a time on
``[b:b+1]`` views.  The shapes follow libgpk's selection rules (``include/gpk.h``): a batch-1 product is emulated when
M, N, K >= 256 and M N K >= 1.5e9, and the recursive solve of ``rows`` right-hand sides is when its largest product
``rows x (n_pad - h) x h`` (h = n_pad / 2 in 128 tiles) is.

  case            dtype  B  n (n_pad)     k   backward under "auto"
  syrk_only       f64    1  1500 (1536)   1   K^-1 product emulated (1536^3); identity solve native (1536 768 768 < 1.5e9)
  solve_and_syrk  f64    1  2500 (2560)   3   identity solve and product emulated; factor on the 512-wide schedule
  pairs           f64    1  4700 (4736)  17   all emulated; pair-scheduled factor; the alpha product is 32 wide
  batched_views   f64    2  2500 (2560)   3   batched factor and solve native; per-batch K^-1 products emulated
  hetero          f64    1  2500 (2560)   1   vector noise that requires grad; identity solve and product emulated
  f32_batched     f32    4  2048          1   config 3's shape at a reduced batch: fp32 factor and products
  f32_single      f32    1  1500          3   fp32, batch 1
  dense_mo        f64    1  4 x 1024      1   dense_logpdf of an assembled ILMM joint: all emulated

Every fp64 case runs under "auto", "int8x8" and "fp64".  The in-situ launch profile around ``backward()`` shows the
emulation kernel ran (or, under "fp64", did not), and a spy on ``ops._emulation`` shows which operations asked for it
and with how many slices: under "auto" the backward's solve and products take 7, the factorisation the gradient is read
from takes 8 (a 7-slice factor costs the gradients up to 45x native fp64's error; see the sweep)."""
import math
import sys

import numpy as np
import pytest
import torch

PRECISIONS = ["auto", "int8x8", "fp64"]

#: the model of tests/test_autograd.py: var EQ(stretch scale) + var2 Matern52(stretch scale2); "variance" = var + var2
PARAMS = {"var": 1.3, "scale": 0.8, "var2": 0.6, "scale2": 1.7, "noise": 0.15, "lin": 0.3, "s": 0.05}
VARIANCE = PARAMS["var"] + PARAMS["var2"]

#: name -> (dtype, B, n, d, k, extras, operations the backward emulates under "auto" / "int8x8")
CASES = {
    "syrk_only": (torch.float64, 1, 1500, 5, 1, ("linear",), {"gemm_nt"}),
    "solve_and_syrk": (torch.float64, 1, 2500, 3, 3, (), {"gemm_nt", "solve_rows_"}),
    "pairs": (torch.float64, 1, 4700, 3, 17, ("delta",), {"gemm_nt", "solve_rows_"}),
    "batched_views": (torch.float64, 2, 2500, 3, 3, (), {"gemm_nt"}),
    "hetero": (torch.float64, 1, 2500, 3, 1, ("hetero",), {"gemm_nt", "solve_rows_"}),
    "f32_batched": (torch.float32, 4, 2048, 8, 1, (), set()),
    "f32_single": (torch.float32, 1, 1500, 5, 3, (), set()),
}
#: cases whose factorisation is emulated (n_pad >= 2048, batch 1): with 8 slices under "auto" too, because the backward
#: reads alpha and K^-1 element by element off the factor
FACTOR_EMULATED = {"solve_and_syrk", "pairs", "hetero", "dense_mo"}
F64_CASES = [c for c, v in CASES.items() if v[0] == torch.float64]
F32_CASES = [c for c, v in CASES.items() if v[0] == torch.float32]

#: B.epsilon of the fp64 cases and of the fp32 ones (the jitter the reference's examples use for float32)
EPS = {torch.float64: 1e-12, torch.float32: 1e-6}


# ---- inputs and the host reference --------------------------------------------------------------------------------------
def _weights(B, k):
    """Column weights of the loss ``sum w_bc lp_bc``: a negative and a zero among them (so ``g`` is not all ones), and a
    nonzero sum per batch member (so the ``K^-1`` term is not cancelled)."""
    base = torch.tensor([-0.75, 1.5, 0.0, 0.5, -1.25, 1.0], dtype=torch.float64)
    return base.repeat(-(-B * k // base.numel()))[: B * k].reshape(B, k)


def _inputs(case, dtype):
    """Seeded host inputs ``x [B, n, d]``, ``y [B, n, k]`` and the heteroscedastic profile ``t [n]``, in fp64 holding
    ``dtype``-representable values (fp32 cases: the reference sees the rounded inputs the GPU sees)."""
    _, B, n, d, k, _, _ = CASES[case]
    g = torch.Generator().manual_seed(n + 7 * k + B)
    x = torch.randn(B, n, d, dtype=torch.float64, generator=g) / math.sqrt(d)
    y = torch.sin(2 * x.sum(-1, keepdim=True)) + 0.5 * torch.randn(B, n, k, dtype=torch.float64, generator=g)
    t = torch.linspace(0, 1, n, dtype=torch.float64)
    return x.to(dtype).double(), y.to(dtype).double(), t


def _param_values(extras, dtype, noise):
    vals = dict(PARAMS, noise=noise)
    keep = {"var", "scale", "var2", "scale2", "noise"} | ({"lin"} if "linear" in extras else set()) | (
        {"s"} if "delta" in extras else set())
    return {name: float(torch.tensor(v, dtype=dtype)) for name, v in vals.items() if name in keep}


def _d2(x, s):
    """Squared distances of ``x / s`` in the difference form, one input dimension at a time."""
    xs = x / s
    out = 0.0
    for j in range(xs.shape[-1]):
        diff = xs[:, None, j] - xs[None, :, j]
        out = out + diff * diff
    return out


def ref_cov(p, x, extras):
    """The model's ``k(x, x)`` ``[n, n]`` in torch, differentiable w.r.t. ``p`` and ``x``."""
    K = p["var"] * torch.exp(-0.5 * _d2(x, p["scale"]))
    r2 = _d2(x, p["scale2"])
    s = math.sqrt(5.0) * torch.sqrt(torch.clamp_min(r2, 1e-30))
    K = K + p["var2"] * (1 + s + 5.0 / 3.0 * r2) * torch.exp(-s)
    if "linear" in extras:
        K = K + p["lin"] * (x @ x.T)
    if "delta" in extras:
        K = K + p["s"] * torch.eye(x.shape[0], dtype=x.dtype)
    return K


def ref_gaussian_logpdf(K, y, diag):
    """``log N(y_c; 0, K + diag(diag))`` for every column of ``y [n, k]`` -> ``[k]``."""
    n = K.shape[0]
    L = torch.linalg.cholesky(K + torch.diag(diag))
    a = torch.linalg.solve_triangular(L, y, upper=False)
    return -0.5 * (2 * torch.log(torch.diagonal(L)).sum() + n * math.log(2 * math.pi) + (a * a).sum(0))


def ref_logpdf(values, x, y, t, extras, eps, w, want_kappa=False):
    """fp64 autograd on the host: ``(lp [B, k], {name: gradient}, kappa)`` of ``sum w_bc lp_bc``, with kappa the largest
    condition number of the batch's ``K + noise + eps I`` (when asked)."""
    p = {name: torch.tensor(v, dtype=torch.float64, requires_grad=True) for name, v in values.items()}
    x, y = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    lps, kappa = [], 0.0
    for b in range(x.shape[0]):
        K = ref_cov(p, x[b], extras)
        diag = (p["noise"] * (1 + t) if "hetero" in extras else p["noise"] * torch.ones_like(t)) + eps
        lps.append(ref_gaussian_logpdf(K, y[b], diag))
        if want_kappa:
            ev = torch.linalg.eigvalsh((K + torch.diag(diag)).detach())
            kappa = max(kappa, (ev[-1] / ev[0]).item())
    lp = torch.stack(lps)
    (w * lp).sum().backward()
    grads = {name: v.grad for name, v in p.items()}
    grads.update(x=x.grad, y=y.grad)
    return lp.detach(), grads, kappa


@pytest.fixture(scope="module")
def refs():
    """One host reference per case (and per noise level of the sweep), shared between the precisions of the case."""
    return {}


def _reference(refs, case, noise=PARAMS["noise"]):
    key = (case, noise)
    if key not in refs:
        dtype, B, _, _, k, extras, _ = CASES[case]
        x, y, t = _inputs(case, dtype)
        values = _param_values(extras, dtype, noise)
        refs[key] = ref_logpdf(values, x, y, t, extras, EPS[dtype], _weights(B, k), want_kappa=dtype == torch.float32)
    return refs[key]


# ---- the GPU side -------------------------------------------------------------------------------------------------------
@pytest.fixture
def S():
    import stheno_b200 as S

    before = S.B.epsilon, S.B.precision
    yield S
    S.B.epsilon, S.B.precision = before


@pytest.fixture
def emulation_spy(monkeypatch):
    """``[(operation, slices)]`` of every ``ops._emulation`` request (slices 0: that call runs on the fp64 tensor cores)."""
    from stheno_b200 import ops

    calls = []
    real = ops._emulation

    def spy(*args, **kwargs):
        em = real(*args, **kwargs)
        calls.append((sys._getframe(1).f_code.co_name, em[0] if em else 0))
        return em

    monkeypatch.setattr(ops, "_emulation", spy)
    return calls


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


def _asked(spy):
    """``{operation: {slices}}`` of the emulated requests recorded by the spy since it was last cleared; clears it."""
    asked = {}
    for op, slices in spy:
        if slices:
            asked.setdefault(op, set()).add(slices)
    spy.clear()
    return asked


def _backward(loss, spy):
    """Run ``loss.backward()``: ``(emulation kernel launches, fp64 DMMA kernel launches, {operation: slices})`` of it."""
    from stheno_b200 import ops

    spy.clear()
    ops.gemm_profile(True)
    try:
        loss.backward()
        n_dmma, n_oz = ops.gemm_profile_read(0)[2], ops.gemm_profile_read(1)[2]
    finally:
        ops.gemm_profile(False)
    return n_oz, n_dmma, _asked(spy)


def gpu_logpdf(S, case, precision, spy, noise=PARAMS["noise"]):
    """``(lp [B, k], {name: gradient}, launches)`` of the library's ``logpdf`` and its backward, on the case's inputs."""
    dtype, B, n, _, k, extras, _ = CASES[case]
    S.B.epsilon, S.B.precision = EPS[dtype], precision
    x0, y0, t0 = _inputs(case, dtype)
    p = {name: torch.tensor(v, dtype=dtype, device="cuda", requires_grad=True)
         for name, v in _param_values(extras, dtype, noise).items()}
    # batch 1 goes through the unbatched API: x [n, d], y [n, k]
    x = (x0[0] if B == 1 else x0).to("cuda", dtype).requires_grad_(True)
    y = (y0[0] if B == 1 else y0).to("cuda", dtype).requires_grad_(True)
    kern = p["var"] * S.EQ().stretch(p["scale"]) + p["var2"] * S.Matern52().stretch(p["scale2"])
    if "linear" in extras:
        kern = kern + p["lin"] * S.Linear()
    if "delta" in extras:
        kern = kern + p["s"] * S.Delta()
    nz = p["noise"] * (1 + t0.to("cuda", dtype)) if "hetero" in extras else p["noise"]
    fdd = S.GP(kern)(x, nz)
    assert type(fdd.var).__name__ == "KernelDense", type(fdd.var).__name__  # not the Woodbury route of Linear()
    spy.clear()
    lp = fdd.logpdf(y).reshape(B, k)
    factor = _asked(spy)
    assert "_KernelLogpdfBackward" in _graph_nodes(lp)  # the analytic backward, not a torch restatement
    launches = _backward((_weights(B, k).to("cuda", dtype) * lp).sum(), spy)
    grads = {name: v.grad for name, v in p.items()}
    grads.update(x=x.grad.reshape(B, n, -1), y=y.grad.reshape(B, n, k))
    return lp.detach(), grads, (factor,) + launches


def _errors(got, want):
    """``{name: (max |got - want|, max(1, max |want|))}``."""
    return {name: ((got[name].double().cpu() - w).abs().max().item(), max(1.0, w.abs().max().item()))
            for name, w in want.items()}


def _check_path(case, precision, launches):
    """The factorisation asked for 8 slices where it is emulated (none under "fp64"); the backward launched the
    emulation kernel for the case's operations with 7 slices under "auto", 8 under "int8x8", and not at all under
    "fp64"."""
    factor, n_oz, _, asked = launches
    want_factor = {"_potrf": {8}} if case in FACTOR_EMULATED and precision != "fp64" else {}
    assert factor == want_factor, (case, precision, factor)
    want_ops = CASES[case][6] if case in CASES else {"gemm_nt", "solve_rows_"}
    if precision == "fp64":
        assert n_oz == 0 and not asked, (case, n_oz, asked)
    else:
        assert n_oz > 0, (case, precision, n_oz)
        slices = {"auto": 7, "int8x8": 8}[precision]
        assert asked == {op: {slices} for op in want_ops}, (case, precision, asked)


# ---- fp64 at the documented bar -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", F64_CASES)
def test_fp64_gradients(case, precision, refs, S, emulation_spy):
    """Noise >= 1e-2 of the variance (0.15 / 1.9): every gradient within ``1e-8 max(1, max |want|)`` -- the bar DESIGN.md
    documents for hyper-parameter gradients -- and every log-pdf within 1e-10 relative, the parity bar of the forward
    quantities."""
    want_lp, want, _ = _reference(refs, case)
    lp, got, launches = gpu_logpdf(S, case, precision, emulation_spy)
    errs = _errors(got, want)
    print(f"\n{case} {precision}: lp {((lp.cpu() - want_lp).abs() / want_lp.abs()).max().item():.2e} "
          + " ".join(f"{k} {e:.2e}/{s:.1e}" for k, (e, s) in errs.items()) + f" launches {launches}")
    assert ((lp.cpu() - want_lp).abs() <= 1e-10 * want_lp.abs()).all(), (lp, want_lp)
    for name, (err, scale) in errs.items():
        assert err <= 1e-8 * scale, (case, precision, name, err, scale)
    _check_path(case, precision, launches)


# ---- fp64 under a sweep of the conditioning --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("rel_noise", [1e-2, 1e-4, 1e-6])
def test_conditioning_sweep(rel_noise, refs, S, emulation_spy):
    """``solve_and_syrk`` with noise = rel_noise x variance and eps = 1e-12.  The condition number grows like 1 / rel_noise,
    and with it the reference's own error (``u kappa``), so the absolute bar is not the test: the emulated backwards must
    lose no more than native fp64 loses, ``err <= 10 err_fp64 + 1e-10 max(1, max |want|)`` per gradient and log-pdf.

    Measured on an H100 80GB HBM3 (400 W power limit), the largest gradient error over all gradients, relative to
    ``max(1, max |want|)``:

      noise / variance   fp64      auto      int8x8
      1e-2               2.0e-11   7.1e-12   1.6e-11
      1e-4               1.4e-9    1.5e-9    2.6e-10
      1e-6               6.2e-7    2.3e-7    1.3e-7

    With a 7-slice factorisation (what "auto" chose for a well-conditioned logpdf before it was given a gradient) the
    1e-2 row read 1.7e-10 for "auto", and the x gradient was 45x native fp64's error.  On an 8-slice factor, the 7-slice
    solve and products of the backward keep "auto" within 1.1x of native fp64's error in every row."""
    case = "solve_and_syrk"
    noise = rel_noise * VARIANCE
    want_lp, want, _ = _reference(refs, case, noise)
    res = {}
    for precision in ("fp64", "auto", "int8x8"):
        lp, got, launches = gpu_logpdf(S, case, precision, emulation_spy, noise)
        res[precision] = ((lp.cpu() - want_lp).abs().max().item(), _errors(got, want))
        print(f"\nsweep {rel_noise:.0e} {precision}: lp {res[precision][0]:.2e} "
              + " ".join(f"{k} {e:.2e}/{s:.1e}" for k, (e, s) in res[precision][1].items()) + f" launches {launches}")
        _check_path(case, precision, launches)
    lp_scale = want_lp.abs().max().item()
    for precision in ("auto", "int8x8"):
        assert res[precision][0] <= 10 * res["fp64"][0] + 1e-10 * lp_scale, (rel_noise, precision, "lp", res)
        for name, (err, scale) in res[precision][1].items():
            err64 = res["fp64"][1][name][0]
            assert err <= 10 * err64 + 1e-10 * scale, (rel_noise, precision, name, err, err64, scale)


# ---- fp32 ---------------------------------------------------------------------------------------------------------------
#: fp32 bar: err <= C32 2^-24 kappa(K) max(1, max |want|).  Measured on an H100 (both cases, kappa 8e3 and 1e4): at most
#: 6.5 u kappa max|want|, for var2.  Its gradient sum_ij G_ij phi_ij cancels about 7e5-fold, so the ~2e-4 element-wise
#: error of the fp32 K^-1 in G dominates; the K1-backward's own fp32 reduction contributes under 2 % of it.  C32 = 16 leaves
#: a 2.5x margin; a wrong batch offset or column gives O(1) relative errors, ~1e3 times the bar.
C32 = 16.0


@pytest.mark.gpu
@pytest.mark.parametrize("case", F32_CASES)
def test_fp32_gradients(case, refs, S, emulation_spy):
    """fp32 factor, solves and products against the fp64 reference on the fp32-rounded inputs and parameters.  The
    gradients are fp32 and within ``C32 2^-24 kappa max(1, max |want|)`` (kappa from the reference's eigenvalues); the
    log-pdfs within 1e-4 relative, config 3's parity bar.  No fp64 GEMM kernel runs."""
    want_lp, want, kappa = _reference(refs, case)
    lp, got, (factor, n_oz, n_dmma, asked) = gpu_logpdf(S, case, "auto", emulation_spy)
    assert lp.dtype == torch.float32 and all(g.dtype == torch.float32 for g in got.values())
    errs = _errors(got, want)
    u = 2.0**-24
    print(f"\n{case}: kappa {kappa:.3e} lp {((lp.cpu().double() - want_lp).abs() / want_lp.abs()).max().item():.2e} "
          + " ".join(f"{k} {e / (u * kappa * s):.2e}" for k, (e, s) in errs.items()))
    assert ((lp.cpu().double() - want_lp).abs() <= 1e-4 * want_lp.abs()).all(), (lp, want_lp)
    for name, (err, scale) in errs.items():
        assert err <= C32 * u * kappa * scale, (case, name, err, kappa, scale)
    assert (factor, n_oz, n_dmma, asked) == ({}, 0, 0, {})


# ---- assembled multi-output joint (dense_logpdf) ------------------------------------------------------------------------
MO_N, MO_P = 1024, 4
MO_H = [[1.0, 0.5], [-0.7, 1.2], [0.3, -0.9], [0.8, 0.4]]
MO_ELLS, MO_NOISE = [0.8, 1.9], 0.3


def _mo_inputs():
    g = torch.Generator().manual_seed(5)
    x = torch.linspace(0, 5, MO_N, dtype=torch.float64)
    y = torch.randn(MO_P * MO_N, dtype=torch.float64, generator=g)
    return x, y


def ref_mo(H, ells, noise, x, y, eps):
    """The ILMM joint ``logpdf``: blocks ``K_ik = sum_j H_ij H_kj EQ_j``, plus ``(noise + eps) I``."""
    m = H.shape[1]
    d2 = (x[:, None] - x[None, :]) ** 2
    Ks = [torch.exp(-0.5 * d2 / ells[j] ** 2) for j in range(m)]
    p = H.shape[0]
    K = torch.cat([torch.cat([sum(H[i, j] * H[k, j] * Ks[j] for j in range(m)) for k in range(p)], 1) for i in range(p)])
    return ref_gaussian_logpdf(K, y[:, None], (noise + eps) * torch.ones(K.shape[0], dtype=K.dtype))[0]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
def test_dense_multi_output_gradients(precision, refs, S, emulation_spy):
    """p = 4 outputs of m = 2 latent GPs on 1024 points each (N = 4096): the route of BASELINE config 5 (the assembled
    joint through ``dense_logpdf``), at a size where its factor, identity solve and product are emulated.  Gradients to
    H, both length scales, the noise and y at the fp64 bar (noise 0.3, variance <= 2.2)."""
    x0, y0 = _mo_inputs()
    w = -0.75
    if "dense_mo" not in refs:
        H, ells, noise = (torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (MO_H, MO_ELLS, MO_NOISE))
        y = y0.clone().requires_grad_(True)
        lp = ref_mo(H, ells, noise, x0, y, 1e-12)
        (w * lp).backward()
        refs["dense_mo"] = lp.detach(), {"H": H.grad, "ells": ells.grad, "noise": noise.grad, "y": y.grad}
    want_lp, want = refs["dense_mo"]

    S.B.epsilon, S.B.precision = 1e-12, precision
    H, ells, noise = (torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True)
                      for v in (MO_H, MO_ELLS, MO_NOISE))
    x, y = x0.cuda(), y0.cuda().requires_grad_(True)
    meas = S.Measure()
    us = [S.GP(S.EQ().stretch(ells[j]), measure=meas) for j in range(2)]
    fs = [H[i, 0] * us[0] + H[i, 1] * us[1] for i in range(MO_P)]
    emulation_spy.clear()
    lp = meas.logpdf(*[(fs[i](x, noise), y[i * MO_N:(i + 1) * MO_N]) for i in range(MO_P)])
    factor = _asked(emulation_spy)
    assert "_DenseLogpdfBackward" in _graph_nodes(lp)
    launches = (factor,) + _backward(w * lp, emulation_spy)
    got = {"H": H.grad, "ells": ells.grad, "noise": noise.grad, "y": y.grad}
    errs = _errors(got, want)
    print(f"\ndense_mo {precision}: lp {abs(lp.item() - want_lp.item()) / abs(want_lp.item()):.2e} "
          + " ".join(f"{k} {e:.2e}/{s:.1e}" for k, (e, s) in errs.items()) + f" launches {launches}")
    assert abs(lp.item() - want_lp.item()) <= 1e-10 * abs(want_lp.item())
    for name, (err, scale) in errs.items():
        assert err <= 1e-8 * scale, (precision, name, err, scale)
    _check_path("dense_mo", precision, launches)


# ---- the references themselves (host only) ------------------------------------------------------------------------------
def test_references_agree_with_independent_restatements():
    """At a tiny n on the host: ``ref_logpdf`` gives tests/test_autograd.py's ``torch_ref`` loss and gradients, and both
    references' log-pdfs equal SciPy's multivariate normal on the same covariance."""
    from scipy.stats import multivariate_normal

    from tests.test_autograd import torch_ref

    g = torch.Generator().manual_seed(0)
    n, d = 40, 3
    x = torch.randn(1, n, d, dtype=torch.float64, generator=g)
    y = torch.randn(1, n, 1, dtype=torch.float64, generator=g)
    t = torch.linspace(0, 1, n, dtype=torch.float64)
    values = _param_values((), torch.float64, 0.15)
    lp, grads, _ = ref_logpdf(values, x, y, t, (), 1e-12, torch.ones(1, 1))

    p = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in values.items()}
    xr, yr = x[0].clone().requires_grad_(True), y[0, :, 0].clone().requires_grad_(True)
    lr = torch_ref(xr, yr, p["var"], p["scale"], p["noise"], p["var2"], p["scale2"])
    lr.backward()
    assert abs(lp.item() - lr.item()) <= 1e-12 * abs(lr.item())
    for name in ("var", "scale", "var2", "scale2", "noise"):
        assert abs(grads[name].item() - p[name].grad.item()) <= 1e-11 * max(1.0, abs(p[name].grad.item())), name
    assert torch.allclose(grads["x"][0], xr.grad, rtol=1e-11, atol=1e-12)
    assert torch.allclose(grads["y"][0, :, 0], yr.grad, rtol=1e-11, atol=1e-12)

    # the extras and columns against SciPy
    extras = ("linear", "delta", "hetero")
    values = _param_values(extras, torch.float64, 0.15)
    y3 = torch.randn(1, n, 3, dtype=torch.float64, generator=g)
    lp3, _, _ = ref_logpdf(values, x, y3, t, extras, 1e-12, torch.ones(1, 3))
    pt = {k: torch.tensor(v, dtype=torch.float64) for k, v in values.items()}
    C = (ref_cov(pt, x[0], extras) + torch.diag(pt["noise"] * (1 + t) + 1e-12)).numpy()
    for c in range(3):
        want = multivariate_normal(np.zeros(n), C).logpdf(y3[0, :, c].numpy())
        assert abs(lp3[0, c].item() - want) <= 1e-11 * abs(want), c

    xm = torch.linspace(0, 5, 30, dtype=torch.float64)
    ym = torch.randn(60, dtype=torch.float64, generator=g)
    H = torch.tensor(MO_H[:2], dtype=torch.float64)
    lm = ref_mo(H, torch.tensor(MO_ELLS, dtype=torch.float64), torch.tensor(MO_NOISE, dtype=torch.float64), xm, ym, 1e-12)
    Ks = [np.exp(-0.5 * (xm.numpy()[:, None] - xm.numpy()[None, :]) ** 2 / ell**2) for ell in MO_ELLS]
    Hn = H.numpy()
    Cm = sum(np.kron(np.outer(Hn[:, j], Hn[:, j]), Ks[j]) for j in range(2)) + (MO_NOISE + 1e-12) * np.eye(60)
    want = multivariate_normal(np.zeros(60), Cm).logpdf(ym.numpy())
    assert abs(lm.item() - want) <= 1e-11 * abs(want)
