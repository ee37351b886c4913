"""Gradients w.r.t. the shape parameter of ``RQ(alpha)`` given as a torch tensor.

The K1-backward kernels form ``param_sum[f] = sum_ij G_ij c_t prod_{f' != f} phi_f' d phi_f / d alpha_f`` in the launches
that already form the term sums (``csrc/kernel_matrix_bwd.cu``).  ``d phi / d alpha = -phi h(w)``, ``w = d2 / (2 alpha)``,
``h(w) = log1p(w) - w / (1 + w)``; ``tests/_rq_model.py`` restates the device's ``h`` operation for operation.

The GPU references are torch fp64 autograd on the host of dense restatements.  Their RQ factor is a custom Function whose
alpha-derivative sums ``t^k / k`` (``t = w / (1 + w)``) for ``t <= 1/2`` and takes the direct form above: a different
formula from the kernel's, and one without the small-``w`` cancellation (else the reference, not the kernel, would set
the error there)."""
import math
import warnings

import numpy as np
import pytest
import torch

from tests import _rq_model as R

BAR = 1e-8  # relative to max(1, max |want|): the fp64 bar of tests/test_logpdf_grad_paths.py / test_sparse_elbo_grad.py
BAR32 = 1e-4  # fp32 kernel-level bar of tests/test_kernel_bwd.py


# ---- the host reference ---------------------------------------------------------------------------------------------------
def _h_ref(w):
    t = w / (1 + w)
    small = t <= 0.5
    ts = torch.where(small, t, torch.zeros_like(t))
    acc, tk = torch.zeros_like(w), ts * ts
    for k in range(2, 64):
        acc = acc + tk / k
        tk = tk * ts
    return torch.where(small, acc, torch.log1p(w) - t)


class _RQRef(torch.autograd.Function):
    """``(1 + d2 / (2 alpha))^-alpha`` with a stable alpha-derivative."""

    @staticmethod
    def forward(ctx, d2, alpha):
        w = d2 / (2 * alpha)
        phi = torch.exp(-alpha * torch.log1p(w))
        ctx.save_for_backward(w, phi)
        return phi

    @staticmethod
    def backward(ctx, g):
        w, phi = ctx.saved_tensors
        d_d2 = -phi / (2 * (1 + w))
        d_a = torch.where(phi == 0, torch.zeros_like(phi), -phi * _h_ref(w))
        return g * d_d2, (g * d_a).sum().reshape(())


def _d2(x, y):
    out = 0.0
    for j in range(x.shape[-1]):
        diff = x[..., :, None, j] - y[..., None, :, j]
        out = out + diff * diff
    return out


def ref_factor(kind, xs, ys, alpha=None, elwise=False):
    if kind == "lin":
        return (xs * ys).sum(-1) if elwise else xs @ ys.transpose(-1, -2)
    d2 = ((xs - ys) ** 2).sum(-1) if elwise else _d2(xs, ys)
    if kind == "eq":
        return torch.exp(-0.5 * d2)
    if kind == "m52":
        s = math.sqrt(5.0) * torch.sqrt(torch.clamp_min(d2, 1e-30))
        return (1 + s + 5.0 / 3.0 * d2) * torch.exp(-s)
    if kind == "rq":
        return _RQRef.apply(d2, alpha)
    raise ValueError(kind)


# A model: a list of terms (coefficient name, [(kind, length-scale name or None, alpha name or None)]); P maps names to
# tensors.  build() makes the library's kernel, ref() the dense restatement.
def build(S, model, P):
    k = 0
    for c, fs in model:
        t = None
        for kind, ell, a in fs:
            e = {"rq": lambda: S.RQ(P[a]), "eq": S.EQ, "m52": S.Matern52, "lin": S.Linear}[kind]()
            if ell is not None:
                e = e.stretch(P[ell])
            t = e if t is None else t * e
        k = k + P[c] * t
    return k


def ref(model, P, x, y, elwise=False):
    K = 0
    for c, fs in model:
        t = 1
        for kind, ell, a in fs:
            xs, ys = (x, y) if ell is None else (x / P[ell], y / P[ell])
            t = t * ref_factor(kind, xs, ys, None if a is None else P[a], elwise)
        K = K + P[c] * t
    return K


VALUES = {"c1": 1.3, "c2": 0.7, "l1": 0.8, "l2": 1.6, "a1": 0.7, "a2": 2.5}


def leaves(device, dtype=torch.float64, values=VALUES, grad=None):
    """Tensors for the model parameters; ``grad``: the names that require grad (all by default)."""
    return {k: torch.tensor(v, dtype=dtype, device=device, requires_grad=grad is None or k in grad)
            for k, v in values.items()}


# ---- host only ------------------------------------------------------------------------------------------------------------
def test_rq_construction():
    import stheno_b200 as S

    for a in (0.7, 2, np.float64(0.7), np.float32(0.5), np.array(1.5), torch.tensor(0.7), torch.tensor([0.7])):
        k = S.RQ(a)
        assert float(k.alpha) == pytest.approx(float(np.asarray(a, np.float64).reshape(())))
    assert isinstance(S.RQ(np.float64(0.7)).alpha, float)
    t = torch.tensor(0.7, dtype=torch.float64, requires_grad=True)
    k = S.RQ(t)
    assert k.alpha is t or (k.alpha.requires_grad and k.alpha.shape == ())
    assert k.flat_terms()[0][1][0][2] is k.alpha  # the raw alpha, not a float
    for bad in (0.0, -1.0, float("nan"), torch.tensor(-0.5), np.float64(0.0)):
        with pytest.raises(ValueError):
            S.RQ(bad)
    for vec in (torch.tensor([0.5, 0.7]), np.array([0.5, 0.7]), [0.5, 0.7]):
        with pytest.raises(ValueError):
            S.RQ(vec)
    assert str(S.RQ(0.5)) == "RQ(0.5)"
    assert str(S.RQ(torch.tensor(0.5, requires_grad=True))) == "RQ(0.5)"
    assert str(S.RQ(np.float64(0.7))) == "RQ(0.7)"


def test_grad_tensors_see_alpha():
    import stheno_b200 as S
    from stheno_b200.kernels import _grad_tensors

    a = torch.tensor(0.7, dtype=torch.float64, requires_grad=True)
    k = 1.3 * S.RQ(a).stretch(0.8) + S.EQ()
    assert _grad_tensors(k)
    assert not _grad_tensors(1.3 * S.RQ(0.7).stretch(0.8) + S.EQ())
    assert not _grad_tensors(S.RQ(torch.tensor(0.7)))  # a tensor that does not require grad
    with warnings.catch_warnings():
        warnings.simplefilter("error")  # building the descriptor converts a detached alpha: no UserWarning
        flat, _ = k._flat()
    assert flat.coef_raw is None and flat.param_raw is not None and _grad_tensors(flat)
    assert [p for p in flat.param_raw if p is not None] == [a]
    assert flat.terms[0][1][0] == ("rq", 0, 0.7)
    plain, _ = (1.3 * S.RQ(0.7).stretch(0.8) + S.EQ())._flat()
    assert plain.terms == flat.terms and plain.param_raw is None
    assert any(t is a for t in _grad_tensors(k))
    with torch.no_grad():
        assert _grad_tensors(k) == []


def test_h_model_against_mpmath():
    """``rq_h`` within 4 ulp of ``h`` wherever ``h`` is a normal number, for w from 1e-300 to 1e300; and
    ``-phi h`` (phi correctly rounded) within 4 ulp of ``d phi / d alpha`` for alpha from 1e-3 to 1e6."""
    rng = np.random.default_rng(0)
    ws = np.concatenate([np.logspace(-300, 300, 601), 10 ** rng.uniform(-300, 300, 200), rng.uniform(0, 3, 1500),
                         rng.uniform(3, 50, 200), [1.0, 2.0, 3.0, np.nextafter(3.0, 4.0)]])
    worst = 0.0
    for w in ws:
        want = R.exact_h(w)
        if float(want) < 2.3e-308:
            continue
        worst = max(worst, R.ulps(R.rq_h(w), want))
    print(f"\nh: worst {worst:.2f} ulp")
    assert worst <= 4.0
    import mpmath

    worst = 0.0
    for a in np.logspace(-3, 6, 10):
        for w in np.concatenate([np.logspace(-300, 300, 31), rng.uniform(0, 5, 10)]):
            d2 = float(w) * 2 * float(a)
            with mpmath.workdps(50):
                phi = float(mpmath.power(1 + mpmath.mpf(d2) / (2 * mpmath.mpf(a)), -mpmath.mpf(a)))
            want = R.exact_dphi_dalpha(d2, a)
            if abs(float(want)) < 2.3e-308:
                continue
            worst = max(worst, R.ulps(R.rq_dphi_dalpha(d2 / (2 * float(a)), phi), want))
    print(f"d phi / d alpha: worst {worst:.2f} ulp")
    assert worst <= 4.0
    # edges: w = 0, w = inf (phi = 0), NaN
    assert R.rq_h(0.0) == 0.0 and R.rq_dphi_dalpha(0.0, 1.0) == 0.0
    assert R.rq_dphi_dalpha(math.inf, 0.0) == 0.0
    assert math.isnan(R.rq_h(math.nan))


def test_kernel_torch_alpha_gradient_on_host():
    """``generic_grad.kernel_torch`` (the torch restatement of the sparse ELBO's torch route) differentiates alpha."""
    import mpmath

    import stheno_b200 as S
    from stheno_b200 import generic_grad

    a = torch.tensor(1.7, dtype=torch.float64, requires_grad=True)
    x = torch.linspace(0, 3, 7, dtype=torch.float64)[:, None]
    y = torch.linspace(0.5, 5, 5, dtype=torch.float64)[:, None]
    generic_grad.kernel_torch(S.RQ(a), x, y).sum().backward()
    want = sum(float(R.exact_dphi_dalpha(float((xi - yj) ** 2), 1.7)) for xi in x[:, 0].tolist() for yj in y[:, 0].tolist())
    assert abs(a.grad.item() - want) <= 1e-12 * abs(want)
    assert mpmath  # the derivative above is mpmath's


# ---- GPU: the kernels -----------------------------------------------------------------------------------------------------
@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.Measure, "default", None)
    return s


def _rect_pairs(dtype, ds, alphas):
    """``d phi / d alpha`` of single pairs (0, sqrt(d2)) through the rectangular backward: batch of m = n = 1, W = 1."""
    from stheno_b200 import _lib, ops

    B = len(ds)
    xs = torch.zeros(1, B, 1, 1, dtype=dtype, device="cuda")
    x = torch.tensor(ds, dtype=dtype, device="cuda").reshape(1, B, 1, 1)
    out = []
    for a in alphas:
        flat = ops.FlatKernel([(1.0, [("rq", 0, float(a))])], 1)
        W = torch.ones(B, 1, 1, dtype=dtype, device="cuda")
        ts = torch.zeros(B, _lib.GPK_MAX_TERMS, dtype=dtype, device="cuda")
        ps = torch.zeros(B, _lib.GPK_MAX_FACTORS, dtype=dtype, device="cuda")
        ops.kernel_cross_bwd(flat, xs, x, W=W, term_sum=ts, param_sum=ps)
        out.append((ts[:, 0].cpu(), ps[:, 0].cpu(), ps[:, 1:].cpu()))
    return out


@pytest.mark.gpu
def test_pair_derivative_against_mpmath():
    """Per pair: the rectangular backward (m = n = 1) and the square one (n = 2, G = off-diagonal ones) give
    ``d phi / d alpha`` within 4 ulp of ``-phi h_model(w)`` and of ``-phi h`` with mpmath's ``h`` (phi: the kernel's own
    value, read off term_sum; its rounding, up to alpha 2^-53 relative from 1 + w, is the forward's); 0 at d2 = 0 and where
    phi underflows."""
    from stheno_b200 import _lib, autograd, ops

    rng = np.random.default_rng(3)
    ds = np.concatenate([[0.0, 1e-160, 1e-9, 1e-4, 0.3, 1.0, 2.0, 3.5, 1e3, 1e9], 10 ** rng.uniform(-8, 4, 54)])
    alphas = [1e-3, 0.5, 2.5, 1e3, 1e6]
    for a, (phi, dpa, rest) in zip(alphas, _rect_pairs(torch.float64, ds.tolist(), alphas)):
        assert torch.all(rest == 0)  # no parameter: no sum
        for d, p, g in zip(ds.tolist(), phi.tolist(), dpa.tolist()):
            d2 = d * d
            w = d2 / (2 * a)
            model = R.rq_dphi_dalpha(w, p)
            if d2 == 0 or p == 0:
                assert g == 0.0, (a, d, g)
                continue
            want = -p * R.exact_h(w)  # mpmath's h times the kernel's phi (phi's rounding is the forward's own)
            if abs(float(want)) < 2.3e-308 or abs(model) < 2.3e-308:
                continue
            assert R.ulps(g, model) <= 4.0, (a, d, g, model)
            assert R.ulps(g, want) <= 4.0, (a, d, g, float(want))
    # the square kernel: n = 2, G off-diagonal ones -> param_sum = 2 d phi / d alpha
    for a in (0.5, 2.5):
        flat = ops.FlatKernel([(1.0, [("rq", 0, a)])], 1)
        for d in (1e-4, 0.7, 2.0, 40.0):
            xg = torch.tensor([[0.0], [d]], dtype=torch.float64, device="cuda").reshape(1, 1, 2, 1)
            G = torch.tensor([[0.0, 1.0], [1.0, 0.0]], dtype=torch.float64, device="cuda").reshape(1, 2, 2)
            ps = torch.zeros(1, _lib.GPK_MAX_FACTORS, dtype=torch.float64, device="cuda")
            ts, _, _ = autograd._bwd_kernel(flat, xg, G, 2, ps)
            phi = ts[0, 0].item() / 2
            assert R.ulps(ps[0, 0].item() / 2, R.rq_dphi_dalpha(d * d / (2 * a), phi)) <= 4.0
    # fp32: the factor and its derivative are formed in double, then rounded
    (phi, dpa, _), = _rect_pairs(torch.float32, [0.3, 1.0, 2.0], [0.7])
    for d, g in zip((0.3, 1.0, 2.0), dpa.tolist()):
        want = float(R.exact_dphi_dalpha(float(np.float32(d)) ** 2, 0.7))
        assert abs(g - want) <= 2 ** -22 * abs(want)


MODELS = {
    "rq": [("c1", [("rq", "l1", "a1")])],
    "rq_eq": [("c1", [("rq", "l1", "a1"), ("eq", "l2", None)])],
    "rq_m52": [("c1", [("rq", "l1", "a1"), ("m52", None, None)])],
    "rq_lin": [("c1", [("rq", "l1", "a1"), ("lin", None, None)])],
    "two_rq": [("c1", [("rq", "l1", "a1"), ("eq", "l2", None), ("rq", None, "a2"), ("m52", "l1", None)])],
    "two_groups": [("c1", [("rq", "l1", "a1")]), ("c2", [("rq", "l2", "a1"), ("eq", None, None)])],
}


def _kernel_case(S, model, x, z=None, *, dtype=torch.float64, grad=None, diag=False, seed=0):
    """``(got, want)`` gradient dicts of ``sum G o K`` for ``K = k(x)`` (``z`` None), ``k(x, z)``, or ``k.elwise(x)``
    (``diag``) through the library's differentiable kernel evaluations, and of the host restatement."""
    from stheno_b200 import autograd
    from stheno_b200.kernels import Input

    P = leaves("cuda", dtype, grad=grad)
    Q = leaves("cpu", torch.float64, grad=grad)
    k = build(S, model, P)
    flat, scales = k._flat()
    xg = Input(x.to("cuda", dtype)).scaled(scales)
    if diag:
        K = autograd.kernel_diag_grad(flat, xg)
        Kr = ref(model, Q, x.double(), x.double(), elwise=True)
    elif z is None:
        K = autograd.kernel_matrix_grad(flat, xg)
        Kr = ref(model, Q, x.double(), x.double())
    else:
        K = autograd.kernel_cross_grad(flat, xg, Input(z.to("cuda", dtype)).scaled(scales))
        Kr = ref(model, Q, x.double(), z.double())
    Kr = Kr.reshape(K.shape)
    g = torch.Generator().manual_seed(seed)
    Gw = torch.randn(K.shape, dtype=torch.float64, generator=g)
    (Gw.to("cuda", dtype) * K).sum().backward()
    (Gw * Kr).sum().backward()
    names = [n for n in P if P[n].requires_grad and any(n in (c,) + tuple(v for f in fs for v in f[1:]) for c, fs in model)]
    got = {n: P[n].grad for n in names}
    want = {n: Q[n].grad for n in names}
    return got, want


def _check(got, want, bar):
    for name, w in want.items():
        g = got[name]
        assert g is not None, name
        err = (g.double().cpu() - w).abs().max().item()
        scale = max(1.0, w.abs().max().item())
        assert err <= bar * scale, (name, err, scale)


def _points(n, d, seed, B=None, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    shape = (n, d) if B is None else (B, n, d)
    return (torch.randn(shape, dtype=torch.float64, generator=g) / math.sqrt(d)).to(dtype).double()


@pytest.mark.gpu
@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("route", ["square", "rect", "diag"])
def test_param_sum_models(S, model, route):
    x = _points(150, 3, 1)
    z = _points(70, 3, 2) if route == "rect" else None
    got, want = _kernel_case(S, MODELS[model], x, z, diag=route == "diag", grad={"a1", "a2"})
    assert set(got) <= {"a1", "a2"} and "a1" in got
    _check(got, want, BAR)
    if route == "diag":  # k(x_i, x_i) does not depend on alpha
        assert got["a1"].item() == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["batch3", "n1", "n63", "n65", "n300", "d132", "col_split", "dup_far"])
def test_param_sum_shapes(S, shape):
    model = MODELS["rq_eq"]
    if shape == "batch3":
        x = _points(90, 2, 4, B=3)
        got, want = _kernel_case(S, model, x)
        _check(got, want, BAR)
        got, want = _kernel_case(S, model, x, _points(40, 2, 5, B=3))
    elif shape.startswith("n"):
        n = int(shape[1:])
        got, want = _kernel_case(S, model, _points(n, 2, n))
        _check(got, want, BAR)
        got, want = _kernel_case(S, model, _points(n, 2, n + 1), _points(n + 2, 2, n + 2))
    elif shape == "d132":  # several dimension chunks: chunk 0 alone adds to param_sum (one length scale: K1's limit at d 132)
        x = _points(130, 132, 6)
        got, want = _kernel_case(S, MODELS["rq"], x)
        _check(got, want, BAR)
        got, want = _kernel_case(S, MODELS["rq"], x, _points(70, 132, 7))
    elif shape == "col_split":  # 3 rows x 5000 columns: the columns are split over CTAs, partials added atomically
        got, want = _kernel_case(S, model, _points(3, 2, 8), _points(5000, 2, 9))
    else:  # duplicated points (d2 = 0) and far ones (scaled distance 1e9); alpha alone requires grad (the length scales'
        # gradients through inputs of size 1e9 carry 1e9 ulp of cancellation in any restatement)
        x = _points(40, 2, 10)
        x = torch.cat([x, x[:5], x[5:8] + 1e9 * VALUES["l1"]])
        got, want = _kernel_case(S, model, x, grad={"a1"})
        _check(got, want, BAR)
        got, want = _kernel_case(S, model, x, torch.cat([x[:10], x[-2:]]), grad={"a1"})
    _check(got, want, BAR)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["square", "rect"])
def test_param_sum_fp32(S, route):
    x = _points(200, 3, 11, dtype=torch.float32)
    z = _points(90, 3, 12, dtype=torch.float32) if route == "rect" else None
    got, want = _kernel_case(S, MODELS["two_rq"], x, z, dtype=torch.float32, grad={"a1", "a2"})
    _check(got, want, BAR32)


@pytest.mark.gpu
def test_public_kernel_calls(S):
    """``k(x)``, ``k(x, y)`` and ``k.elwise(x)`` with alpha the only tensor that requires grad."""
    model = MODELS["rq_eq"]
    x, y = _points(120, 2, 13), _points(50, 2, 14)
    for call in ("kx", "kxy", "elwise"):
        P = leaves("cuda", grad={"a1"})
        Q = leaves("cpu", grad={"a1"})
        k = build(S, model, P)
        xc, yc = x.cuda(), y.cuda()
        if call == "kx":
            K, Kr = S.B.dense(k(xc)), ref(model, Q, x, x)
        elif call == "kxy":
            K, Kr = S.B.dense(k(xc, yc)), ref(model, Q, x, y)
        else:
            K, Kr = S.B.dense(k.elwise(xc)).reshape(-1), ref(model, Q, x, x, elwise=True)
        assert K.requires_grad, call
        Gw = torch.cos(torch.arange(Kr.numel(), dtype=torch.float64)).reshape(Kr.shape)
        (Gw.cuda() * K).sum().backward()
        (Gw * Kr).sum().backward()
        _check({"a1": P["a1"].grad}, {"a1": Q["a1"].grad}, BAR)


# ---- GPU: the model layer -------------------------------------------------------------------------------------------------
LP = {"v": 1.3, "l": 0.8, "alpha": 0.7, "noise": 0.1}


def _lp_inputs(n, B, dtype):
    g = torch.Generator().manual_seed(n + (B or 0))
    shape = (n, 3) if B is None else (B, n, 3)
    x = torch.randn(shape, dtype=torch.float64, generator=g)
    y = torch.sin(2 * x.sum(-1)) + 0.3 * torch.randn(x.shape[:-1], dtype=torch.float64, generator=g)
    return x.to(dtype).double(), y.to(dtype).double()


def _lp_ref(x, y, grad, eps):
    """fp64 host autograd of ``v RQ(alpha).stretch(l) + EQ()`` + noise: ``(lp [B], grads, kappa)``."""
    p = {k: torch.tensor(v, dtype=torch.float64, requires_grad=k in grad) for k, v in LP.items()}
    xs = x if x.dim() == 3 else x[None]
    ys = y if y.dim() == 2 else y[None]
    lps, kappa = [], 0.0
    for b in range(xs.shape[0]):
        d2 = _d2(xs[b] / p["l"], xs[b] / p["l"])
        K = p["v"] * _RQRef.apply(d2, p["alpha"]) + torch.exp(-0.5 * _d2(xs[b], xs[b]))
        K = K + (p["noise"] + eps) * torch.eye(K.shape[0], dtype=K.dtype)
        L = torch.linalg.cholesky(K)
        a = torch.linalg.solve_triangular(L, ys[b][:, None], upper=False)
        n = K.shape[0]
        lps.append(-0.5 * (2 * torch.log(torch.diagonal(L)).sum() + n * math.log(2 * math.pi) + (a * a).sum()))
        ev = torch.linalg.eigvalsh(K.detach())
        kappa = max(kappa, (ev[-1] / ev[0]).item())
    lp = torch.stack(lps)
    lp.sum().backward()
    return lp.detach(), {k: v.grad for k, v in p.items() if v.requires_grad}, kappa


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


def _lp_gpu(S, x, y, grad, dtype, alpha=None):
    p = {k: torch.tensor(v, dtype=dtype, device="cuda", requires_grad=k in grad) for k, v in LP.items()}
    a = p["alpha"] if alpha is None else alpha
    f = S.GP(p["v"] * S.RQ(a).stretch(p["l"]) + S.EQ())
    fdd = f(x.to("cuda", dtype), p["noise"])
    assert type(fdd.var).__name__ == "KernelDense"
    lp = fdd.logpdf(y.to("cuda", dtype) if y.dim() == 1 else y.to("cuda", dtype)[..., None])  # batched: [B, n, 1]
    return lp, p


@pytest.fixture(scope="module")
def lp_refs():
    return {}


@pytest.mark.gpu
@pytest.mark.parametrize("n", [700, 2500])
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
@pytest.mark.parametrize("which", ["alpha", "all"])
def test_logpdf_alpha_gradient(S, monkeypatch, lp_refs, n, precision, which):
    grad = {"alpha"} if which == "alpha" else set(LP)
    x, y = _lp_inputs(n, None, torch.float64)
    key = (n, which)
    if key not in lp_refs:
        lp_refs[key] = _lp_ref(x, y, grad, 1e-12)
    want_lp, want, _ = lp_refs[key]
    monkeypatch.setattr(S.B, "precision", precision)
    lp, p = _lp_gpu(S, x, y, grad, torch.float64)
    assert "_KernelLogpdfBackward" in _graph_nodes(lp)
    lp.sum().backward()
    assert abs(lp.item() - want_lp.item()) <= 1e-10 * abs(want_lp.item())
    _check({k: p[k].grad for k in grad}, want, BAR)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_logpdf_alpha_gradient_batched_and_fp32(S, monkeypatch, dtype):
    """Batch 2 in fp64; batch 1 and 2 in fp32 at the bar of the fp32 log-pdf gradients,
    16 2^-24 kappa max(1, max |want|)."""
    eps = 1e-12 if dtype == torch.float64 else 1e-6
    monkeypatch.setattr(S.B, "epsilon", eps)
    for B in ((2,) if dtype == torch.float64 else (None, 2)):
        x, y = _lp_inputs(500, B, dtype)
        lp_w, want, kappa = _lp_ref(x, y, set(LP), eps)
        lp, p = _lp_gpu(S, x, y, set(LP), dtype)
        assert "_KernelLogpdfBackward" in _graph_nodes(lp)
        lp.sum().backward()
        bar = BAR if dtype == torch.float64 else 16 * 2 ** -24 * kappa
        _check({k: p[k].grad for k in LP}, want, bar)


@pytest.mark.gpu
def test_exact_posterior_alpha_only(S):
    """mean, marginals and the full covariance of the posterior at m = 5000 test points (two 4096-chunks for the
    marginals), alpha the only tensor that requires grad, against the host restatement."""
    g = torch.Generator().manual_seed(21)
    n, m = 400, 5000
    x = torch.randn(n, 2, dtype=torch.float64, generator=g)
    y = torch.sin(x.sum(-1)) + 0.2 * torch.randn(n, dtype=torch.float64, generator=g)
    xs = 1.5 * torch.randn(m, 2, dtype=torch.float64, generator=g)
    wm = torch.cos(torch.arange(m, dtype=torch.float64))
    wv = torch.sin(torch.arange(m, dtype=torch.float64))

    a = torch.tensor(LP["alpha"], dtype=torch.float64, requires_grad=True)
    v, l, nz = LP["v"], LP["l"], LP["noise"]

    def kf(p, q):
        return v * _RQRef.apply(_d2(p / l, q / l), a) + torch.exp(-0.5 * _d2(p, q))

    L = torch.linalg.cholesky(kf(x, x) + (nz + 1e-12) * torch.eye(n, dtype=torch.float64))
    V = torch.linalg.solve_triangular(L, kf(xs, x).T, upper=False)  # [n, m]
    mean_r = V.T @ torch.linalg.solve_triangular(L, y[:, None], upper=False)[:, 0]
    var_r = (v + 1.0) - (V * V).sum(0)
    Vm, Vv = V @ wm, V @ wv
    cov_r = wm @ kf(xs, xs) @ wv - Vm @ Vv  # wm^T C wv
    want = {}
    for name, loss in (("mean", wm @ mean_r), ("marginals", wm @ mean_r + wv @ var_r), ("cov", cov_r)):
        want[name] = torch.autograd.grad(loss, a, retain_graph=True)[0]

    for name in want:
        ag = torch.tensor(LP["alpha"], dtype=torch.float64, device="cuda", requires_grad=True)
        f = S.GP(LP["v"] * S.RQ(ag).stretch(LP["l"]) + S.EQ())
        fdd = (f | (f(x.cuda(), LP["noise"]), y.cuda()))(xs.cuda())
        if name == "mean":
            loss = wm.cuda() @ S.B.dense(fdd.mean).reshape(-1)
        elif name == "marginals":
            mu, var = fdd.marginals()
            loss = wm.cuda() @ mu.reshape(-1) + wv.cuda() @ var.reshape(-1)
        else:
            loss = wm.cuda() @ S.B.dense(fdd.var) @ wv.cuda()
        assert loss.requires_grad, name
        loss.backward()
        _check({"a": ag.grad}, {"a": want[name]}, BAR)


def _sparse_problem(S, method, n, m, alpha):
    g = torch.Generator().manual_seed(n + m)
    x = (torch.randn(n, 2, dtype=torch.float64, generator=g)).cuda()
    z = (torch.randn(m, 2, dtype=torch.float64, generator=g)).cuda()
    y = (torch.sin(x.sum(-1).cpu()) + 0.3 * torch.randn(n, dtype=torch.float64, generator=g)).cuda()
    k = 1.2 * S.RQ(alpha).stretch(0.9) + 0.3 * S.EQ()
    gp = S.GP(k)
    cls = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[method]
    return gp, x, z, y, cls


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["vfe", "fitc", "dtc"])
def test_sparse_elbo_shared_alpha(S, monkeypatch, method):
    """One alpha tensor in k_z, k_zx and k_x: the streamed analytic route, against ``sparse_compute_torch``."""
    from stheno_b200 import autograd
    from stheno_b200.generic_grad import sparse_compute_torch

    calls = []
    real = autograd.sparse_elbo
    monkeypatch.setattr(autograd, "sparse_elbo", lambda *a, **kw: calls.append(1) or real(*a, **kw))
    a = torch.tensor(0.6, dtype=torch.float64, device="cuda", requires_grad=True)
    gp, x, z, y, cls = _sparse_problem(S, method, 900, 40, a)
    e = cls(gp(z), gp(x, 0.1), y).elbo(gp.measure)
    assert calls, "the streamed analytic route was not taken"
    (got,) = torch.autograd.grad(e, a)
    meas = gp.measure
    er = sparse_compute_torch(method, meas.kernels[gp], meas.kernels[gp, gp], meas.kernels[gp], z, x,
                              torch.full((900,), 0.1, dtype=torch.float64, device="cuda"), None, y[:, None],
                              torch.zeros(40, 1, dtype=torch.float64, device="cuda"), S.B.epsilon)[3]
    (want,) = torch.autograd.grad(er, a)
    assert abs(float(e) - float(er)) <= 1e-10 * abs(float(er))
    assert abs(got.item() - want.item()) <= BAR * max(1.0, abs(want.item())), (got.item(), want.item())


@pytest.mark.gpu
def test_sparse_elbo_batched_torch_route(S):
    """A batched problem goes through the torch restatement: alpha's gradient against a finite difference."""
    def elbo(av):
        a = torch.tensor(av, dtype=torch.float64, device="cuda", requires_grad=True)
        g = torch.Generator().manual_seed(3)
        x = torch.randn(2, 200, 2, dtype=torch.float64, generator=g).cuda()
        z = torch.randn(2, 15, 2, dtype=torch.float64, generator=g).cuda()
        y = torch.randn(2, 200, dtype=torch.float64, generator=g).cuda()
        gp = S.GP(S.RQ(a).stretch(0.9))
        return S.PseudoObs(gp(z), gp(x, 0.1), y[..., None]).elbo(gp.measure), a

    e, a = elbo(0.8)
    e.sum().backward()
    h = 1e-5
    with torch.no_grad():
        fd = (elbo(0.8 + h)[0].sum() - elbo(0.8 - h)[0].sum()).item() / (2 * h)
    assert abs(a.grad.item() - fd) <= 1e-6 * max(1.0, abs(fd)), (a.grad.item(), fd)


@pytest.mark.gpu
def test_multi_output_joint_rq_latent(S):
    """A 4-output ILMM whose first latent is RQ(alpha): the joint logpdf through ``Measure.logpdf``."""
    n, p = 300, 4
    H = torch.tensor([[1.0, 0.3], [0.5, -0.8], [-0.4, 0.9], [0.7, 0.2]], dtype=torch.float64)
    xg = torch.linspace(0, 5, n, dtype=torch.float64)
    yg = torch.randn(p * n, dtype=torch.float64, generator=torch.Generator().manual_seed(9))
    a_r = torch.tensor(0.9, dtype=torch.float64, requires_grad=True)
    d2 = (xg[:, None] - xg[None, :]) ** 2
    Ks = [_RQRef.apply(d2 / 0.7 ** 2, a_r), torch.exp(-0.5 * d2 / 1.3 ** 2)]
    K = torch.cat([torch.cat([sum(H[i, j] * H[k, j] * Ks[j] for j in range(2)) for k in range(p)], 1) for i in range(p)])
    K = K + (0.3 + 1e-12) * torch.eye(p * n, dtype=torch.float64)
    L = torch.linalg.cholesky(K)
    al = torch.linalg.solve_triangular(L, yg[:, None], upper=False)
    lp_r = -0.5 * (2 * torch.log(torch.diagonal(L)).sum() + p * n * math.log(2 * math.pi) + (al * al).sum())
    lp_r.backward()

    a = torch.tensor(0.9, dtype=torch.float64, device="cuda", requires_grad=True)
    meas = S.Measure()
    us = [S.GP(S.RQ(a).stretch(0.7), measure=meas), S.GP(S.EQ().stretch(1.3), measure=meas)]
    Hc = H.cuda()
    fs = [Hc[i, 0] * us[0] + Hc[i, 1] * us[1] for i in range(p)]
    x, y = xg.cuda(), yg.cuda()
    lp = meas.logpdf(*[(fs[i](x, 0.3), y[i * n:(i + 1) * n]) for i in range(p)])
    lp.backward()
    assert abs(lp.item() - lp_r.item()) <= 1e-10 * abs(lp_r.item())
    _check({"a": a.grad}, {"a": a_r.grad}, BAR)


# ---- unchanged behaviour --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_forward_values_and_other_gradients_unchanged(S):
    """Float alpha, tensor alpha and tensor alpha that requires grad give bit-identical log-pdf, posterior marginals and
    ELBO.  With every other parameter requiring grad, their gradients are bit-identical whether alpha requires grad or not
    (n = 64: one CTA forms each term sum, so no atomic order differs between runs), within 1e-14 at n = 600 (the term sums
    are added atomically across CTAs, in an order that varies from run to run), and backward() launches the same kernels."""
    from stheno_b200 import ops

    for n in (64, 600):
        x, y = _lp_inputs(n, None, torch.float64)
        xc, yc = x.cuda(), y.cuda()
        xs = xc[:50] + 0.1

        def values(alpha):
            f = S.GP(LP["v"] * S.RQ(alpha).stretch(LP["l"]) + S.EQ())
            lp = f(xc, LP["noise"]).logpdf(yc)
            mu, var = (f | (f(xc, LP["noise"]), yc))(xs).marginals()
            e = S.PseudoObs(f(xc[:30]), f(xc, LP["noise"]), yc).elbo(f.measure)
            return [torch.as_tensor(t).detach().reshape(-1).cpu() for t in (lp, mu, var, e)]

        base = values(LP["alpha"])
        for alpha in (torch.tensor(LP["alpha"], dtype=torch.float64, device="cuda"),
                      torch.tensor(LP["alpha"], dtype=torch.float64, device="cuda", requires_grad=True)):
            for a_, b_ in zip(base, values(alpha)):
                assert torch.equal(a_, b_), n

        out = []
        for alpha_grad in (False, True):
            grad = set(LP) - ({"alpha"} if not alpha_grad else set())
            p = {k: torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=k in grad) for k, v in LP.items()}
            alpha = p["alpha"] if alpha_grad else LP["alpha"]
            lp = S.GP(p["v"] * S.RQ(alpha).stretch(p["l"]) + S.EQ())(xc, p["noise"]).logpdf(yc)
            ops.launch_count(reset=True)
            lp.backward()
            torch.cuda.synchronize()
            out.append(({k: p[k].grad.clone() for k in ("v", "l", "noise")}, ops.launch_count()))
        (g0, n0), (g1, n1) = out
        assert n0 == n1, (n, n0, n1)
        for k in g0:
            if n == 64 or k != "v":  # l and noise come from grad_xg and diag, written without atomics
                assert torch.equal(g0[k], g1[k]), (n, k)
            else:
                assert abs(g0[k].item() - g1[k].item()) <= 1e-14 * abs(g0[k].item()), (n, k)


@pytest.mark.gpu
def test_kernel_outputs_bit_identical_with_param_sum():
    """term_sum, grad_xg and diag of the square backward and term_sum and both gradients of the rectangular one are the
    same with and without param_sum: bit for bit where one CTA forms each sum (64 rows, 64 columns; d = 132: several
    dimension chunks), within 1e-14 where CTAs add their partials atomically (300 rows, 5000 columns split over CTAs)."""
    from stheno_b200 import _lib, autograd, ops

    for n, m, d, exact in ((64, 64, 3, True), (60, 50, 132, True), (300, 5000, 3, False)):
        G_ = 1 if d > 100 else 2  # two length-scale groups of 132 dimensions do not fit the kernels' shared memory
        flat = ops.FlatKernel([(1.3, [("rq", 0, 0.7), ("eq", G_ - 1)]), (0.4, [("rq", G_ - 1, 2.0)])], G_)
        g = torch.Generator().manual_seed(n)
        xg = torch.randn(G_, 1, n, d, dtype=torch.float64, generator=g).cuda()
        zg = torch.randn(G_, 1, m, d, dtype=torch.float64, generator=g).cuda()
        G = torch.randn(1, n, n, dtype=torch.float64, generator=g).cuda()
        G = G + G.transpose(1, 2)
        W = torch.randn(1, n, m, dtype=torch.float64, generator=g).cuda()
        outs = []
        for want in (False, True):
            ps = torch.zeros(1, _lib.GPK_MAX_FACTORS, dtype=torch.float64, device="cuda") if want else None
            sq = autograd._bwd_kernel(flat, xg, G, n, ps)
            ts = torch.zeros(1, _lib.GPK_MAX_TERMS, dtype=torch.float64, device="cuda")
            gx, gz = torch.zeros_like(xg), torch.zeros_like(zg)
            ps2 = torch.zeros(1, _lib.GPK_MAX_FACTORS, dtype=torch.float64, device="cuda") if want else None
            ops.kernel_cross_bwd(flat, xg, zg, W=W, term_sum=ts, grad_xsg=gx, grad_xg=gz, param_sum=ps2)
            outs.append(list(sq) + [ts, gx, gz])
            if want:  # sums for the RQ factors 0 and 2, none for EQ (1) or past the last factor
                for q in (ps, ps2):
                    assert q[0, 0] != 0 and q[0, 2] != 0 and q[0, 1] == 0 and torch.all(q[0, 3:] == 0)
        for i, (a_, b_) in enumerate(zip(*outs)):
            if exact or i in (1, 2):  # the square kernel's grad_xg and diag are written without atomics
                assert torch.equal(a_, b_), (n, m, d, i)
            else:
                assert (a_ - b_).abs().max() <= 1e-14 * max(1.0, a_.abs().max().item()), (n, m, d, i)


# ---- end to end -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_end_to_end_learns_alpha(S):
    """n = 3000 points sampled from an RQ(0.5) GP: the first gradient of logpdf w.r.t. log alpha, log l and log noise
    matches central differences of the GPU forward, and a short Adam run moves alpha toward 0.5."""
    g = torch.Generator().manual_seed(17)
    n = 3000
    x = torch.rand(n, 1, dtype=torch.float64, generator=g) * 10
    d2 = (x - x.T) ** 2
    K = (1 + d2 / (2 * 0.5 * 0.8 ** 2)) ** -0.5 + 0.05 * torch.eye(n, dtype=torch.float64)
    y = torch.linalg.cholesky(K) @ torch.randn(n, dtype=torch.float64, generator=g)
    xc, yc = x.cuda(), y.cuda()

    def lp_of(la, ll, ln):
        f = S.GP(S.RQ(torch.exp(la)).stretch(torch.exp(ll)))
        return f(xc, torch.exp(ln)).logpdf(yc)

    theta = [torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True)
             for v in (math.log(2.0), math.log(1.0), math.log(0.1))]
    lp = lp_of(*theta)
    grads = torch.autograd.grad(lp, theta)
    h = 1e-5
    with torch.no_grad():
        for i in range(3):
            up = [t.detach().clone() for t in theta]
            dn = [t.detach().clone() for t in theta]
            up[i] += h
            dn[i] -= h
            fd = (lp_of(*up) - lp_of(*dn)).item() / (2 * h)
            assert abs(grads[i].item() - fd) <= 1e-6 * max(1.0, abs(fd)), (i, grads[i].item(), fd)
    opt = torch.optim.Adam(theta, lr=0.1)
    start = abs(math.exp(theta[0].item()) - 0.5)
    for _ in range(15):
        opt.zero_grad()
        (-lp_of(*theta) / n).backward()
        opt.step()
    assert abs(math.exp(theta[0].item()) - 0.5) < 0.7 * start, math.exp(theta[0].item())
