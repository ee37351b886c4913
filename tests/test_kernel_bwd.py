"""K1 backward (``csrc/kernel_matrix_bwd.cu``) against torch fp64 autograd of ``sum(G * K(xg, coefs))`` with K restated in
torch in the reference library's convention: distance ``|x - y|`` at d = 1 and ``sqrt(max(d2, 1e-30))`` for d > 1 (so
Matern-1/2 has the subgradient 0 at coincident points), Delta = the identity.  Covers every kind, products of up to four
factors, several groups, batches, ragged row counts, fp32, duplicated and nearly coincident inputs, and widths up to
d = 132 -- beyond what one launch's shared memory holds, so the kernel runs in chunks of dimensions."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _phi(kind, x, param):
    """``phi(x_i, x_j)`` ``[B, n, n]`` for ``x [B, n, d]`` (differentiable)."""
    B, n, d = x.shape
    if kind == "linear":
        return x @ x.transpose(1, 2)
    if kind == "delta":
        return torch.eye(n, dtype=x.dtype, device=x.device).expand(B, n, n)
    if kind == "one":
        return torch.ones(B, n, n, dtype=x.dtype, device=x.device)
    diff = x[:, :, None, :] - x[:, None, :, :]
    d2 = (diff * diff).sum(-1)
    if kind == "eq":
        return torch.exp(-0.5 * d2)
    if kind == "rq":
        return (1 + d2 / (2 * param)) ** (-param)
    r = diff.abs()[..., 0] if d == 1 else torch.sqrt(torch.clamp_min(d2, 1e-30))
    if kind == "matern12":
        return torch.exp(-r)
    if kind == "matern32":
        s = math.sqrt(3.0) * r
        return (1 + s) * torch.exp(-s)
    s = math.sqrt(5.0) * r
    return (1 + s + 5.0 / 3.0 * d2) * torch.exp(-s)


def reference(terms, xg, Gm):
    """``(term_sum [B, T], grad_xg, diag)`` by fp64 autograd, ``xg [groups, B, n, d]``, ``Gm [B, n, n]``."""
    x = xg.detach().double().requires_grad_(True)
    G = Gm.double()
    loss = (0.0 * x).sum()  # kinds like One and Delta do not depend on x: their gradient is 0
    sums = []
    for c, fs in terms:
        prod = 1.0
        for f in fs:
            prod = prod * _phi(f[0], x[f[1]], f[2] if len(f) > 2 else None)
        sums.append((G * prod).sum((1, 2)).detach())
        loss = loss + c * (G * prod).sum()
    loss.backward()
    return torch.stack(sums, 1), x.grad, torch.diagonal(G, dim1=1, dim2=2)


def run_case(terms, *, n_groups=1, n=65, d=3, batch=1, dtype=torch.float64, dup=None, seed=0):
    """Random inputs (scaled so that d2 ~ 2 at any d), a random symmetric G; ``dup``: ``"exact"`` duplicates rows,
    a float separates pairs of rows by that distance."""
    from stheno_b200 import autograd, ops

    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n_groups, batch, n, d, dtype=torch.float64, device="cuda", generator=g) / math.sqrt(d)
    if dup is not None and n >= 4:
        h = n // 2
        step = torch.randn(n_groups, batch, h - h // 2, d, dtype=torch.float64, device="cuda", generator=g)
        step = step / step.norm(dim=-1, keepdim=True) * (0.0 if dup == "exact" else float(dup))
        x[:, :, h // 2:h] = x[:, :, : h - h // 2] + step  # rows h/2 .. h-1 repeat rows 0 .. at distance `dup`
        x[:, :, -1] = x[:, :, 0]  # and a repeat in another column tile
    xg = x.to(dtype).contiguous()
    Gm = torch.randn(batch, n, n, dtype=torch.float64, device="cuda", generator=g)
    Gm = (Gm + Gm.transpose(1, 2)).to(dtype).contiguous()
    flat = ops.FlatKernel(terms, n_groups)
    term_sum, grad_xg, diag = autograd._bwd_kernel(flat, xg, Gm, n)
    ref_t, ref_x, ref_d = reference(terms, xg, Gm)
    tol = 1e-10 if dtype == torch.float64 else 1e-4
    T = len(terms)
    for name, got, want in (("term_sum", term_sum[:, :T], ref_t), ("grad_xg", grad_xg, ref_x), ("diag", diag, ref_d)):
        got = got.double()
        scale = max(want.abs().max().item(), 1e-300)
        err = (got - want).abs().max().item()
        assert torch.isfinite(got).all(), name
        assert err <= tol * scale, (name, err, scale, got.flatten()[:4].tolist(), want.flatten()[:4].tolist())


SINGLE = {
    "eq": [(1.3, [("eq", 0)])],
    "matern12": [(1.3, [("matern12", 0)])],
    "matern32": [(1.3, [("matern32", 0)])],
    "matern52": [(1.3, [("matern52", 0)])],
    "linear": [(0.7, [("linear", 0)])],
    "rq": [(1.3, [("rq", 0, 0.7)])],
    "delta": [(0.4, [("delta", 0)])],
    "one": [(0.9, [("one", 0)])],
}


@pytest.mark.parametrize("kind", list(SINGLE))
def test_each_kind(kind):
    run_case(SINGLE[kind], n=130, d=3)


PRODUCTS = {
    "eq_x_m32_same_group": ([(1.3, [("eq", 0), ("matern32", 0)])], 1),
    "linear_x_m12": ([(0.7, [("linear", 0), ("matern12", 0)])], 1),
    "four_factors_two_groups": ([(0.8, [("eq", 0), ("matern52", 1), ("rq", 0, 0.7), ("linear", 1)])], 2),
    "sum_of_terms": ([(1.0, [("eq", 0)]), (0.5, [("matern12", 1)]), (0.2, [("delta", 0)]), (0.1, [("one", 0)]),
                      (0.3, [("matern32", 1), ("matern12", 0)])], 2),
}


@pytest.mark.parametrize("name", list(PRODUCTS))
def test_products_and_groups(name):
    terms, G = PRODUCTS[name]
    run_case(terms, n_groups=G, n=100, d=3, seed=1)


@pytest.mark.parametrize("n", [1, 63, 64, 65, 300])
def test_row_counts(n):
    run_case(PRODUCTS["sum_of_terms"][0], n_groups=2, n=n, d=2, seed=n)


def test_batch():
    run_case(PRODUCTS["four_factors_two_groups"][0], n_groups=2, n=90, d=3, batch=3, seed=2)


@pytest.mark.parametrize("name", ["eq", "matern12", "matern52", "linear"])
def test_fp32(name):
    run_case(SINGLE[name], n=100, d=3, dtype=torch.float32, seed=3)


@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("dup", ["exact", 1e-12, 1e-8], ids=["exact", "1e-12", "1e-8"])
@pytest.mark.parametrize("kind", list(SINGLE))
def test_coincident_and_close_points(kind, dup, d):
    """Duplicated rows (subgradient 0 for Matern-1/2) and pairs at 1e-12 / 1e-8, where Matern-1/2's d phi / d(d2)
    grows like 1/r and must not cancel catastrophically against the rest of the row."""
    run_case(SINGLE[kind], n=200, d=d, dup=dup, seed=4)


@pytest.mark.parametrize("d", [1, 3, 8, 21, 22, 32, 64, 132])
def test_widths(d):
    """Up to d = 22 one launch holds all partial sums; from 23 on (one group) the launch runs in chunks of dimensions."""
    run_case([(1.0, [("eq", 0)]), (0.5, [("matern12", 0)])], n=70, d=d, seed=d)


def test_widths_two_groups():
    """Two groups: d = 11 is the widest that fits one launch, d = 66 (G * d = 132) runs in chunks of dimensions."""
    run_case(PRODUCTS["four_factors_two_groups"][0], n_groups=2, n=70, d=11, seed=11)
    run_case([(1.0, [("matern32", 0)]), (0.5, [("eq", 1)])], n_groups=2, n=70, d=66, seed=66)


def _exp_logpdf_ref(x, y, scale, noise):
    n, d = x.shape
    xs = x / scale
    diff = xs[:, None, :] - xs[None, :, :]
    r = diff.abs()[..., 0] if d == 1 else torch.sqrt(torch.clamp_min((diff * diff).sum(-1), 1e-30))
    K = torch.exp(-r) + (noise + 1e-12) * torch.eye(n, dtype=x.dtype, device=x.device)
    L = torch.linalg.cholesky(K)
    a = torch.linalg.solve_triangular(L, y[:, None], upper=False)
    return -0.5 * (2 * torch.log(torch.diagonal(L)).sum() + n * np.log(2 * np.pi) + (a * a).sum())


@pytest.mark.parametrize("d", [1, 3])
def test_exp_gp_logpdf_gradients_with_repeated_inputs(d):
    """``GP(Exp().stretch(l))(x, noise).logpdf(y).backward()`` on inputs with repeated values (every value twice, some
    three times), against torch autograd on a dense restatement."""
    import stheno_b200 as S

    S.B.epsilon = 1e-12
    g = torch.Generator(device="cuda").manual_seed(10 + d)
    base = torch.randn(60, d, dtype=torch.float64, device="cuda", generator=g)
    x = torch.cat([base, base, base[:10]])
    y = torch.randn(x.shape[0], dtype=torch.float64, device="cuda", generator=g)

    def params():
        return [torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True) for v in (0.7, 0.2)]

    scale, noise = params()
    xa = x.clone().requires_grad_(True)
    lp = S.GP(S.Exp().stretch(scale))(xa, noise).logpdf(y)
    lp.backward()
    got = [scale.grad.clone(), noise.grad.clone(), xa.grad.clone()]

    scale, noise = params()
    xr = x.clone().requires_grad_(True)
    ref = _exp_logpdf_ref(xr, y, scale, noise)
    ref.backward()
    want = [scale.grad, noise.grad, xr.grad]
    assert abs(lp.item() - ref.item()) < 1e-10 * abs(ref.item())
    for a, b, name in zip(got, want, ["scale", "noise", "x"]):
        err = (a - b).abs().max().item()
        assert err < 1e-8 * max(1.0, b.abs().max().item()), (name, err, a.flatten()[:3], b.flatten()[:3])
