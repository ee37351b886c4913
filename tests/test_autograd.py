"""Hyper-parameter gradients of logpdf (SURVEY 8 row a16): analytic backward on the GPU vs torch autograd through a
plain torch-fp64 restatement of the same model (exp / cholesky / triangular_solve, as the reference does it)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def torch_ref(x, y, var, scale, noise, var2=None, scale2=None, kind2=None):
    def d2(xs):
        return ((xs[:, None, :] - xs[None, :, :]) ** 2).sum(-1)

    K = var * torch.exp(-0.5 * d2(x / scale))
    if var2 is not None:
        r2 = d2(x / scale2)
        r = torch.sqrt(torch.clamp_min(r2, 1e-30))
        s = np.sqrt(5.0) * r
        K = K + var2 * (1 + s + 5.0 / 3.0 * r2) * torch.exp(-s)
    n = x.shape[0]
    K = K + (noise + 1e-12) * torch.eye(n, dtype=x.dtype, device=x.device)
    L = torch.linalg.cholesky(K)
    a = torch.linalg.solve_triangular(L, y[:, None], upper=False)
    return -0.5 * (2 * torch.log(torch.diagonal(L)).sum() + n * np.log(2 * np.pi) + (a * a).sum())


@pytest.mark.parametrize("n,d", [(50, 1), (300, 3), (700, 8)])
def test_logpdf_gradients(n, d):
    import stheno_b200 as S

    S.B.epsilon = 1e-12
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, d, device="cuda", dtype=torch.float64, generator=g)
    y = torch.randn(n, device="cuda", dtype=torch.float64, generator=g)

    def params():
        return [torch.tensor(v, device="cuda", dtype=torch.float64, requires_grad=True) for v in (1.3, 0.8, 0.15, 0.6, 1.7)]

    var, scale, noise, var2, scale2 = params()
    xg_ = x.clone().requires_grad_(True)
    yg_ = y.clone().requires_grad_(True)
    f = S.GP(var * S.EQ().stretch(scale) + var2 * S.Matern52().stretch(scale2))
    lp = f(xg_, noise).logpdf(yg_)
    assert lp.requires_grad
    lp.backward()
    got = [p.grad.clone() for p in (var, scale, noise, var2, scale2)] + [xg_.grad.clone(), yg_.grad.clone()]

    var, scale, noise, var2, scale2 = params()
    xr = x.clone().requires_grad_(True)
    yr = y.clone().requires_grad_(True)
    ref = torch_ref(xr, yr, var, scale, noise, var2, scale2)
    ref.backward()
    want = [p.grad for p in (var, scale, noise, var2, scale2)] + [xr.grad, yr.grad]
    assert abs(lp.item() - ref.item()) < 1e-10 * abs(ref.item())
    for a, b, name in zip(got, want, ["var", "scale", "noise", "var2", "scale2", "x", "y"]):
        err = (a - b).abs().max().item()
        tol = 1e-8 * max(1.0, b.abs().max().item())
        assert err < tol, (name, err, a.flatten()[:3], b.flatten()[:3])


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_kernel_functions_launch_the_callers_descriptor(dtype, monkeypatch):
    """The differentiable kernel matrix, cross-covariance, diagonal and log-pdf launch the descriptor their caller holds:
    they build no ``ops.FlatKernel`` of their own, and each value equals, bit for bit, the no-grad launch of that
    descriptor."""
    import stheno_b200 as S
    from stheno_b200 import autograd, ops
    from stheno_b200.kernels import Input

    g = torch.Generator(device="cuda").manual_seed(3)
    c = torch.tensor(1.3, device="cuda", dtype=dtype, requires_grad=True)
    ell = torch.tensor(0.7, device="cuda", dtype=dtype, requires_grad=True)
    flat, scales = (c * S.EQ()).stretch(ell)._flat()
    xg = Input(torch.randn(40, 2, device="cuda", dtype=dtype, generator=g)).scaled(scales)
    zg = Input(torch.randn(24, 2, device="cuda", dtype=dtype, generator=g)).scaled(scales)
    y = torch.randn(1, 1, 40, device="cuda", dtype=dtype, generator=g)
    noise, jitter = 0.125, 1e-9

    built = []
    init = ops.FlatKernel.__init__

    def spy(self, *args, **kwargs):
        built.append(args)
        init(self, *args, **kwargs)

    monkeypatch.setattr(ops.FlatKernel, "__init__", spy)
    got = [autograd.kernel_matrix_grad(flat, xg), autograd.kernel_cross_grad(flat, xg, zg),
           autograd.kernel_diag_grad(flat, xg)]
    assert not built
    got.append(autograd.kernel_logpdf(flat, xg, noise, None, y, jitter))
    sum(t.sum() for t in got).backward()
    assert not built
    assert c.grad is not None and ell.grad is not None

    with torch.no_grad():
        want = [ops.kernel_matrix(flat, xg), ops.kernel_matrix(flat, xg, zg, same=False), ops.kernel_diag(flat, xg),
                ops.chol_from_kernel(flat, xg, noise_scalar=noise, jitter=jitter, rhs_t=y, full_precision=True).logpdf()]
    for name, a, b in zip(("matrix", "cross", "diag", "logpdf"), got, want):
        assert torch.equal(a.detach(), b), name


def test_optimisation_loop_decreases_loss():
    # the shape of readme_example13_optimisation_torch.py:46-53 with plain torch.optim
    import stheno_b200 as S

    S.B.epsilon = 1e-10
    rng = np.random.default_rng(0)
    x = torch.linspace(0, 5, 200, dtype=torch.float64, device="cuda")
    y = torch.sin(2 * x) + 0.2 * torch.as_tensor(rng.standard_normal(200), device="cuda")
    raw = torch.zeros(3, device="cuda", dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([raw], lr=0.1)
    losses = []
    for _ in range(25):
        opt.zero_grad()
        var, scale, noise = torch.exp(raw[0]), torch.exp(raw[1]), 0.1 * torch.exp(raw[2])
        loss = -S.GP(var * S.EQ().stretch(scale))(x, noise).logpdf(y)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0] - 10


def test_multi_output_joint_gradients():
    """BASELINE config 5 in miniature: p = 3 outputs mixing m = 2 latent GPs (ILMM, readme_example4_multi-output.py),
    loss = -joint logpdf, gradients w.r.t. the mixing matrix H, the latent length scales and the noise -- through the block
    assembly of stheno/mo -- against torch autograd on a plain dense restatement."""
    import stheno_b200 as S

    S.B.epsilon = 1e-12
    torch.manual_seed(0)
    n, p, m = 60, 3, 2
    x = torch.linspace(0, 5, n, dtype=torch.float64, device="cuda")
    y = torch.randn(p * n, dtype=torch.float64, device="cuda")

    def params():
        H = torch.tensor([[1.0, 0.5], [-0.7, 1.2], [0.3, -0.9]], dtype=torch.float64, device="cuda", requires_grad=True)
        ells = torch.tensor([0.8, 1.9], dtype=torch.float64, device="cuda", requires_grad=True)
        noise = torch.tensor(0.3, dtype=torch.float64, device="cuda", requires_grad=True)
        return H, ells, noise

    H, ells, noise = params()
    meas = S.Measure()
    us = [S.GP(S.EQ().stretch(ells[j]), measure=meas) for j in range(m)]
    fs = [H[i, 0] * us[0] + H[i, 1] * us[1] for i in range(p)]
    lp = meas.logpdf(*[(fs[i](x, noise), y[i * n:(i + 1) * n]) for i in range(p)])
    assert lp.requires_grad
    (-lp).backward()
    got = [H.grad.clone(), ells.grad.clone(), noise.grad.clone()]

    H, ells, noise = params()
    d2 = (x[:, None] - x[None, :]) ** 2
    Ks = [torch.exp(-0.5 * d2 / ells[j] ** 2) for j in range(m)]
    K = torch.cat([torch.cat([sum(H[i, j] * H[k, j] * Ks[j] for j in range(m)) for k in range(p)], dim=1) for i in range(p)], dim=0)
    K = K + (noise + 1e-12) * torch.eye(p * n, dtype=torch.float64, device="cuda")
    L = torch.linalg.cholesky(K)
    a = torch.linalg.solve_triangular(L, y[:, None], upper=False)
    ref = -0.5 * (2 * torch.log(torch.diagonal(L)).sum() + p * n * np.log(2 * np.pi) + (a * a).sum())
    (-ref).backward()
    assert abs(lp.item() - ref.item()) < 1e-10 * abs(ref.item())
    for a_, b_, name in zip(got, [H.grad, ells.grad, noise.grad], ["H", "ells", "noise"]):
        err = (a_ - b_).abs().max().item()
        assert err < 1e-7 * max(1.0, b_.abs().max().item()), (name, err, a_, b_)
