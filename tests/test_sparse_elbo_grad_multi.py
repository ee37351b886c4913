"""Analytic gradient of the sparse ELBO when the inducing points and / or the observations span several processes
(``PseudoObs*((u1(z1), u2(z2)), (f1(x1, n1), y1), ...)`` under grad; ``autograd.sparse_elbo``, ``ops.sparse_elbo_bwd``, the
route of single-process problems too, with one block per process pair) against torch fp64 autograd through the same ELBO
written from blocks assembled with ``generic_grad.kernel_torch``, in the formula of ``generic_grad.sparse_compute_torch``.

Three models cover the three multi-output forms: ``mix4`` (inducing points on two independent latents, observations of a
mixture ``f1 + 2 f2`` and of ``f1``: zero blocks and sums of scaled kernels), ``shared2`` (one set of inducing points serving two
outputs, heteroscedastic noise) and ``rq3`` (inducing points on two latents of one observed sum, one of them an ``RQ(alpha)``
process with alpha requiring grad)."""
import gc
import math

import pytest
import torch

from stheno_b200.generic_grad import kernel_diag_torch, kernel_torch

METHODS = ["vfe", "fitc", "dtc"]
MODELS = ["mix4", "shared2", "rq3"]


@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.Measure, "default", None)
    return s


def elbo_torch(method, Kz, Kzx, kd, kn, ybar, eps):
    """The ELBO of ``generic_grad.sparse_compute_torch`` from assembled ``K_z [m, m]``, ``K_zx [m, n]``, ``diag K_x [n]``
    (None for DTC), ``kn [n]`` and ``ybar [n]``."""
    m = Kz.shape[0]
    eye = torch.eye(m, dtype=Kz.dtype, device=Kz.device)
    L = torch.linalg.cholesky(Kz + eps * eye)
    W = torch.linalg.solve_triangular(L, Kzx, upper=False)
    trace_part = 0.0
    if method in ("vfe", "fitc"):
        corr = kd - (W * W).sum(0)
        if method == "vfe":
            trace_part = (corr / kn).sum()
        else:
            kn = kn + corr
    Ws = W / kn
    A = eye + Ws @ W.T
    L_A = torch.linalg.cholesky(A + eps * eye)
    t = torch.linalg.solve_triangular(L_A, (Ws @ ybar)[:, None], upper=False)
    det_part = torch.log(2 * math.pi * kn).sum() + 2 * torch.log(torch.diagonal(L_A)).sum()
    iqf_part = (ybar ** 2 / kn).sum() - (t * t).sum()
    return -0.5 * (det_part + iqf_part + trace_part)


class Problem:
    """One multi-output sparse problem over leaf tensors ``params`` that all require grad: :meth:`elbo` is the library's,
    :meth:`ref` the torch fp64 reference; both build fresh models."""

    def __init__(self, S, model, method, sizes_z, sizes_x, d, dtype=torch.float64, seed=0):
        self.S, self.model, self.method, self.d, self.dtype = S, model, method, d, dtype
        g = torch.Generator().manual_seed(seed)
        self.params = []
        self.g = g
        self.z = [self.leaf(torch.randn(m, d, dtype=torch.float64, generator=g) / math.sqrt(d)) for m in sizes_z]
        self.x = [self.leaf(torch.randn(n, d, dtype=torch.float64, generator=g) / math.sqrt(d)) for n in sizes_x]
        self.y = [self.leaf(torch.sin(3 * x.detach().cpu().double().sum(-1)) + 0.3 * torch.randn(x.shape[0], dtype=torch.float64,
                                                                                                  generator=g)) for x in self.x]
        self.b = self.T(0.3)
        T = self.T
        if model == "mix4":  # u = (f1(z1), f2(z2)), observed: f1 + 2 f2 and f1
            self.k1 = T(1.2) * S.Matern52().stretch(T(1.5))
            self.k2 = T(0.8) * S.EQ().stretch(T(0.9))
            self.nz = [self.leaf(1e-3 + 1e-3 * torch.rand(sizes_z[0], dtype=torch.float64, generator=g)), T(2e-3)]
            self.noise = [self.leaf(0.05 + 0.1 * torch.rand(sizes_x[0], dtype=torch.float64, generator=g)), T(0.15)]
        elif model == "shared2":  # u = f(z), observed: f and f + e, heteroscedastic noise
            self.k1 = T(1.1) * S.Matern32().stretch(T(1.3)) + T(0.2) * S.EQ()
            self.k2 = T(0.5) * S.Matern12().stretch(T(0.7))
            self.nz = [self.leaf(1e-3 + 1e-3 * torch.rand(sizes_z[0], dtype=torch.float64, generator=g))]
            self.noise = [self.leaf(0.05 + 0.1 * torch.rand(n, dtype=torch.float64, generator=g)) for n in sizes_x]
        elif model == "rq3":  # u = (f1(z1), f2(z2)), observed: f1 + f2, f2 of kernel RQ(alpha)
            self.k1 = T(1.0) * S.EQ().stretch(T(1.2))
            self.k2 = T(0.7) * S.RQ(T(1.5)).stretch(T(0.8))
            self.nz = [None, self.leaf(1e-3 + 1e-3 * torch.rand(sizes_z[1], dtype=torch.float64, generator=g))]
            self.noise = [self.leaf(0.05 + 0.1 * torch.rand(sizes_x[0], dtype=torch.float64, generator=g))]
        else:
            raise ValueError(model)

    def T(self, v):
        t = torch.tensor(v, dtype=self.dtype, device="cuda", requires_grad=True)
        self.params.append(t)
        return t

    def leaf(self, t):
        t = t.to(device="cuda", dtype=self.dtype).requires_grad_()
        self.params.append(t)
        return t

    def processes(self):
        """``(us, fs)``: the inducing and the observed processes of a fresh model."""
        S, b = self.S, self.b
        f1 = S.GP(lambda t: b * t.sum(-1), self.k1)
        f2 = S.GP(self.k2, measure=f1.measure)
        if self.model == "mix4":
            return [f1, f2], [f1 + f2 * 2.0, f1]
        if self.model == "shared2":
            return [f1], [f1, f1 + f2]
        return [f1, f2], [f1 + f2]

    def elbo(self):
        S = self.S
        us, fs = self.processes()
        cls = {"vfe": S.PseudoObs, "fitc": S.PseudoObsFITC, "dtc": S.PseudoObsDTC}[self.method]
        u = tuple(p(z, nz) for p, z, nz in zip(us, self.z, self.nz))
        obs = [(p(x, n), y) for p, x, n, y in zip(fs, self.x, self.noise, self.y)]
        obj = cls(u if len(u) > 1 else u[0], *obs) if len(obs) > 1 else cls(u, obs[0][0], obs[0][1])
        return obj.elbo(us[0].measure)

    def blocks(self):
        """``(K_z, K_zx, diag K_x, kn, ybar)`` assembled in torch with graphs to ``params``."""
        us, fs = self.processes()
        K = us[0].measure.kernels
        Kz = torch.cat([torch.cat([kernel_torch(K[a, b], za, zb) for b, zb in zip(us, self.z)], 1)
                        for a, za in zip(us, self.z)], 0)
        nz = torch.cat([torch.zeros(z.shape[0], dtype=z.dtype, device=z.device) if v is None else v.expand(z.shape[0])
                        for z, v in zip(self.z, self.nz)])
        Kz = Kz + torch.diag(nz)
        Kzx = torch.cat([torch.cat([kernel_torch(K[a, f], za, x) for f, x in zip(fs, self.x)], 1)
                         for a, za in zip(us, self.z)], 0)
        kd = torch.cat([kernel_diag_torch(K[f], x) for f, x in zip(fs, self.x)])
        kn = torch.cat([n.expand(x.shape[0]) for n, x in zip(self.noise, self.x)])
        ybar = torch.cat([y - self.b * x.sum(-1) for y, x in zip(self.y, self.x)])  # every f_p has f1's mean
        return Kz, Kzx, kd, kn, ybar

    def ref(self):
        Kz, Kzx, kd, kn, ybar = self.blocks()
        return elbo_torch(self.method, Kz, Kzx, kd, kn, ybar, self.S.B.epsilon)


def _grad(e, params):
    gs = torch.autograd.grad(e, params, allow_unused=True)
    return [torch.zeros_like(p) if g_ is None else g_ for p, g_ in zip(params, gs)]


def _errors(got, want):
    return [float((a - w).abs().max()) / max(1.0, float(w.abs().max())) for a, w in zip(got, want)]


def _check(pb, bar=1e-8):
    ref = pb.ref()
    want = _grad(ref, pb.params)
    e = pb.elbo()
    assert e.requires_grad
    got = _grad(e, pb.params)
    assert abs(float(e) - float(ref)) <= 1e-10 * max(1.0, abs(float(ref))), (float(e), float(ref))
    errs = _errors(got, want)
    print(f"\n{pb.model} {pb.method}: max gradient error {max(errs):.2e}")
    assert max(errs) <= bar, errs
    return errs


SMALL = {"mix4": ((13, 9), (200, 150)), "shared2": ((17,), (180, 130)), "rq3": ((11, 14), (260,))}


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("method", METHODS)
def test_gradients_match_reference(S, monkeypatch, method, model, precision):
    """Every coefficient, length scale, RQ's alpha, x_p, z_q, noise, y and the mean parameter; chunks of 96 points, ragged
    inside each process and at the boundary between processes."""
    monkeypatch.setattr(S.B, "precision", precision)
    monkeypatch.setattr(S.B, "sparse_chunk", 96)
    sz, sx = SMALL[model]
    _check(Problem(S, model, method, sz, sx, 2, seed=len(model)))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "int8x8", "fp64"])
@pytest.mark.parametrize("method", METHODS)
def test_gradients_emulated_shape(S, monkeypatch, method, precision):
    """m = 600 + 500 (m_pad 1152) and n = 12000 + 9000 at chunk 8192: under "auto" / "int8x8" the factor of K_z, the solves and
    the GEMMs run on the int8-slice emulation."""
    monkeypatch.setattr(S.B, "precision", precision)
    monkeypatch.setattr(S.B, "sparse_chunk", 8192)
    _check(Problem(S, "mix4", method, (600, 500), (12000, 9000), 2, seed=3))


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("method", METHODS)
def test_value_under_grad_equals_no_grad(S, monkeypatch, method, model):
    """The ELBO under grad is the no-grad ELBO bit for bit (every K_z here is factored with 8 slices either way)."""
    monkeypatch.setattr(S.B, "sparse_chunk", 96)
    sz, sx = SMALL[model]
    pb = Problem(S, model, method, sz, sx, 3, seed=7)
    e = pb.elbo()
    with torch.no_grad():
        e0 = pb.elbo()
    assert e.requires_grad and not e0.requires_grad
    assert torch.equal(e.detach(), e0), (float(e), float(e0))


#: fp32 bar as in tests/test_sparse_elbo_grad.py: err <= C32 2^-24 kappa max(1, max |want|), kappa the condition number of
#: K_z + eps I (eps = 1e-6)
C32 = 16.0


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_fp32_gradients(S, monkeypatch, method):
    monkeypatch.setattr(S.B, "epsilon", 1e-6)
    monkeypatch.setattr(S.B, "sparse_chunk", 300)
    sz, sx = (30, 25), (500, 400)
    p32 = Problem(S, "mix4", method, sz, sx, 3, dtype=torch.float32, seed=9)
    p64 = Problem(S, "mix4", method, sz, sx, 3, dtype=torch.float64, seed=9)
    with torch.no_grad():  # the reference sees the fp32-rounded inputs and parameters
        for a, b in zip(p64.params, p32.params):
            a.copy_(b.double())
    e = p32.elbo()
    got = torch.autograd.grad(e, p32.params)
    assert e.dtype == torch.float32 and all(g_.dtype == torch.float32 for g_ in got)
    ref = p64.ref()
    want = torch.autograd.grad(ref, p64.params)
    with torch.no_grad():
        Kz = p64.blocks()[0]
        ev = torch.linalg.eigvalsh(Kz + 1e-6 * torch.eye(Kz.shape[0], dtype=Kz.dtype, device=Kz.device))
        kappa = float(ev[-1] / ev[0])
    u = 2.0 ** -24
    errs = _errors([g_.double() for g_ in got], want)
    print(f"\n{method}: kappa {kappa:.3e} " + " ".join(f"{r / (u * kappa):.2e}" for r in errs))
    assert max(errs) <= C32 * u * kappa, (kappa, errs)
    assert abs(float(e) - float(ref)) <= 1e-4 * abs(float(ref))


@pytest.mark.gpu
def test_only_one_length_scale_requires_grad(S):
    """Nothing but one kernel's length scale requires grad: the ELBO still has its graph (the blocks' kernels are looked at,
    not only the joint one), and the one gradient matches."""
    pb = Problem(S, "mix4", "fitc", (13, 9), (200, 150), 2, seed=4)
    ell = pb.params[len(pb.z) + 2 * len(pb.x) + 2]  # after z, x, y, the mean parameter and k1's coefficient
    with torch.no_grad():
        for p in pb.params:
            p.requires_grad_(p is ell)
    ref = pb.ref()
    e = pb.elbo()
    assert e.requires_grad
    (got,) = torch.autograd.grad(e, [ell])
    (want,) = torch.autograd.grad(ref, [ell])
    assert _errors([got], [want])[0] <= 1e-8


def _four_by_four(S, cls, n_p, m_q, d, seed):
    """4 observed and 4 inducing processes: two latents, their sum and their difference; vector noises; Matern52 / EQ."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = [torch.randn(n_p, d, device="cuda", dtype=torch.float64, generator=gen) for _ in range(4)]
    z = [torch.randn(m_q, d, device="cuda", dtype=torch.float64, generator=gen) for _ in range(4)]
    y = [torch.randn(n_p, device="cuda", dtype=torch.float64, generator=gen) for _ in range(4)]

    def elbo(p, zs):
        f1 = S.GP(p[0] * S.Matern52().stretch(p[1]))
        f2 = S.GP(p[2] * S.EQ().stretch(p[3]), measure=f1.measure)
        ps = [f1, f2, f1 + f2, f1 + f2 * -0.5]
        u = tuple(q(zq, 1e-3) for q, zq in zip(ps, zs))
        return cls(u, *[(q(xq, p[4]), yq) for q, xq, yq in zip(ps, x, y)]).elbo(f1.measure)

    p0 = torch.tensor([1.0, 1.5, 0.6, 1.0, 0.1], dtype=torch.float64, device="cuda")
    return elbo, p0, z


@pytest.mark.gpu
def test_central_differences(S):
    """4 x 16384 points, 4 x 256 inducing points, d = 4: the analytic directional derivative along 3 random directions in
    (coefficients, length scales, noise, z) against central differences of the no-grad ELBO."""
    gen = torch.Generator(device="cuda").manual_seed(5)
    for cls in (S.PseudoObs, S.PseudoObsFITC, S.PseudoObsDTC):
        elbo, p0, z0 = _four_by_four(S, cls, 16384, 256, 4, seed=1)
        p = p0.clone().requires_grad_()
        zs = [z.clone().requires_grad_() for z in z0]
        e = elbo(p, zs)
        gs = torch.autograd.grad(e, [p] + zs)
        for k in range(3):
            dp = torch.randn(5, device="cuda", dtype=torch.float64, generator=gen) * p0
            dz = [torch.randn(z.shape, device="cuda", dtype=torch.float64, generator=gen) for z in z0]
            ana = float((gs[0] * dp).sum() + sum((g_ * d_).sum() for g_, d_ in zip(gs[1:], dz)))
            fds = []
            with torch.no_grad():
                for h in (1e-4, 1e-5):
                    up = elbo(p0 + h * dp, [z + h * d_ for z, d_ in zip(z0, dz)])
                    dn = elbo(p0 - h * dp, [z - h * d_ for z, d_ in zip(z0, dz)])
                    fds.append(float(up - dn) / (2 * h))
            print(f"\n{cls.method} direction {k}: analytic {ana:.12e} fd {fds[0]:.12e} {fds[1]:.12e}")
            assert min(abs(fd - ana) for fd in fds) <= 1e-6 * abs(ana), (cls.method, k, ana, fds)


@pytest.mark.gpu
def test_backward_memory_does_not_grow_with_n(S, monkeypatch):
    """The backward's device memory above what the forward holds: four chunk x m_pad buffers and a few m_pad x m_pad ones,
    whatever n is, plus a few dozen numbers per data point (the noise, ybar and diag K_x, their gradients and torch's
    temporaries for them), at 4 x 8192 and at 4 x 32768 points (4 x 256 inducing points, chunk 4096).  Forming K_zx or W for
    all points at once would take m_pad = 1024 numbers per point: 256 MiB and 1 GiB here."""
    from stheno_b200 import ops

    monkeypatch.setattr(S.B, "sparse_chunk", 4096)
    d, m_q = 4, 256
    c_pad, m_pad = 4096, ops.round_up(4 * m_q)
    extras = []
    for n_p in (8192, 32768):
        elbo, p0, z0 = _four_by_four(S, S.PseudoObs, n_p, m_q, d, seed=2)
        p = p0.clone().requires_grad_()
        zs = [z.clone().requires_grad_() for z in z0]
        torch.autograd.grad(elbo(p, zs), [p] + zs)  # warm the emulation scratch and the kernels
        e = elbo(p, zs)
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        torch.autograd.grad(e, [p] + zs)
        torch.cuda.synchronize()
        extra = torch.cuda.max_memory_allocated() - base
        n = 4 * n_p
        bound = 8 * (6 * c_pad * m_pad + 8 * m_pad * m_pad) + 8 * 32 * n
        print(f"\nn = {n}: backward peak {extra / 2**20:.0f} MiB above the forward (bound {bound / 2**20:.0f} MiB)")
        assert extra <= bound, (n, extra, bound)
        extras.append(extra)
        del e
    assert extras[1] - extras[0] <= 8 * 32 * 4 * (32768 - 8192), extras


# ---- what stays refused ------------------------------------------------------------------------------------------------------
MSG = "gradients of a sparse approximation over multi-output inputs are not implemented"


def _two_latents(S, k1, k2):
    ell = torch.tensor(1.3, dtype=torch.float64, device="cuda", requires_grad=True)
    f1 = S.GP(k1.stretch(ell))
    f2 = S.GP(k2, measure=f1.measure)
    return f1, f2


@pytest.mark.gpu
def test_dense_inducing_noise_is_refused(S):
    f1, f2 = _two_latents(S, S.EQ(), S.Matern32())
    z = torch.randn(5, 1, dtype=torch.float64, device="cuda")
    x = torch.randn(40, 1, dtype=torch.float64, device="cuda")
    y = torch.randn(40, dtype=torch.float64, device="cuda")
    dense = 1e-2 * torch.eye(5, dtype=torch.float64, device="cuda") + 1e-3
    obs = S.PseudoObs((f1(z, dense), f2(z)), (f1(x, 0.1), y), (f2(x, 0.1), y))
    with pytest.raises(NotImplementedError, match=MSG):
        obs.elbo(f1.measure)


@pytest.mark.gpu
def test_block_that_does_not_flatten_is_refused(S):
    f1, f2 = _two_latents(S, S.EQ(), S.EQ().periodic(1.0))
    z = torch.randn(5, 1, dtype=torch.float64, device="cuda")
    x = torch.randn(40, 1, dtype=torch.float64, device="cuda")
    y = torch.randn(40, dtype=torch.float64, device="cuda")
    obs = S.PseudoObs((f1(z), f2(z)), (f1(x, 0.1), y), (f2(x, 0.1), y))
    with pytest.raises(NotImplementedError, match=MSG):
        obs.elbo(f1.measure)


@pytest.mark.gpu
def test_batched_problem_is_refused(S):
    f1, f2 = _two_latents(S, S.EQ(), S.Matern52())
    z = torch.randn(3, 5, 1, dtype=torch.float64, device="cuda")
    x = torch.randn(3, 40, 1, dtype=torch.float64, device="cuda")
    y = torch.randn(3, 40, 1, dtype=torch.float64, device="cuda")
    obs = S.PseudoObs((f1(z), f2(z)), (f1(x, 0.1), y), (f2(x, 0.1), y))
    with pytest.raises(NotImplementedError, match=MSG):
        obs.elbo(f1.measure)
