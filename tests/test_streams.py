"""Every GPU route on caller-owned streams, on two streams at once and from two host threads, against the same call on the
default stream.

(a) Gated launches: each route runs under ``with torch.cuda.stream(s)`` on a fresh stream, the data its launches read NaN
    until a ~100 ms sleep on ``s`` ends and the real data is copied in behind it.  A launch on another stream -- or on a
    libgpk side stream that did not first wait on ``s`` -- runs during the sleep and reads NaN.  A read back to the host on
    ``s`` would wait for the sleep, so whatever a route reads on the host happens before the sleep (``prepare``): the
    observations' NaN check reads the real ``y``, and a backward route runs its forward on real data, then NaN-gates what
    its backward reads (the factors and inputs its autograd nodes hold, and the upstream gradient).  Every route asserts
    that the host enqueued all of its gated launches before the sleep ended, except two whose forward reads back on the
    host at a point the test cannot reach (``host_reads``: the Woodbury log-pdf and the multi-output joint); for those the
    test asserts that they still do, so their gate is asserted once they stop.
(b) Two problems enqueued back to back on two streams from one host thread, each against its serial result.
(c) Two host threads, each on its own stream, started together; one runs a log-pdf backward (``ops.product_slices(7)`` on
    autograd's device thread), the other exact posterior marginals.
(d) ``ops.product_slices`` belongs to the thread that enters it: the slice count another thread asks for while it is held.

Forward values must equal the default-stream results bit for bit (the factorisations, solves, products and sparse sums are
reproducible).  Gradients must agree to ``GRAD_RTOL`` of their largest entry: the K1-backward term sums and the column-split
cross backward add their partial sums with atomics, in an order that varies from run to run.  The sparse ELBO's gradients are a
small difference of terms of the ELBO's size and vary with that order more: they are held to ``OBJECTIVE_RTOL`` of the ELBO.
Measured on an H100 80GB HBM3, six default-stream runs of each sparse ELBO of ``elbo_*`` below give variance gradients (about
2e2) up to 1.9e-7 apart, 5e-13 of the ELBO (3.8e5), and length-scale gradients 6.5e-12 of their own size; the other
gradients here stay within 2.2e-14 of their largest entry.  A launch that reads unordered data gives NaN."""
import ctypes
import threading
import types

import pytest
import torch

SLEEP_MS = 100
GRAD_RTOL = 1e-12
OBJECTIVE_RTOL = 4e-12
OBS = {"vfe": "PseudoObs", "fitc": "PseudoObsFITC", "dtc": "PseudoObsDTC"}


@pytest.fixture
def S(monkeypatch):
    import stheno_b200 as s

    monkeypatch.setattr(s.B, "epsilon", 1e-12)
    monkeypatch.setattr(s.B, "precision", "auto")
    monkeypatch.setattr(s.Measure, "default", None)
    return s


@pytest.fixture(scope="module")
def sleep_cycles():
    """Clock cycles of ``torch.cuda._sleep`` that last about ``SLEEP_MS``, measured once with CUDA events."""
    torch.cuda._sleep(1000)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    torch.cuda._sleep(10**7)
    b.record()
    b.synchronize()
    return int(10**7 * SLEEP_MS / a.elapsed_time(b))


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _u(g, *shape, lo=-3.0, hi=3.0):
    return torch.rand(*shape, dtype=torch.float64, device="cuda", generator=g) * (hi - lo) + lo


def _spd(batch, n, seed):
    """``G G^T / 64 + I`` (condition number ~1e2), fp64 on the device."""
    G = torch.randn(batch, n, 64, device="cuda", dtype=torch.float64, generator=_gen(seed))
    return G @ G.transpose(1, 2) / 64 + torch.eye(n, device="cuda", dtype=torch.float64)


def _consume(out):
    """Copies of a route's results, made on the current stream."""
    return {k: v.detach().clone() for k, v in out.items()}


def _call(route):
    """A route's results, prepared and launched on the current stream."""
    launch, _ = route.prepare(*route.inputs)
    return launch()


def _run(route):
    return _consume(_call(route))


class Route:
    """``prepare(*inputs) -> (launch, held)``: ``prepare`` does what reads data back to the host; ``launch()`` enqueues the
    launches under test and returns their results; ``held``: tensors ``prepare`` made that ``launch`` reads (gated with the
    inputs).  ``real``: indices of inputs ``prepare`` reads (real data before the sleep); ``until``: ``(owner, name)`` of a
    host read inside ``launch`` the gate ends at; ``objective``: the result whose size bounds the gradients' error;
    ``host_reads``: why ``launch`` reads data back on the host at a point the test cannot reach (its gate is then not
    asserted to cover the whole route)."""

    def __init__(self, inputs, prepare, real=(), until=None, objective=None, host_reads=None):
        self.inputs, self.prepare, self.real, self.until, self.objective = inputs, prepare, set(real), until, objective
        self.host_reads = host_reads


def _launch_only(fn):
    """A route with nothing to prepare: ``fn(*inputs)`` is all launches."""
    return lambda *bufs: ((lambda: fn(*bufs)), [])


def _held(v, depth=0):
    """Tensors of ``v``, of its list / tuple items and of the attributes of the objects it holds (two levels: a spec, its
    factors)."""
    if isinstance(v, torch.Tensor):
        return [v]
    if isinstance(v, (list, tuple)):
        return [t for u in v for t in _held(u, depth)]
    if depth < 2 and hasattr(v, "__dict__") and not callable(v) and not isinstance(v, (type, types.ModuleType)):
        return [t for u in list(vars(v).values()) for t in _held(u, depth + 1)]
    return []


def _backward_state(out):
    """What the custom backward nodes of ``out``'s graph hold: their factors, saved inputs and spec tensors."""
    seen, found, stack = {}, {}, [out.grad_fn]
    while stack:
        node = stack.pop()
        if node is None or id(node) in seen:
            continue
        seen[id(node)] = node  # kept alive: a freed node wrapper's id could be reused by the next one
        for t in _held([u for u in getattr(node, "__dict__", {}).values()]):
            # a broadcast view (a scalar noise expanded to n) has no memory of its own to gate
            broadcast = any(st == 0 and sz > 1 for st, sz in zip(t.stride(), t.shape))
            if t.is_cuda and t.is_floating_point() and t.numel() and not broadcast:
                found[id(t)] = t
        stack.extend(f for f, _ in node.next_functions)
    assert found, "no custom backward node in the graph"
    return list(found.values())


def _gated(stream, route, cycles, monkeypatch):
    """``route`` on ``stream`` with the data its launches read NaN until a sleep on ``stream`` ends -> (results, whether the
    host enqueued every gated launch before the sleep ended)."""
    bufs = [t.clone() if i in route.real else torch.full_like(t, float("nan")) for i, t in enumerate(route.inputs)]
    torch.cuda.synchronize()
    slept, early = torch.cuda.Event(), []
    if route.until is not None:
        owner, name = route.until
        inner = getattr(owner, name)

        def at_host_read(*args, **kwargs):
            early.append(not slept.query())
            return inner(*args, **kwargs)

        monkeypatch.setattr(owner, name, at_host_read)
    with torch.cuda.stream(stream):
        launch, held = route.prepare(*bufs)
        keep = [t.detach().clone() for t in held]
        for t in held:  # through .data: the autograd version counters of the held tensors stay as they are
            t.data.fill_(float("nan"))
        torch.cuda._sleep(cycles)
        slept.record(stream)
        for i, (b, t) in enumerate(zip(bufs, route.inputs)):
            if i not in route.real:
                b.copy_(t)
        for t, k in zip(held, keep):
            t.data.copy_(k)
        out = launch()
        early.append(not slept.query())
        out = _consume(out)
    torch.cuda.synchronize()
    if route.until is not None:
        monkeypatch.setattr(owner, name, inner)
    return out, early[0]


def _same(got, want, what="", objective=None):
    """Forward values bit for bit; ``grad*`` to ``GRAD_RTOL`` of their largest entry, or to ``OBJECTIVE_RTOL`` of the result
    ``objective`` when that is larger."""
    assert got.keys() == want.keys()
    floor = OBJECTIVE_RTOL * want[objective].abs().max().item() if objective else 0.0
    for k, w in want.items():
        g = got[k]
        assert g.shape == w.shape and g.dtype == w.dtype, (what, k)
        if k.startswith("grad"):
            err = (g - w).abs().max().item()
            bar = max(GRAD_RTOL * w.abs().max().item(), floor)
            assert err <= bar, (what, k, err, bar)
        else:
            assert torch.equal(g, w), (what, k, (g - w).abs().max().item())


# ---- the routes -----------------------------------------------------------------------------------------------------------
# Schedules of the Cholesky driver, as in tests/test_cholesky_schedules.py: name -> (dtype, batch, n, precision, k).
SCHEDULES = {
    "native_1000": (torch.float64, 1, 1000, "fp64", 1),
    "emulated_512_2500": (torch.float64, 1, 2500, "auto", 3),
    "pairs_4700_x8": (torch.float64, 1, 4700, "int8x8", 1),
    "f32_b4_2048": (torch.float32, 4, 2048, "auto", 3),
    "tf32x3_3000": (torch.float64, 1, 3000, "tf32x3", 1),
}


def _schedule(S, monkeypatch, name):
    dtype, batch, n, prec, k = SCHEDULES[name]
    monkeypatch.setattr(S.B, "precision", prec)
    from stheno_b200 import ops

    A = _spd(batch, n, n).to(dtype)
    rhs = torch.randn(batch, k, n, device="cuda", dtype=torch.float64, generator=_gen(7)).to(dtype)

    def route(A, rhs):
        ch = ops.chol_from_dense(A, rhs_t=rhs)
        return {"W": ch.W, "logdet": ch.logdet, "info": ch.info, "logpdf": ch.logpdf()}

    return Route([A, rhs], _launch_only(route))


def _abi(S, monkeypatch):
    """``gpk_potrf_f64`` (n = 2560, pair-free 512-wide emulated schedule) and an emulated ``gpk_gemm_nt_f64``, each with its
    own scratch and the stream passed explicitly."""
    from stheno_b200 import _lib, ops

    lib = _lib.load()
    n_pad, M, N, K, slices = 2560, 1152, 1024, 1280, 8
    A = _spd(1, n_pad, 3)
    g = _gen(4)
    P, Q = torch.randn(1, M, K, device="cuda", dtype=torch.float64, generator=g), torch.randn(
        1, N, K, device="cuda", dtype=torch.float64, generator=g)

    def route(A, P, Q):
        st = torch.cuda.current_stream()
        stream = ctypes.c_void_p(st.cuda_stream)
        W = A.clone()
        logdet = torch.zeros(1, device="cuda", dtype=torch.float64)
        info = torch.zeros(1, device="cuda", dtype=torch.int32)
        ws = ops._aligned_bytes(lib.gpk_potrf_oz_ws_bytes(n_pad, 0, slices), st.device)
        rc = ops._fn("gpk_potrf", torch.float64)(ops._ptr(W), W.stride(1), W.stride(0), n_pad, 0, ops._ptr(logdet),
                                                 ops._ptr(info), 1, slices, ops._ptr(ws), ws.numel(), stream)
        _lib.check(rc, "gpk_potrf_f64")
        C = torch.empty(1, M, N, device="cuda", dtype=torch.float64)
        ws2 = ops._aligned_bytes(lib.gpk_gemm_nt_oz_ws_bytes(M, N, K, slices), st.device)
        assert ws2.numel() > 0  # the emulated product
        rc = ops._fn("gpk_gemm_nt", torch.float64)(M, N, K, 1.0, ops._ptr(P), P.stride(1), P.stride(0), ops._ptr(Q),
                                                   Q.stride(1), Q.stride(0), 0.0, ops._ptr(C), C.stride(1), C.stride(0), 0,
                                                   1, slices, ops._ptr(ws2), ws2.numel(), stream)
        _lib.check(rc, "gpk_gemm_nt_f64")
        return {"W": W, "logdet": logdet, "info": info, "C": C}

    return Route([A, P, Q], _launch_only(route))


def _ops_posterior(S, monkeypatch):
    """``chol_from_kernel`` with a fused right-hand side and ``gpk_posterior_marginals`` (n = 4096, m = 3000: emulated)."""
    from stheno_b200 import ops

    g = _gen(5)
    x, xs, y = _u(g, 1, 1, 4096, 3), _u(g, 1, 1, 3000, 3), torch.randn(1, 1, 4096, device="cuda", dtype=torch.float64, generator=g)
    flat = ops.FlatKernel([(1.3, [("eq", 0)]), (0.4, [("matern52", 0)])], 1)

    def route(x, xs, y):
        ch = ops.chol_from_kernel(flat, x, noise_scalar=0.1, rhs_t=y, full_precision=True)
        dot, sq = ops.posterior_marginals(flat, xs, x, ch, half_y=ch.rhs_half()[0, 0])
        return {"L": ch.L(), "half_y": ch.rhs_half(), "dot": dot, "sq": sq}  # K1 leaves the upper triangle of W unwritten

    return Route([x, xs, y], _launch_only(route))


def _ops_sparse(S, monkeypatch):
    """``SparseAccumulator`` over 40000 points in chunks of 16384 through 600 inducing points (FITC; emulated products)."""
    from stheno_b200 import ops

    g = _gen(6)
    n, m = 40000, 600
    x, z = _u(g, 1, 1, n, 3), _u(g, 1, 1, m, 3)
    y = torch.randn(n, device="cuda", dtype=torch.float64, generator=g)
    flat = ops.FlatKernel([(1.2, [("eq", 0)])], 1)

    def route(x, z, y):
        ch = ops.chol_from_kernel(flat, z, jitter=1e-9, full_precision=True)
        acc = ops.SparseAccumulator(flat, z, ch, "fitc", chunk=16384)
        for a in range(0, n, 16384):
            c = min(n, a + 16384) - a
            acc.add(x[:, :, a : a + c], torch.full((c,), 1.2, device="cuda", dtype=torch.float64),
                    torch.full((c,), 0.05, device="cuda", dtype=torch.float64), y[a : a + c])
        return {"A": acc.A, "prod": acc.prod, "scalars": acc.scalars}

    return Route([x, z, y], _launch_only(route))


def _gp(S, var=1.3, ell=2.0):
    return S.GP(var * S.EQ().stretch(ell) + 0.4 * S.Matern52())


def _logpdf(S, n, k=1, nan=False, seed=8):
    """A log-pdf with ``k`` fused right-hand sides.  With ``nan``, some observations are NaN: the device flag is read on
    the host once the whole log-pdf is enqueued, and the gather path that follows sizes the observed set on the host, so the
    gate ends at that read (the observed subset's log-pdf launches like any other)."""
    from stheno_b200 import random as random_mod

    g = _gen(seed)
    x = _u(g, n, 3)
    y = torch.randn(n, k, device="cuda", dtype=torch.float64, generator=g)
    if nan:
        y[:: 97] = float("nan")

    def route(x, y):
        return {"logpdf": _gp(S)(x, 0.1).logpdf(y if k > 1 else y[:, 0])}

    return Route([x, y], _launch_only(route), until=(random_mod._NanFlag, "read") if nan else None)


def _linear(S, monkeypatch):
    g = _gen(9)
    x, y = _u(g, 3000, 4), torch.randn(3000, device="cuda", dtype=torch.float64, generator=g)
    return Route([x, y], _launch_only(lambda x, y: {"logpdf": S.GP(0.7 * S.Linear())(x, 0.2).logpdf(y)}),
                 host_reads="the Woodbury log-pdf reads back inside its forward")


def _backward(out, wrt, names, forward):
    """``(launch, held)`` of a backward route: ``launch`` takes the gradient of ``out`` w.r.t. ``wrt`` through an upstream
    gradient of ones, gated like the factors and inputs the backward nodes hold; ``forward``: results of the forward."""
    g = torch.ones_like(out)

    def launch():
        gs = torch.autograd.grad(out, wrt, grad_outputs=g)
        return {**forward, **{f"grad_{name}": t for name, t in zip(names, gs)}}

    return launch, _backward_state(out) + [g]


def _logpdf_bwd(S, monkeypatch, n=2500, seed=10):
    g = _gen(seed)
    x, y = _u(g, n, 3), torch.randn(n, device="cuda", dtype=torch.float64, generator=g)

    def prepare(x, y):
        p = [torch.tensor(v, device="cuda", dtype=torch.float64, requires_grad=True) for v in (1.3, 2.0, 0.1)]
        x = x.detach().requires_grad_(True)
        lp = S.GP(p[0] * S.EQ().stretch(p[1]))(x, p[2]).logpdf(y)
        return _backward(lp, p + [x], ("var", "scale", "noise", "x"), {"logpdf": lp.detach().clone()})

    return Route([x, y], prepare, real=(0, 1))


def _posterior_inputs(n, m, seed):
    g = _gen(seed)
    return [_u(g, n, 3), torch.randn(n, device="cuda", dtype=torch.float64, generator=g), _u(g, m, 3)]


def _marginals(S, monkeypatch, n=4096, m=3000, seed=11):
    def prepare(x, y, xs):  # the observations check y for NaN on the host
        f = _gp(S)
        obs = S.Obs(f(x, 0.1), y)
        return (lambda: dict(zip(("mean", "var"), (f | obs)(xs).marginals()))), []

    return Route(_posterior_inputs(n, m, seed), prepare, real=(1,))


def _full_var(S, monkeypatch):
    from stheno_b200 import matrix as M

    def prepare(x, y, xs):
        f = _gp(S)
        obs = S.Obs(f(x, 0.1), y)

        def launch():
            p = (f | obs)(xs)
            return {"mean": p.mean, "var": M.dense(p.var)}

        return launch, []

    return Route(_posterior_inputs(4096, 1024, 12), prepare, real=(1,))


def _acq(mean, var):
    return (mean + 2 * var.sqrt()).sum()


def _posterior_bwd(S, monkeypatch):
    def prepare(x, y, xs):
        f = _gp(S)
        xs = xs.detach().requires_grad_(True)
        mean, var = (f | (f(x, 0.1), y))(xs).marginals()
        return _backward(_acq(mean, var), [xs], ("xs",), {"mean": mean.detach().clone(), "var": var.detach().clone()})

    return Route(_posterior_inputs(3000, 600, 13), prepare, real=(0, 1, 2))


def _elbo_inputs():
    g = _gen(14)
    return [_u(g, 40000, 3), _u(g, 600, 3), torch.randn(40000, device="cuda", dtype=torch.float64, generator=g)]


def _elbo(method):
    """The forward (no grad) with the data and inducing points gated, after the observations read y."""
    def build(S, monkeypatch):
        def prepare(x, z, y):
            f = S.GP(1.2 * S.EQ().stretch(1.5))
            obs = getattr(S, OBS[method])(f(z), f(x, 0.05), y)
            return (lambda: {"elbo": obs.elbo(f.measure)}), []

        return Route(_elbo_inputs(), prepare, real=(2,))

    return build


def _elbo_bwd(method):
    """The backward, after a forward on real data: gradients w.r.t. variance, length scale and noise."""
    def build(S, monkeypatch):
        def prepare(x, z, y):
            p = [torch.tensor(v, device="cuda", dtype=torch.float64, requires_grad=True) for v in (1.2, 1.5, 0.05)]
            f = S.GP(p[0] * S.EQ().stretch(p[1]))
            e = getattr(S, OBS[method])(f(z), f(x, p[2]), y).elbo(f.measure)
            return _backward(e, p, ("var", "scale", "noise"), {"elbo": e.detach().clone()})

        return Route(_elbo_inputs(), prepare, real=(0, 1, 2), objective="elbo")

    return build


def _sparse_inputs():
    g = _gen(15)
    x, z, xs = _u(g, 20000, 3), _u(g, 500, 3), _u(g, 5000, 3)
    return [x, z, torch.randn(20000, device="cuda", dtype=torch.float64, generator=g), xs]


def _sparse_marginals(S, monkeypatch):
    def prepare(x, z, y, xs):
        f = _gp(S)
        obs = S.PseudoObs(f(z), f(x, 0.05), y)
        return (lambda: dict(zip(("mean", "var"), (f | obs)(xs).marginals()))), []

    return Route(_sparse_inputs(), prepare, real=(2,))


def _sparse_marginals_bwd(S, monkeypatch):
    def prepare(x, z, y, xs):
        f = _gp(S)
        xs = xs.detach().requires_grad_(True)
        mean, var = (f | S.PseudoObs(f(z), f(x, 0.05), y))(xs).marginals()
        return _backward(_acq(mean, var), [xs], ("xs",), {"mean": mean.detach().clone(), "var": var.detach().clone()})

    return Route(_sparse_inputs(), prepare, real=(0, 1, 2, 3))


def _multi_output(S, monkeypatch):
    g = _gen(16)
    n = 1100
    x, y = _u(g, n, 2), torch.randn(2 * n, device="cuda", dtype=torch.float64, generator=g)

    def route(x, y):
        meas = S.Measure()
        us = [S.GP(S.EQ().stretch(ell), measure=meas) for ell in (1.0, 2.0)]
        fs = [0.8 * us[0] + 0.5 * us[1], -0.3 * us[0] + 1.1 * us[1]]
        return {"logpdf": meas.logpdf(*[(fs[i](x, 0.1), y[i * n : (i + 1) * n]) for i in range(2)])}

    return Route([x, y], _launch_only(route), host_reads="the joint's block assembly reads back inside its forward")


ROUTES = {
    **{f"logpdf_{name}": (lambda S, mp, name=name: _schedule(S, mp, name)) for name in SCHEDULES},
    "c_abi": _abi,
    "ops_posterior_marginals": _ops_posterior,
    "ops_sparse_accumulate": _ops_sparse,
    "logpdf_rhs3": lambda S, mp: _logpdf(S, 2500, k=3),
    "logpdf_nan": lambda S, mp: _logpdf(S, 2500, nan=True),
    "logpdf_linear": _linear,
    "logpdf_backward": _logpdf_bwd,
    "posterior_marginals": _marginals,
    "posterior_full_var": _full_var,
    "posterior_backward": _posterior_bwd,
    **{f"elbo_{m}": _elbo(m) for m in OBS},
    **{f"elbo_{m}_backward": _elbo_bwd(m) for m in OBS},
    "sparse_marginals": _sparse_marginals,
    "sparse_marginals_backward": _sparse_marginals_bwd,
    "multi_output_logpdf": _multi_output,
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ROUTES))
def test_launches_follow_the_callers_stream(S, monkeypatch, sleep_cycles, name):
    route = ROUTES[name](S, monkeypatch)
    want = _run(route)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):  # warm-up on s: its memory pool and its emulation scratch exist before the gated call
        _run(route)
    torch.cuda.synchronize()
    got, gated = _gated(s, route, sleep_cycles, monkeypatch)
    _same(got, want, name, route.objective)
    if route.host_reads is None:
        assert gated, f"{name}: the host waited for the sleep before enqueuing every gated launch"
    else:
        assert not gated, f"{name} no longer reads back on the host ({route.host_reads}): assert its gate"


# ---- (b) two streams, one host thread ----------------------------------------------------------------------------------
def _pair(S, monkeypatch, a, b, warm_b=None):
    """Problem ``a`` on one stream and ``b`` on another, enqueued back to back, against their serial default-stream results.
    ``warm_b``: a route run first on b's stream, with the emulation scratch dropped before it, so that b's stream holds the
    scratch ``warm_b`` asked for (the 64 MiB minimum) and b grows it."""
    from stheno_b200 import ops

    want_a, want_b = _run(a), _run(b)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    if warm_b is not None:
        ops.release_scratch()
        with torch.cuda.stream(s2):
            _run(warm_b)
        torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        out_a = _call(a)
    with torch.cuda.stream(s2):
        out_b = _call(b)
    with torch.cuda.stream(s1):
        got_a = _consume(out_a)
    with torch.cuda.stream(s2):
        got_b = _consume(out_b)
    torch.cuda.synchronize()
    _same(got_a, want_a, "a", a.objective)
    _same(got_b, want_b, "b", b.objective)


@pytest.mark.gpu
def test_two_streams_logpdf_and_posterior(S, monkeypatch):
    """An emulated log-pdf (n = 4700: the pair schedule, 7 slices) against emulated posterior marginals (n = 4096, 8 slices).
    Both factorisations come from one host thread, so their look-ahead chains share that thread's side streams; the solves,
    products and the rest overlap."""
    _pair(S, monkeypatch, _logpdf(S, 4700, seed=20), _marginals(S, monkeypatch, seed=21))


@pytest.mark.gpu
def test_two_streams_elbo_and_logpdf(S, monkeypatch):
    _pair(S, monkeypatch, _elbo_bwd("vfe")(S, monkeypatch), _logpdf(S, 4700, seed=22))


@pytest.mark.gpu
def test_two_streams_scratch_grows_in_flight(S, monkeypatch):
    """b's factorisation (n = 6400) needs more scratch than the 64 MiB its stream holds, so b's stream grows its scratch
    while a (n = 4700) is enqueued on the other stream: both results stay those of the serial calls.  (The factorisations
    come from one host thread and share its look-ahead side streams, so they overlap less than two threads' would.)"""
    from stheno_b200 import _lib, ops

    need = _lib.load().gpk_potrf_oz_ws_bytes(6400, 128, ops._oz_slices(True))
    assert need > 64 << 20 > _lib.load().gpk_potrf_oz_ws_bytes(4736, 128, ops._oz_slices(True)), need
    _pair(S, monkeypatch, _logpdf(S, 4700, seed=23), _logpdf(S, 6400, seed=24), warm_b=_logpdf(S, 2500, seed=25))


@pytest.mark.gpu
def test_release_scratch(S, monkeypatch):
    """``ops.release_scratch(s)`` drops the scratch of ``s`` alone; the next emulated call on ``s`` gets a new one and the
    same result."""
    from stheno_b200 import ops

    route = _logpdf(S, 2500, seed=50)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    out = []
    for s in (s1, s2):
        with torch.cuda.stream(s):
            out.append(_run(route))
    torch.cuda.synchronize()
    key1, key2 = [(s.device_index, s.cuda_stream) for s in (s1, s2)]
    assert key1 in ops._OZ_SCRATCH and key2 in ops._OZ_SCRATCH
    held = ops._OZ_SCRATCH[key1].numel()
    before = torch.cuda.memory_allocated()
    ops.release_scratch(s1)
    assert key1 not in ops._OZ_SCRATCH and key2 in ops._OZ_SCRATCH
    assert torch.cuda.memory_allocated() <= before - held
    with torch.cuda.stream(s1):
        again = _run(route)
    torch.cuda.synchronize()
    _same(again, out[0])
    _same(out[1], out[0])


# ---- (c) two host threads, each on its own stream ----------------------------------------------------------------------
@pytest.mark.gpu
def test_two_threads_backward_and_posterior(S, monkeypatch):
    """Thread 1: an emulated log-pdf and its backward (which enters ``product_slices(7)``); thread 2: exact posterior
    marginals under "auto".  Both against their single-threaded results."""
    work = [_logpdf_bwd(S, monkeypatch, seed=30), _marginals(S, monkeypatch, seed=31)]
    want = [_run(route) for route in work]
    torch.cuda.synchronize()
    barrier = threading.Barrier(2)
    got, errors = [None, None], []

    def run(i):
        try:
            s = torch.cuda.Stream()
            barrier.wait()
            with torch.cuda.stream(s):
                got[i] = _run(work[i])
            s.synchronize()
        except BaseException as exc:  # reported by the main thread
            errors.append(exc)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    for i in range(2):
        _same(got[i], want[i], f"thread {i + 1}", work[i].objective)


# ---- (d) product_slices belongs to one thread ----------------------------------------------------------------------------
class _HeldElsewhere:
    """``ops.product_slices(7)`` entered on another thread and held there until the block ends."""

    def __enter__(self):
        from stheno_b200 import ops

        self.entered, self.release, self.inside = threading.Event(), threading.Event(), []

        def hold():
            with ops.product_slices(7):
                self.inside.append(ops._oz_slices())
                self.entered.set()
                self.release.wait(60)

        self.thread = threading.Thread(target=hold)
        self.thread.start()
        assert self.entered.wait(60)
        return self

    def __exit__(self, *exc):
        self.release.set()
        self.thread.join()


def test_product_slices_stay_on_their_thread(monkeypatch):
    """While another thread holds ``product_slices(7)``, this thread's "auto" calls still get 8 slices (7 only for a
    well-conditioned factorisation); the holder sees 7.  Host only."""
    from stheno_b200 import B, ops

    monkeypatch.setattr(B, "precision", "auto")
    with _HeldElsewhere() as held:
        assert ops._oz_slices() == 8
        assert ops._oz_slices(True) == 7
    assert held.inside == [7]
    assert ops._oz_slices() == 8


@pytest.mark.gpu
def test_posterior_while_another_thread_holds_product_slices(S, monkeypatch):
    """An emulated posterior mean (n = 4096) computed while another thread holds ``product_slices(7)`` is bit-equal to the
    same call with no other thread."""
    route = _marginals(S, monkeypatch, seed=40)
    want = _run(route)
    with _HeldElsewhere():
        got = _run(route)
    _same(got, want)
