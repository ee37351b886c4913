"""Every schedule of the Cholesky driver (``potrf.cu``: ``potrf_driver`` / ``potrf_driver_pairs``) against an fp64
reference: the factor element by element (backward and forward error), the log-det, the fused right-hand-side rows,
bit-for-bit reproducibility and ``info`` for a batch member with a bad pivot, NaN or inf.

  schedule          dtype  batch  n            precision          reached because
  one_panel         f64    2      300          fp64               n_pad <= 512
  no_lookahead      f64    2      1000         fp64               n_pad <= 2 * 512
  dmma_lookahead    f64    2      2500         fp64               n_pad > 1024, batched (native fp64 only)
  emulated_512      f64    1      2500         auto               2048 <= n_pad < 4096
  pairs             f64    1      4096 .. 6400 auto / int8x8      n_pad >= 4096 (ragged tails at 4700, 6400)
  (the emulated rows also with GPK_NO_LOOKAHEAD: the same schedule on the caller's stream)
  f32_lookahead     f32    4      2048         -                  diag_step<float>
  tf32x3            f64    1      3000         tf32x3             fp32 panel copies, fp32-level bound

Each factorisation asserts its schedule: the number of trailing-update launches on the fp64 DMMA kernel and on the
emulation (in-situ launch profile) must equal what that schedule launches (``updates_512`` / ``updates_pairs``), which
tells one panel, no look-ahead, look-ahead, 512-wide and pairs apart; a GPK_NO_LOOKAHEAD row must launch differently from
the same factorisation without it.  tf32x3 reports ``info`` like the others: its fp32 panel copies carry a NaN / inf and
a negative pivot through to the same leaf.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# name -> (dtype, batch, n, precision, GPK_NO_LOOKAHEAD, fused right-hand sides k, unit roundoff of the products)
SCHEDULES = {
    "one_panel": (torch.float64, 2, 300, "fp64", False, 1, 2.0**-53),
    "no_lookahead": (torch.float64, 2, 1000, "fp64", False, 130, 2.0**-53),
    "dmma_lookahead": (torch.float64, 2, 2500, "fp64", False, 300, 2.0**-53),
    "emulated_512": (torch.float64, 1, 2500, "auto", False, 130, 2.0**-53),
    "emulated_512_nola": (torch.float64, 1, 2500, "auto", True, 1, 2.0**-53),
    "pairs_4096": (torch.float64, 1, 4096, "auto", False, 300, 2.0**-53),
    "pairs_4096_nola": (torch.float64, 1, 4096, "auto", True, 130, 2.0**-53),
    "pairs_4700_x8": (torch.float64, 1, 4700, "int8x8", False, 1, 2.0**-53),
    "pairs_4700_x8_nola": (torch.float64, 1, 4700, "int8x8", True, 300, 2.0**-53),
    "pairs_6400": (torch.float64, 1, 6400, "auto", False, 130, 2.0**-53),
    "pairs_6400_x8_nola": (torch.float64, 1, 6400, "int8x8", True, 1, 2.0**-53),
    "f32_lookahead": (torch.float32, 4, 2048, "fp64", False, 130, 2.0**-24),
    "tf32x3": (torch.float64, 1, 3000, "tf32x3", False, 300, 2.0**-22),
}


@pytest.fixture(scope="module")
def ops():
    from stheno_b200 import ops

    return ops


@pytest.fixture
def schedule(request, monkeypatch):
    from stheno_b200 import B

    dtype, batch, n, prec, nola, k, u = SCHEDULES[request.param]
    if nola:
        monkeypatch.setenv("GPK_NO_LOOKAHEAD", "1")
    else:
        monkeypatch.delenv("GPK_NO_LOOKAHEAD", raising=False)
    monkeypatch.setattr(B, "precision", prec)
    return request.param, dtype, batch, n, k, u


def spd(batch, n, seed):
    """Well-conditioned SPD matrices (condition number ~1e2): G G^T / 64 + I, in fp64 on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    G = torch.randn(batch, n, 64, device="cuda", dtype=torch.float64, generator=g)
    return G @ G.transpose(1, 2) / 64 + torch.eye(n, device="cuda", dtype=torch.float64)


def factor(ops, A, rhs, dtype):
    """-> (Chol, (v3 launches, emulation launches, all library launches)) of one factorisation."""
    ops.gemm_profile(True)
    try:
        torch.cuda.synchronize()
        ops.launch_count(reset=True)
        ch = ops.chol_from_dense(A.to(dtype), rhs_t=None if rhs is None else rhs.to(dtype))
        launches = (ops.gemm_profile_read(0)[2], ops.gemm_profile_read(1)[2], ops.launch_count())
    finally:
        ops.gemm_profile(False)
    return ch, launches


P = 512  # outer panel width of the driver


def _g(M, N):
    return 1 if M > 0 and N > 0 else 0  # an update with an empty operand launches nothing


def updates_512(n_pad, R, lookahead):
    """Trailing-update GEMM launches of the 512-wide schedule (potrf_driver): with look-ahead the update of each panel
    that has a successor is split into the next panel's diagonal block, the rows below it and everything to its right."""
    cnt, kb = 0, 0
    while kb + P < n_pad:
        ke = kb + P
        ke2 = min(ke + P, n_pad)
        more = ke2 < n_pad
        if lookahead and more:
            cnt += _g(ke2 - ke, ke2 - ke) + _g(R - ke2, ke2 - ke) + _g(R - ke2, n_pad - ke2)
        else:
            cnt += _g(R - ke, ke2 - ke) + (_g(R - ke2, n_pad - ke2) if more else 0)
        kb += P
    return cnt


def updates_pairs(n_pad, R):
    """Emulated-GEMM launches of the pair schedule (potrf_driver_pairs), with or without look-ahead (the same launches,
    on one stream or on three)."""
    a1, b1 = min(P, n_pad), min(2 * P, n_pad)
    cnt = _g(R - a1, b1 - a1) if b1 > a1 else 0
    kb = 0
    while kb + 2 * P < n_pad:
        ke = kb + 2 * P
        ke1, ke2 = min(ke + P, n_pad), min(ke + 2 * P, n_pad)
        W1, W2 = ke1 - ke, ke2 - ke1
        cnt += _g(W1, W1) + _g(R - ke1, W1) + _g(R - ke1, W2)
        if W2 > 0:
            cnt += _g(W2, W2) + _g(R - ke2, W2)
        cnt += _g(R - ke2, n_pad - ke2)
        kb += 2 * P
    return cnt


def check_path(name, ch, launches):
    """The schedule of the table, from the in-situ launch profile: how many trailing updates ran on the fp64 DMMA kernel
    (v3) and how many on the emulation, against the count each schedule launches."""
    n_v3, n_oz = launches[:2]
    n_pad, R = ch.n_pad, ch.W.shape[1]
    nola = name.endswith("_nola")
    if name in ("one_panel", "no_lookahead", "dmma_lookahead"):
        want = (updates_512(n_pad, R, n_pad > 2 * P), 0)
    elif name.startswith("emulated_512"):
        want = (0, updates_512(n_pad, R, not nola))
    elif name.startswith("pairs"):
        want = (0, updates_pairs(n_pad, R))
    else:  # fp32 / tf32x3: neither fp64 GEMM kernel
        want = (0, 0)
    assert (n_v3, n_oz) == want, (name, (n_v3, n_oz), want)


def test_schedule_launch_model():
    """The launch counts the table is checked against tell the schedules apart (host-side arithmetic)."""
    assert updates_512(384, 512, True) == 0  # one panel: no trailing update
    assert updates_512(1024, 1152, False) == 1
    assert updates_512(2560, 2688, True) == 10 and updates_512(2560, 2688, False) == 7
    assert updates_pairs(4096, 4480) == 18 and updates_512(4096, 4480, True) == 19


@pytest.mark.parametrize("schedule", list(SCHEDULES), indirect=True)
def test_factor_logdet_rhs_reproducible(ops, schedule, monkeypatch):
    name, dtype, batch, n, k, u = schedule
    A = spd(batch, n, n)
    g = torch.Generator(device="cuda").manual_seed(7)
    rhs = torch.randn(batch, k, n, device="cuda", dtype=torch.float64, generator=g)
    ch, launches = factor(ops, A, rhs, dtype)
    check_path(name, ch, launches)
    if name.endswith("_nola"):
        # GPK_NO_LOOKAHEAD really changes the schedule: the panels are factorised without the split chain (other
        # launches), and the 512-wide schedule does not split its trailing updates
        with monkeypatch.context() as m:
            m.delenv("GPK_NO_LOOKAHEAD")
            _, la_launches = factor(ops, A, rhs, dtype)
        assert la_launches[2] != launches[2], (la_launches, launches)
        if name.startswith("pairs"):
            assert la_launches[1] == launches[1]
    assert ch.W.shape[1] - ch.n_pad == -(-k // 128) * 128  # extra_rows
    assert not ch.info.any()
    L = ch.L().double()
    # backward error, element by element: |A - L L^T|_ij <= c n u sqrt(A_ii A_jj)
    Ar = A.to(dtype).double()
    d = Ar.diagonal(dim1=1, dim2=2).sqrt()
    back = (Ar - L @ L.transpose(1, 2)).abs() / (d[:, :, None] * d[:, None, :])
    assert back.max().item() <= 4 * n * u, back.max().item()
    # forward error against the fp64 Cholesky of the same (rounded) matrix
    Lref = torch.linalg.cholesky(Ar)
    fwd = ((L - Lref).abs().amax((1, 2)) / Lref.abs().amax((1, 2))).max().item()
    assert fwd <= 200 * n * u, fwd
    logdet = 2 * Lref.diagonal(dim1=1, dim2=2).log().sum(1)
    assert ((ch.logdet.double() - logdet).abs() / logdet.abs()).max().item() <= 40 * n * u
    # fused right-hand sides: rows (L^-1 b)^T
    want = torch.linalg.solve_triangular(Lref, rhs.to(dtype).double().transpose(1, 2), upper=False).transpose(1, 2)
    got = ch.rhs_half().double()
    assert ((got - want).abs().max() / want.abs().max()).item() <= 200 * n * u
    # reproducible: the same input factorises to the same bits (the multi-stream schedules included)
    ch2, _ = factor(ops, A, rhs, dtype)
    assert torch.equal(ch.W, ch2.W) and torch.equal(ch.logdet, ch2.logdet) and torch.equal(ch.info, ch2.info)


INFO_SCHEDULES = list(SCHEDULES)


def _spoil(A, n, case):
    """Put the defect into member 0 of A (in place).  Returns the row it is in."""
    if case == "negative_diag_late":
        p = n - 200
        A[0, p, p] = -1.0
    elif case == "negative_diag_last":
        p = n - 1
        A[0, p, p] = -1.0
    else:
        p = (7 * n) // 10
        A[0, p, 100] = A[0, 100, p] = float("nan") if case == "nan_lower" else float("inf")
    return p


@pytest.mark.parametrize("case", ["negative_diag_late", "negative_diag_last", "nan_lower", "inf_lower"])
@pytest.mark.parametrize("schedule", INFO_SCHEDULES, indirect=True)
def test_info_bad_member(ops, schedule, case, monkeypatch):
    """``info`` = the first pivot the defect reaches, the one native fp64 reports; the other batch members are unaffected."""
    from stheno_b200 import B

    name, dtype, batch, n, k, u = schedule
    A = spd(batch, n, 3 * n)
    clean, _ = factor(ops, A, None, dtype)
    p = _spoil(A, n, case)
    ch, launches = factor(ops, A, None, dtype)
    check_path(name, ch, launches)
    with monkeypatch.context() as m:  # the native fp64 pivot, on the batch-1 native path
        m.setattr(B, "precision", "fp64")
        native, _ = factor(ops, A[:1], None, torch.float64)
    assert int(native.info[0]) == p + 1
    assert int(ch.info[0]) == p + 1, (int(ch.info[0]), p + 1)
    if batch > 1:
        assert not ch.info[1:].any()
        assert torch.equal(ch.W[1:], clean.W[1:]) and torch.equal(ch.logdet[1:], clean.logdet[1:])


def test_dense_normal_with_nan_is_not_finite():
    """A dense covariance with one off-diagonal NaN: under the default precision the log-pdf must not come out finite
    where native fp64 gives NaN (n = 4096: the emulated pair schedule)."""
    import stheno_b200 as S
    from stheno_b200 import B

    n = 4096
    A = spd(1, n, 11)[0]
    A[3000, 100] = A[100, 3000] = float("nan")
    var = A.cpu().numpy()
    y = np.random.default_rng(0).standard_normal(n)
    before = B.precision
    try:
        out = {}
        for prec in ("fp64", "auto"):
            B.precision = prec
            out[prec] = float(S.Normal(var).logpdf(y))
    finally:
        B.precision = before
    assert np.isnan(out["fp64"])
    assert not np.isfinite(out["auto"]), out["auto"]
