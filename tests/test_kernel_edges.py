"""K1 (``csrc/kernel_matrix.cu``) at the edges of its input range and of its launch layouts.

* CPU: the host model of the fast fp64 ``exp`` (``tests/_fexp_model.py``) against a correctly rounded ``exp``.
* GPU: every path that evaluates EQ / Matern-1/2 / 3/2 / 5/2 -- the fast strip kernel, the generic descriptor kernel,
  ``kernel_diag``, fp32 -- at distances from 0 to 1e9 and on NaN / inf inputs, against the closed form evaluated in fp64
  on direct differences with the ``exp`` taken in 40-digit decimal; and the launch layouts (strips, ragged tiles, bulk-copy and
  plain-load staging, LOWER, padding, strided / offset outputs, misaligned inputs, batches, groups, widths) against
  NumPy, with a sentinel checking that nothing outside the written window is touched."""
import math
from decimal import Decimal, localcontext

import numpy as np
import pytest
import torch

from tests._fexp_model import GUARD, TABLE, exact_exp, fast_exp, table_index

KINDS = ["eq", "matern12", "matern32", "matern52"]
DISTANCES = [0.0, 1e-8, 1.0, 37.0, 38.6, 700.0, 746.0, 6819.0, 6821.0, 7000.0, 9000.0, 16383.0, 2e4, 1e5, 1e7, 2.4e7, 1e9]
TINY64 = 2.2250738585072014e-308
SQRT3, SQRT5, FIVE_THIRDS = 1.7320508075688772, 2.23606797749979, 1.6666666666666667  # the kernels' constants

# ---------------------------------------------------------------------------------------------------------------------
# CPU: host model of fast_exp_nonpos
# ---------------------------------------------------------------------------------------------------------------------


def _ulps(got, want):
    return abs(got - want) / math.ulp(want)


def _table_boundaries():
    step = math.log(2) / 64
    pts = []
    for j in range(0, int(745.2 / step) + 1, 7):
        c = -j * step
        pts += [c, math.nextafter(c, -math.inf), math.nextafter(c, math.inf)]
    return [p for p in pts if p <= 0.0 and p > GUARD]


def test_fast_exp_model_matches_correctly_rounded_exp():
    xs = list(np.linspace(GUARD, 0.0, 12001)) + _table_boundaries() + [-708.3964185322641, -708.39641853226, -0.0]
    worst = 0.0
    for x in xs:
        x = float(x)
        got, want = fast_exp(x), exact_exp(x)
        if want >= TINY64:
            worst = max(worst, _ulps(got, want))
            assert _ulps(got, want) <= 2.0, (x, got, want)
        else:  # below the normal range the fast path flushes towards 0 (the library returns a denormal)
            assert 0.0 <= got <= 2.3e-308, (x, got, want)
    assert worst > 0.5  # the sweep reaches the inexact cases


@pytest.mark.parametrize("x", [-746.0, -1e3, -2.3e7, -2.4e7, -1e9, -1e15, -1e300, -math.inf])
def test_fast_exp_far_arguments_give_zero(x):
    assert fast_exp(x) == 0.0 and math.copysign(1.0, fast_exp(x)) == 1.0


def test_fast_exp_nan_stays_nan():
    assert math.isnan(fast_exp(math.nan))


@pytest.mark.parametrize("D,wrapped", [(6821, -4.1e-262), (7000, -2.9e121), (9000, 3.6e87), (16383, -5.1e48),
                                       (1e6, -2.1e20)])
def test_unguarded_fast_exp_wraps(D, wrapped):
    """Without its range guard the exponent arithmetic wraps once k leaves int32: EQ at these scaled distances came out
    huge or negative instead of 0.  The guarded model (the kernel's) gives 0."""
    x = -0.5 * D * D
    assert fast_exp(x, guard=False) == pytest.approx(wrapped, rel=0.03)
    assert fast_exp(x) == 0.0
    assert math.isfinite(fast_exp(math.nan, guard=False))  # and a NaN came out as a number
    assert math.isnan(fast_exp(-math.inf, guard=False))


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------


def _exp_arg_and_prefactor(kind, d2, dtype):
    """The ``exp`` argument and the polynomial prefactor, formed in ``dtype`` from ``d2`` as the kernels form them
    (d = 1: ``r = sqrt(d2)``)."""
    t = np.float64 if dtype == torch.float64 else np.float32
    d2 = t(d2)
    if kind == "eq":
        return t(-0.5) * d2, t(1.0)
    r = np.sqrt(d2)
    if kind == "matern12":
        return -r, t(1.0)
    if kind == "matern32":
        s = t(SQRT3) * r
        return -s, t(1.0) + s
    s = t(SQRT5) * r
    return -s, t(1.0) + s + t(FIVE_THIRDS) * d2


def _ref_value(kind, D, dtype):
    """``phi(|0 - D|)`` with the exp evaluated in 40-digit decimal, and the absolute floor of the normal range."""
    t = np.float64 if dtype == torch.float64 else np.float32
    D = t(D)
    arg, pre = _exp_arg_and_prefactor(kind, D * D, dtype)
    with localcontext() as ctx:
        ctx.prec = 40
        v = float(Decimal(float(pre)) * Decimal(float(arg)).exp()) if math.isfinite(arg) else 0.0
    return v


def _phi_np(kind, d2, d):
    d2 = np.asarray(d2, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.sqrt(d2) if d == 1 else np.sqrt(np.maximum(d2, 1e-30))
        if kind == "eq":
            return np.exp(-0.5 * d2)
        if kind == "matern12":
            return np.exp(-r)
        if kind == "matern32":
            return (1 + SQRT3 * r) * np.exp(-SQRT3 * r)
        return (1 + SQRT5 * r + FIVE_THIRDS * d2) * np.exp(-SQRT5 * r)


def _d2_np(x, y):
    """Direct-difference squared distances ``[n, n2]`` of ``x [n, d]``, ``y [n2, d]``."""
    d2 = np.zeros((x.shape[0], y.shape[0]))
    with np.errstate(invalid="ignore"):
        for k in range(x.shape[1]):
            d2 += (x[:, k, None] - y[None, :, k]) ** 2
    return d2


# ---------------------------------------------------------------------------------------------------------------------
# GPU: values at the edges of the range, every path
# ---------------------------------------------------------------------------------------------------------------------


def _flat(ops, kind, path, group=0, n_groups=1):
    fs = [(kind, group)] if path != "generic" else [(kind, group), ("one", group)]
    return ops.FlatKernel([(1.0, fs)], n_groups)


def _eval_path(ops, kind, x, y, path, dtype):
    """``phi(x_i, y_j)`` ``[n, n2]`` (paths ``fast`` / ``generic``) or ``phi(x_i, y_i)`` ``[n]`` (``diag``) for 1-D ``x``, ``y``."""
    xg = torch.as_tensor(np.asarray(x, np.float64)[None, None, :, None], dtype=dtype, device="cuda")
    yg = torch.as_tensor(np.asarray(y, np.float64)[None, None, :, None], dtype=dtype, device="cuda")
    if path == "diag":
        return ops.kernel_diag(_flat(ops, kind, "fast"), xg, yg, same=False)[0].double().cpu().numpy()
    return ops.kernel_matrix(_flat(ops, kind, path), xg, yg, same=False)[0].double().cpu().numpy()


def check_values(ops, kind, path, dtype):
    D = np.array(DISTANCES)
    got = _eval_path(ops, kind, np.zeros(len(D)) if path == "diag" else [0.0], D, path, dtype)
    got = got.reshape(-1)
    for Dv, g in zip(DISTANCES, got):
        want = _ref_value(kind, Dv, dtype)
        if dtype == torch.float64:
            if want >= TINY64:
                assert _ulps(g, want) <= 4.0, (kind, path, Dv, g, want)
            else:
                assert abs(g) <= 2.3e-308, (kind, path, Dv, g, want)
        else:
            tiny32 = float(np.finfo(np.float32).tiny)
            if want >= tiny32:
                assert abs(g - want) <= 6 * float(np.spacing(np.float32(want))), (kind, path, Dv, g, want)
            else:
                assert abs(g) <= 1.2e-38, (kind, path, Dv, g, want)


NONFINITE_X = [0.0, math.nan, math.inf, -math.inf, 1.0]
NONFINITE_Y = [0.0, 2.0, math.nan, math.inf, -math.inf]


def check_nonfinite(ops, kind, path, dtype):
    x, y = np.array(NONFINITE_X), np.array(NONFINITE_Y)
    got = _eval_path(ops, kind, x, y, path, dtype)
    with np.errstate(invalid="ignore"):
        want = _phi_np(kind, (x - y) ** 2 if path == "diag" else (x[:, None] - y[None, :]) ** 2, 1)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (kind, path, got, want)
    assert np.array_equal(np.isposinf(got), np.isposinf(want)) and np.array_equal(np.isneginf(got), np.isneginf(want))
    fin = np.isfinite(want)
    np.testing.assert_allclose(got[fin], want[fin], rtol=1e-12 if dtype == torch.float64 else 1e-6, atol=0)


@pytest.fixture(scope="module")
def ops():
    from stheno_b200 import ops

    return ops


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("path", ["fast", "generic", "diag"])
@pytest.mark.parametrize("kind", KINDS)
def test_values_far_and_near(ops, kind, path, dtype):
    check_values(ops, kind, path, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("path", ["fast", "generic", "diag"])
@pytest.mark.parametrize("kind", KINDS)
def test_nan_and_inf_inputs(ops, kind, path, dtype):
    check_nonfinite(ops, kind, path, dtype)


@pytest.mark.gpu
def test_fast_exp_kernel_matches_host_model_bit_for_bit(ops):
    """The fast fp64 EQ path is ``1.0 * fast_exp_nonpos(-0.5 * fl(D * D))``: the host model must reproduce it exactly.
    The kernel fills its ``2^(j/64)`` table with the device ``exp2``; every entry must be within one ulp of the correctly
    rounded value, and one choice per entry must reproduce every point that reads it."""
    D = np.concatenate([np.linspace(0.0, 38.7, 3001), np.sqrt(2 * np.arange(0, 68800, 97) * math.log(2) / 64),
                        [38.5, 38.6, 40.0, 6819.0, 6821.0, 16383.0, 1e9]])
    got = _eval_path(ops, "eq", [0.0], D, "fast", torch.float64)[0]
    xs = [-0.5 * (v * v) for v in D]
    table = list(TABLE)
    by_entry = {}
    for i, x in enumerate(xs):
        by_entry.setdefault(table_index(x), []).append(i)
    for j, idx in by_entry.items():
        cands = [TABLE[j], math.nextafter(TABLE[j], 0.0), math.nextafter(TABLE[j], 2.0)]
        fits = [c for c in cands if all(fast_exp(xs[i], table=table[:j] + [c] + table[j + 1:]) == got[i] for i in idx)]
        assert fits, (j, [(D[i], got[i], fast_exp(xs[i])) for i in idx[:3]])
        table[j] = fits[0]
    want = np.array([fast_exp(x, table=table) for x in xs])
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (D[bad[:5]], got[bad[:5]], want[bad[:5]])


# ---------------------------------------------------------------------------------------------------------------------
# GPU: launch layouts of the strip / generic kernels
# ---------------------------------------------------------------------------------------------------------------------
SENTINEL = -12345.0


def _layout_case(ops, *, kind="eq", path="fast", dtype=torch.float64, n=129, n2=1000, d=1, batch=1, flags=0,
                 noise=0.0, nv=False, jitter=0.0, ldo_extra=0, row_off=0, col_off=0, misalign=False, group=1,
                 seed=0):
    """Launch K1 through ``ops._km_launch`` into a sentinel-filled buffer and check every element of it."""
    KM_LOWER, KM_SAME, KM_PAD_ID, KM_PAD_ZERO = ops.KM_LOWER, ops.KM_SAME, ops.KM_PAD_IDENTITY, ops.KM_PAD_ZERO
    same = bool(flags & KM_SAME)
    if same:
        n2 = n
    rng = np.random.default_rng(seed)
    n_groups = group + 1
    x = rng.standard_normal((batch, n, d)) / math.sqrt(d)
    y = x if same else rng.standard_normal((batch, n2, d)) / math.sqrt(d)

    def staged(a):
        # [n_groups, B, m, d]; unused groups hold NaN so that reading the wrong group shows.  misalign: the data starts
        # 8 bytes past a 16-byte boundary (a view one row into a larger buffer with d = 1, fp64)
        m = a.shape[1]
        big = torch.full((n_groups, batch, m + (1 if misalign else 0), d), math.nan, dtype=dtype, device="cuda")
        v = big[:, :, 1:, :] if misalign else big
        v[group] = torch.as_tensor(a, dtype=dtype, device="cuda")
        return v

    xg = staged(x)
    yg = xg if same else staged(y)
    if misalign:
        assert xg.data_ptr() % 16 == 8 and xg.is_contiguous()
    pad = flags & (KM_PAD_ID | KM_PAD_ZERO)
    rows_out = ops.round_up(n) if pad else n
    cols_out = ops.round_up(n2) if pad else n2
    ldo = cols_out + col_off + ldo_extra
    R = rows_out + row_off + 3
    buf = torch.full((batch, R, ldo), SENTINEL, dtype=dtype, device="cuda")
    out = buf[:, row_off:, col_off:]
    nvec = torch.as_tensor(rng.uniform(0.1, 0.2, (batch, n)), dtype=dtype, device="cuda") if nv else None
    fs = [(kind, group)] if path == "fast" else [(kind, group), ("one", 0)]
    flat = ops.FlatKernel([(1.3, fs)], n_groups)
    ops._km_launch(flat, xg, yg, n, n2, d, flags, noise, nvec, jitter, out, ldo, R * ldo, batch)
    got = buf.double().cpu().numpy()

    want = np.full((batch, R, ldo), SENTINEL)
    xr = xg[group].double().cpu().numpy()
    yr = yg[group].double().cpu().numpy()
    ri, ci = np.arange(rows_out)[:, None], np.arange(cols_out)[None, :]
    written = np.ones((rows_out, cols_out), bool)
    if flags & KM_LOWER:
        written = (ci // 128) <= (ri // 128)
    for b in range(batch):
        w = np.zeros((rows_out, cols_out))
        w[:n, :n2] = 1.3 * _phi_np(kind, _d2_np(xr[b], yr[b]), d)
        if same:
            idx = np.arange(n)
            w[idx, idx] += noise
            if nv:
                w[idx, idx] += nvec[b].double().cpu().numpy()
            w[idx, idx] += jitter
        if flags & KM_PAD_ID:
            for i in range(min(rows_out, cols_out)):
                if i >= n or i >= n2:
                    w[i, i] = 1.0
        blk = want[b, row_off:row_off + rows_out, col_off:col_off + cols_out]
        blk[written] = w[written]
    if dtype == torch.float64:
        np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-15)
    else:
        np.testing.assert_allclose(got, want, rtol=2e-6, atol=1e-6)
    assert np.array_equal(got == SENTINEL, want == SENTINEL)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 63, 65, 129, 700])
@pytest.mark.parametrize("n2", [513, 999, 1000, 1088, 1600])
def test_layout_strips(ops, n, n2):
    """Several 8-tile strips per row, strips of 1..8 tiles, ragged last tiles; with fp64, d = 1 the strip qualifies for
    the bulk copy when every tile's byte count is a multiple of 16 (n2 = 1000 does, 999 does not)."""
    kind = KINDS[(n + n2) % 4]
    _layout_case(ops, kind=kind, n=n, n2=n2, group=0)


LAYOUT_FLAGS = {
    "lower_same_padid": ("KM_LOWER", "KM_SAME", "KM_PAD_IDENTITY"),
    "same_padid": ("KM_SAME", "KM_PAD_IDENTITY"),
    "lower_same": ("KM_LOWER", "KM_SAME"),
    "padzero": ("KM_PAD_ZERO",),
    "lower_padzero": ("KM_LOWER", "KM_PAD_ZERO"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["fast", "generic"])
@pytest.mark.parametrize("n", [65, 129, 700])
@pytest.mark.parametrize("flags", list(LAYOUT_FLAGS))
def test_layout_flags_noise_and_offsets(ops, flags, n, path):
    """LOWER (tiles above the diagonal at 128-granularity untouched), identity / zero padding with n not a multiple of
    128, noise + noise vector + jitter on the diagonal, and an output view at a row / column offset with ldo > n2 (the way
    blocks of a larger matrix are written)."""
    f = 0
    for name in LAYOUT_FLAGS[flags]:
        f |= getattr(ops, name)
    kind = KINDS[n % 4]
    _layout_case(ops, kind=kind, path=path, n=n, n2=n + 300, flags=f, noise=0.25, nv=True, jitter=1e-3, ldo_extra=37,
                 row_off=5, col_off=3)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["fast", "generic"])
@pytest.mark.parametrize("n,n2", [(129, 1000), (700, 999), (64, 1088)])
def test_layout_misaligned_inputs(ops, path, n, n2):
    """Inputs 8- but not 16-byte aligned: the bulk-copy engine cannot take them, the plain loads must."""
    _layout_case(ops, path=path, kind="matern32", n=n, n2=n2, misalign=True, group=0, seed=n)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("path", ["fast", "generic"])
def test_layout_batch_and_group(ops, path, dtype):
    """batch = 3 and a factor on group 1 of a two-group input (group 0 is NaN): the group offset and the batch stride."""
    _layout_case(ops, path=path, dtype=dtype, kind="matern52", n=200, n2=700, batch=3, group=1,
                 flags=ops.KM_LOWER | ops.KM_SAME | ops.KM_PAD_IDENTITY, noise=0.1, nv=True, jitter=1e-6)
    _layout_case(ops, path=path, dtype=dtype, kind="eq", n=130, n2=513, batch=3, group=1)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 2, 3, 5, 8, 16, 23, 24, 47, 48])
def test_layout_widths_f64(ops, d):
    """fp64, one factor: the fast kernel needs the > 48 KB shared-memory opt-in from d = 24; d = 47 is its last width and
    d = 48 goes to the generic kernel."""
    _layout_case(ops, kind=KINDS[d % 4], n=129, n2=1000, d=d, flags=ops.KM_PAD_ZERO, group=0, seed=d)
    _layout_case(ops, kind=KINDS[(d + 1) % 4], n=200, d=d, flags=ops.KM_LOWER | ops.KM_SAME | ops.KM_PAD_IDENTITY,
                 noise=0.1, jitter=1e-3, group=0, seed=d + 1)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 3, 47, 48, 95, 96])
def test_layout_widths_f32(ops, d):
    """fp32, one factor: the opt-in starts at d = 48 and the switch to the generic kernel is at 95 / 96."""
    _layout_case(ops, dtype=torch.float32, kind=KINDS[d % 4], n=129, n2=1000, d=d, group=0, seed=d)
