"""Host model of ``fast_exp_nonpos`` in ``stheno_b200/csrc/kernel_matrix.cu`` (test infrastructure).

It restates the device function operation for operation: every ``fma`` is evaluated exactly and rounded once (through
``fractions.Fraction``), ``__double2loint`` / ``__double2hiint`` / ``__hiloint2double`` are bit moves done with ``struct``,
the int32 arithmetic wraps like the device's, a NaN result carries the device's bit pattern, and the 64-entry
``2^(i/64)`` table holds the correctly rounded values (the kernel fills it with the device ``exp2``, which may be an ulp
off in some entries: ``table=`` takes another).  ``fast_exp(x, guard=False)`` is the function as it was before its range
check on ``t`` replaced the ``k >> 6 < -1022`` test."""
import math
import struct
from decimal import Decimal, localcontext
from fractions import Fraction

SHIFTER = 6755399441055744.0  # 1.5 * 2^52
INV_LN2_64 = 92.332482616893656877  # 64 / ln2
LN2_64_HI = 0.010830424696249145  # ln2 / 64, high part
LN2_64_LO = 3.623510646634843e-19  # ln2 / 64 minus the high part
POLY = (8.3333333333333332e-3, 4.1666666666666664e-2, 1.6666666666666666e-1, 0.5, 1.0, 1.0)
GUARD = -745.2  # exp(x) rounds to 0 below this


def _table():
    with localcontext() as ctx:
        ctx.prec = 40
        return [float(Decimal(2) ** (Decimal(i) / 64)) for i in range(64)]


TABLE = _table()


#: the GPU's canonical NaN: a floating-point operation that returns NaN returns this bit pattern (low word = -1)
DEVICE_NAN = struct.unpack("<d", struct.pack("<Q", 0x7FFFFFFFFFFFFFFF))[0]


def _dev(v):
    return DEVICE_NAN if v != v else v


def fma(a, b, c):
    """``a * b + c`` with one rounding."""
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        return _dev(a * b + c)  # inf / nan propagate as in the fused operation
    v = Fraction(a) * Fraction(b) + Fraction(c)
    try:
        return float(v)
    except OverflowError:
        return math.inf if v > 0 else -math.inf


def _words(v):
    lo, hi = struct.unpack("<ii", struct.pack("<d", v))
    return lo, hi


def _from_words(hi, lo):
    return struct.unpack("<d", struct.pack("<ii", lo, hi))[0]


def _i32(v):
    return (v + 2**31) % 2**32 - 2**31


def table_index(x):
    """The table entry ``fast_exp(x)`` reads (``k & 63``)."""
    return _words(fma(float(x), INV_LN2_64, SHIFTER))[0] & 63


def fast_exp(x, guard=True, table=TABLE):
    x = float(x)
    t = fma(x, INV_LN2_64, SHIFTER)
    k = _words(t)[0]
    kd = _dev(t - SHIFTER)
    r = fma(kd, -LN2_64_HI, x)
    r = fma(kd, -LN2_64_LO, r)
    p = fma(r, POLY[0], POLY[1])
    for c in POLY[2:]:
        p = fma(p, r, c)
    v = _dev(p * table[k & 63])
    e = k >> 6
    if guard:  # k in [-65408, 0] and t's high word that of 1.5 * 2^52 + k; otherwise 0, or NaN for a NaN
        ht = _words(t)[1]
        if _i32(k + 65408) & 0xFFFFFFFF > 65408 or ht - (k >> 31) != 0x43380000:
            return t if (ht & 0x7FFFFFFF) > 0x7FF00000 else 0.0
    elif e < -1022:  # the check the unguarded function made instead (wrong once k has wrapped)
        return 0.0
    lo, hi = _words(v)
    return _from_words(_i32(hi + _i32(e * 1048576)), lo)


def exact_exp(x):
    """``exp(x)`` correctly rounded to float64 (40 significant digits, then one rounding; 0 below the denormals)."""
    with localcontext() as ctx:
        ctx.prec = 40
        return float(Decimal(x).exp())
