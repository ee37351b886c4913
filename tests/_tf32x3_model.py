"""Host model of the 3xTF32 product of ``gemm_nt_f32_tc_kernel`` in ``stheno_b200/csrc/gemm_tc32.cu`` (test infrastructure).

The kernel splits every fp32 operand ``a`` into ``hi = trunc_tf32(a)`` (``bits & 0xFFFFE000``: sign, exponent and the top 10
mantissa bits) and ``lo = a - hi`` (one fp32 subtraction), and forms ``a b ~= hi_a hi_b + hi_a lo_b + lo_a hi_b`` on the
TF32 tensor cores, which read each operand's top 19 bits -- ``trunc_tf32`` of it.  Here:

- :func:`split` restates the split bit for bit (NumPy fp32 arithmetic is IEEE, like the device's ``-``);
- :func:`gemm_nt` forms the three partial products exactly in fp64 (11 x 11 significant bits), adds them in fp64 and rounds
  the result to fp32 once.

For inputs where at most one ``k`` contributes to an output element and that element's sum of partial products fits in
fp32's 24 bits (operands of at most 13 significant bits do), every step the hardware takes is exact, so the model gives the
kernel's output bit for bit whatever rounding the tensor core's accumulator uses.  ``ftz_products=True`` models an accumulator
that flushes subnormal results to zero instead."""
import numpy as np

MASK = np.uint32(0xFFFFE000)
U32 = 2.0**-24


def trunc_tf32(a):
    """What the TF32 datapath keeps of an fp32 value: ``bits & 0xFFFFE000`` (a NaN whose payload lies only in the low 13 bits
    becomes an infinity)."""
    a = np.asarray(a, np.float32)
    return (a.view(np.uint32) & MASK).view(np.float32)


def split(a):
    """``(hi, lo)`` of the kernel's ``tf32_low_part``: ``hi = trunc_tf32(a)``, ``lo = a - hi`` in fp32.  For every finite
    ``a`` the subtraction is exact (``hi`` and ``a`` share their exponent), so ``hi + lo == a``; for ``a = +-inf`` it is
    ``inf - inf = NaN``."""
    a = np.asarray(a, np.float32)
    hi = trunc_tf32(a)
    with np.errstate(invalid="ignore"):
        lo = (a - hi).astype(np.float32)
    return hi, lo


def partial_products(A, B):
    """The three ``[M, N, K]`` fp64 partial products ``hi_a hi_b``, ``hi_a lo_b``, ``lo_a hi_b`` of ``A [M, K]``, ``B [N, K]``
    as the tensor core reads them (``lo`` truncated to TF32 again).  Each is exact in fp64."""
    ha, la = split(A)
    hb, lb = split(B)
    ha, la, hb, lb = (trunc_tf32(t).astype(np.float64) for t in (ha, la, hb, lb))
    with np.errstate(invalid="ignore", over="ignore"):
        return (ha[:, None, :] * hb[None, :, :], ha[:, None, :] * lb[None, :, :], la[:, None, :] * hb[None, :, :])


def gemm_nt(A, B, ftz_products=False):
    """``A B^T`` as the 3xTF32 kernel forms it (``alpha = 1``, ``beta = 0``), the partial products summed in fp64 and
    rounded to fp32 once."""
    with np.errstate(invalid="ignore", over="ignore"):
        s = sum(partial_products(A, B))
        if ftz_products:
            s = np.where(np.abs(s) < 2.0**-126, 0.0, s)
        out = s.sum(-1).astype(np.float32)
    return out


def ffma_gemm_nt(A, B):
    """``A B^T`` as an fp32 FFMA loop forms it when at most one product per output element is non-zero: IEEE fp32
    (``inf * 0 = NaN``, subnormal results kept)."""
    A64 = np.asarray(A, np.float32).astype(np.float64)
    B64 = np.asarray(B, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return (A64[:, None, :] * B64[None, :, :]).sum(-1).astype(np.float32)
