"""Minimal stand-in for the ``lab`` namespace ``B`` that Stheno users touch: the global Cholesky jitter
``B.epsilon`` (``README.md:820-830``), ``B.dense`` and ``B.to_numpy``."""
import numpy as np
import torch

#: Diagonal jitter added before every dense Cholesky (``B.reg``).  Reference default 1e-12; the reference's
#: examples raise it to 1e-6 for float32 (``README.md:983``).
epsilon = 1e-12

#: Arithmetic of the LARGE GEMM-shaped updates of float64 problems (Cholesky trailing updates for n >= 2048, the GEMMs of
#: the triangular solves and ``gemm_nt`` with M N K >= 1.5e9; single-matrix problems).  Everything else -- kernel-matrix
#: build, leaf factorisations, panel solves, small problems, batched problems -- always runs in native fp64.
#:   "auto" (default): fp64 emulated on the int8 tensor cores (wgmma .s32.s8.s8): operands split error-free into signed
#:       7-bit slices, EXACT int32 slice products, fp64 recombination.  7 slices (49 bits, product error ~3e-14 |a||b|) for
#:       the solve and products of the log-pdf backward and for factorisations of matrices that are well conditioned by
#:       construction (known scalar noise >= 1e-3 of the kernel variance) inside a log-pdf that is not differentiated:
#:       log-pdfs agree with the native path to ~1e-13 relative -- three orders inside the 1e-10 parity bar, ~2x faster.
#:       8 slices (below) for every other factorisation (noise-free kernels on the 1e-12 jitter, posterior covariances,
#:       assembled multi-output joints, factors a gradient is read from) and every other solve and product: those can be
#:       numerically singular, where only fp64-grade products keep the pivots positive when native fp64 does.
#:   "int8x7": 7 slices everywhere the emulation applies.
#:   "int8x8": 8 slices (56 bits >= the 53 of fp64): product error ~1e-15, the same as the fp64 tensor-core kernel itself.
#:   "int8x6": 6 slices (42 bits): ~4e-12 products, log-pdfs ~4e-10 -- faster still, NOT inside the parity bar.
#:   "fp64": native fp64 tensor cores (DMMA) everywhere.
#:   "tf32x3" (opt-in, north_star "tf32/bf16 where the user opts in"): fp32 panel copy + 3xTF32 products, ~1e-6 relative.
precision = "auto"

#: ``True``: every dense Cholesky checks its LAPACK-style ``info`` right away and raises ``torch.linalg.LinAlgError`` for a
#: non-positive-definite matrix, as the reference's backend does.  That costs a host synchronisation per factorisation, so the
#: default leaves ``info`` on the device (``Chol.info`` / ``Chol.check()``): a failed factorisation then shows as NaN results.
strict = False

#: Data points per call of the streamed sparse accumulation (``PseudoObs*``): device memory is two ``sparse_chunk x m_pad``
#: buffers + O(m^2) whatever n is; the reduction length of the tensor-core accumulation is ``sparse_chunk``.
sparse_chunk = 16384

pi = np.pi
log_2_pi = float(np.log(2 * np.pi))


def dense(a):
    """Strip matrix structure: a :class:`stheno_b200.matrix.AbstractMatrix` becomes a plain tensor/array."""
    from .matrix import AbstractMatrix

    if isinstance(a, AbstractMatrix):
        return a.dense_out()
    return a


def to_numpy(a):
    a = dense(a)
    if isinstance(a, torch.Tensor):
        return a.detach().cpu().numpy()
    if isinstance(a, (tuple, list)):
        return type(a)(to_numpy(ai) for ai in a)
    return np.asarray(a)
