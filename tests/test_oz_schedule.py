"""The wgmma schedule of the int8-slice fp64 GEMM (``oz_gemm_kernel<S>`` in csrc/gemm_oz.cu).

Every wgmma of a k-block writes a whole diagonal group of accumulators (or an accumulator of its own), so ptxas can keep
all of them in flight: the SASS guard below fails if the compiler falls back to waiting for each MMA before issuing the
next.  The GPU test checks the result bit for bit against the NumPy integer model at the shape of the Cholesky's trailing
updates (K = 1024, several tiles per CTA)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest


def _cuobjdump():
    for d in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "bin", "cuobjdump")):
            return os.path.join(d, "bin", "cuobjdump")
    return shutil.which("cuobjdump")


def wgmmas_per_kblock(S):
    """wgmmas per 64-byte k-block (two K = 32 steps): A slice s issues one wgmma per diagonal group {2j, 2j + 1} with
    2j >= s, plus, for odd s, one for diagonal s (its own accumulator, or at S = 8 the group {s - 1, s} with a zero
    B slice)."""
    groups = (S + 1) // 2
    return 2 * sum((s & 1) + groups - (s + 1) // 2 for s in range(S))


def test_emulated_gemm_wgmmas_are_not_serialised():
    from stheno_b200 import _lib

    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not available")
    _lib.load()
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for m in re.finditer(r"Function : (\S*oz_gemm_kernelILi(\d)E\S*)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        kernels[int(m.group(2))] = m.group(3)
    assert sorted(kernels) == [5, 6, 7, 8]
    for S, body in kernels.items():
        # the IGMMAs between two WARPGROUP.DEPBARs: the k-blocks of the main loop, each issued in one go
        runs, n = [], 0
        for line in body.splitlines():
            if "IGMMA" in line:
                n += 1
            elif "WARPGROUP.DEPBAR" in line and n:
                runs.append(n)
                n = 0
        if n:
            runs.append(n)
        assert runs and all(r % wgmmas_per_kblock(S) == 0 for r in runs), (S, wgmmas_per_kblock(S), runs)


@pytest.mark.gpu
@pytest.mark.parametrize("slices", [5, 6, 7, 8])
def test_gemm_oz_bit_exact_at_cholesky_shape(slices):
    """K = 1024 like the far trailing updates, and 16 x 66 = 1056 tiles of 128 x 64, so every CTA works through two tiles
    (four 128 x 32 passes through the stage ring).  The model runs on a subset of the rows (each row
    of the result depends only on its own row of A), spread over all tile rows and both consumer warpgroups."""
    import torch

    from stheno_b200 import ops
    from tests._oz_model import gemm as oz_model_gemm

    rng = np.random.default_rng(100 + slices)
    M, N, K = 2048, 4224, 1024
    A = rng.standard_normal((M, K)) * np.exp(2 * rng.standard_normal((M, 1)))
    B = rng.standard_normal((N, K))
    C0 = rng.standard_normal((M, N))
    dev = lambda a: torch.as_tensor(a, device="cuda")
    got = ops.gemm_nt_oz(dev(A), dev(B), dev(C0), alpha=-1.0, beta=1.0, slices=slices).cpu().numpy()
    rows = np.unique(np.concatenate([np.arange(0, M, 128) + o for o in (0, 63, 64, 127)] + [rng.choice(M, 16, replace=False)]))
    want = oz_model_gemm(A[rows], B, C0[rows], -1.0, 1.0, slices)
    assert np.array_equal(got[rows], want), np.abs(got[rows] - want).max()
