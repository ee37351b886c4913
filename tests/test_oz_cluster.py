"""The CTA-pair layout of the int8-slice fp64 GEMM (``oz_gemm_kernel<S>`` in csrc/gemm_oz.cu), read from the SASS.

Each tile's two 128 x 32 halves run on the two CTAs of a cluster, and each CTA loads one 64-row half of the tile's A slices
and multicasts it into both, so a tile reads its A rows from L2 once.  This guard fails if a kernel's A loads stop being
multicast TMA loads, or if the kernel loses the cluster barrier after the mbarrier init or the remote arrives that
release a stage in both CTAs."""
import re
import subprocess

import pytest

from tests.test_oz_schedule import _cuobjdump


def _oz_kernels():
    from stheno_b200 import _lib

    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not available")
    _lib.load()
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    return {int(m.group(1)): m.group(2)
            for m in re.finditer(r"Function : \S*oz_gemm_kernelILi(\d)E\S*\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S)}


def test_emulated_gemm_multicasts_a_within_a_cluster():
    kernels = _oz_kernels()
    assert sorted(kernels) == [5, 6, 7, 8]
    for S, body in kernels.items():
        ops = [op for op in re.findall(r"\b(UTMALDG\S*|UCGABAR_\w+|SYNCS\.ARRIVE\S*RED\S*)", body)]
        loads = [op for op in ops if op.startswith("UTMALDG")]
        # per k-block: A (one 64-row half, multicast to both CTAs of the pair) first, then this CTA's own B rows
        assert loads and len(loads) % 2 == 0, (S, loads)
        assert all(a == "UTMALDG.3D.MULTICAST" and b == "UTMALDG.3D" for a, b in zip(loads[::2], loads[1::2])), (S, loads)
        # cluster barrier after the mbarrier init, before any multicast or remote arrive (the exit is guarded by the
        # producer waiting for the last release of every stage, not by a second cluster barrier)
        assert ops.count("UCGABAR_ARV") == 1 and ops.count("UCGABAR_WAIT") == 1, (S, ops)
        assert ops[:2] == ["UCGABAR_ARV", "UCGABAR_WAIT"], (S, ops)
        # a consumer warp releases a stage in its own CTA and in the peer (mbarrier.arrive.shared::cluster)
        assert sum(op.startswith("SYNCS.ARRIVE") for op in ops) == 2, (S, ops)
