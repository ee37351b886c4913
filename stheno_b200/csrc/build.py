"""Build libgpk.so (hand-written sm_90a CUDA kernels for the H100 + C-ABI) in-tree with nvcc.

Usage: ``python -m stheno_b200.csrc.build`` or ``build_library()`` from ``__graft_entry__.build()``.
nvcc cross-compiles without a GPU; the built ``.so`` is git-ignored."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["kernel_matrix.cu", "kernel_matrix_bwd.cu", "gemm.cu", "gemm_tc32.cu", "gemm_oz.cu", "potrf.cu", "util.cu", "sparse.cu", "posterior.cu", "sample_fn.cu", "loo.cu", "cv.cu"]
LIB = os.path.join(HERE, "libgpk.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    # a non-static function needs an earlier declaration (common.cuh, gpk.h): one whose definition drifts from it fails
    # to compile instead of leaving an undefined symbol that only loading the library reports
    "-Xcompiler", "-Werror=missing-declarations",
    "--expt-relaxed-constexpr",
]


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libgpk.so")
    return nvcc


def needs_rebuild():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(HERE, s) for s in SOURCES] + [
        os.path.join(HERE, "common.cuh"),
        os.path.join(HERE, "wgmma.cuh"),
        os.path.join(HERE, "..", "..", "include", "gpk.h"),
    ]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    if not force and not needs_rebuild():
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for s in SOURCES:
        obj = os.path.join(HERE, s.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(HERE, s), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for s, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {s}")
    tmp = LIB + ".tmp"
    cmd = [nvcc, "-shared", "-o", tmp, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.check_call(cmd)
    os.replace(tmp, LIB)  # atomic: a concurrent reader of the tree never sees a half-written library
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
