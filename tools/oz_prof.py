"""CUDA-event timer of the int8-slice fp64 GEMM (``ops.gemm_nt_oz``) at the largest far trailing update of the benchmark's
n = 16384 Cholesky: C[M x N] -= A B^T, M = 14464, N = 14336, K = 1024, lower mode; and at the same M, N with K = 512 (the
depth of the updates inside a pair of panels).

    python tools/oz_prof.py [--slices 7 8] [-K 1024 512] [--iters 30] [--warmup 5]

Prints one JSON line per slice count and K: ms per call (slicing + GEMM, CUDA events over ``iters`` back-to-back calls),
ms of ``oz_gemm_kernel`` alone (torch.profiler, a separate run of the same calls), the int8 rate of the kernel (S (S + 1) / 2
slice products of the tiles computed), the operand bytes the kernel's TMA loads read from L2 per call and the resulting
L2-to-SM rate, with the GPU name, power limit and SM clock read at the end."""
import argparse
import json
import subprocess

import torch

from stheno_b200 import ops


def tiles_lower(M, N):
    tm, tn = M // 128, N // 64
    tri = min(tm, tn // 2)
    return tri * (tri + 1) + (tm - tri) * tn


def operand_bytes(tiles, K, S):
    """Bytes the TMA loads per call: for each 128 x 64 tile and 64-byte k-block, the CTA pair reads the tile's 128 A rows
    once (each CTA one 64-row half, multicast to both) and each CTA its own 32 B rows, all S slices of each."""
    return tiles * (K // 64) * S * (128 + 2 * 32) * 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slices", type=int, nargs="+", default=[7, 8])
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("-M", type=int, default=14464)
    ap.add_argument("-N", type=int, default=14336)
    ap.add_argument("-K", type=int, nargs="+", default=[1024, 512])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("oz_prof.py times the GPU kernel: no CUDA device")
    M, N = args.M, args.N
    for K in args.K:
        g = torch.Generator(device="cuda").manual_seed(0)
        A = torch.randn(M, K, device="cuda", dtype=torch.float64, generator=g)
        B = torch.randn(N, K, device="cuda", dtype=torch.float64, generator=g)
        C = torch.zeros(M, N, device="cuda", dtype=torch.float64)
        for S in args.slices:
            call = lambda: ops.gemm_nt_oz(A, B, C, alpha=-1.0, beta=1.0, lower=True, slices=S)
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            ms_call = e0.elapsed_time(e1) / args.iters
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.iters):
                    call()
                torch.cuda.synchronize()
            us = [e.device_time for e in prof.events() if "oz_gemm_kernel" in e.name]
            ms_kernel = sum(us) / len(us) / 1e3 if us else None
            tiles = tiles_lower(M, N)
            int8_ops = tiles * 128 * 64 * K * 2 * S * (S + 1) // 2
            nbytes = operand_bytes(tiles, K, S)
            smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip()
            print(json.dumps({"M": M, "N": N, "K": K, "lower": True, "slices": S, "iters": args.iters, "ms_per_call": ms_call,
                              "ms_kernel": ms_kernel, "kernel_int8_tops": ms_kernel and int8_ops / (ms_kernel * 1e-3) / 1e12,
                              "operand_bytes_per_call": nbytes, "int8_ops_per_operand_byte": int8_ops / nbytes,
                              "l2_to_sm_tb_per_s": ms_kernel and nbytes / (ms_kernel * 1e-3) / 1e12, "gpu": smi}), flush=True)
        del A, B, C


if __name__ == "__main__":
    main()
