"""Time sparse-posterior predictions and their gradient in the test inputs at BASELINE config 4 (n = 262144, m = 4096, d = 8,
Matern52().stretch(2), noise 0.1, VFE, fp64 ``auto``), trained without grad, at n* = 4096 and 262144 test points.  Per size:
``marginals()`` without grad, and ``marginals()`` with x* requiring grad followed by the backward of ``sum(mean + var)``
(``autograd._SparsePosteriorMarginals``: four solves per chunk against the forward's two).  The two alternate in one process
after a warm-up of each; per call: host-clock ms around work that ends in a device synchronise, and the peak device memory
above the level before the call.  Prints one JSON line with the card's name and power limit read in the same run."""
import gc
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stheno_b200 as S  # noqa: E402
from stheno_b200 import kernels  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def once(fn):
    """(ms, peak MiB above the pre-call level) of one call."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    return ms, (torch.cuda.max_memory_allocated() - base) / 2**20


def main(n=262144, m=4096, d=8, sizes=(4096, 262144), reps=3):
    S.B.epsilon = 1e-12
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    y = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    z = torch.randn(m, d, dtype=torch.float64, device="cuda", generator=g)
    f = S.GP(S.Matern52().stretch(2.0))
    out = {"n": n, "m": m, "d": d, "card": card(), "sizes": {}}
    with torch.no_grad():
        post = f | S.PseudoObs(f(z), f(x, 0.1), y)
        post(z[:1]).marginals()  # the factors of K_z and A and L_z^-1 (mu - m_z): shared by both calls, not timed
    for ns in sizes:
        xs0 = torch.randn(ns, d, dtype=torch.float64, device="cuda", generator=g)

        def forward():
            with torch.no_grad():
                return post(xs0).marginals()

        def forward_backward():
            xs = xs0.clone().requires_grad_(True)
            fdd = post(xs)
            assert kernels._sparse_posterior(post.mean, post.kernel, fdd.x)
            mean, var = fdd.marginals()
            (mean + var).sum().backward()
            return xs.grad

        calls = (("marginals", forward), ("marginals_fwd_bwd", forward_backward))
        res = {name: [] for name, _ in calls}
        for _, fn in calls:
            once(fn)  # warm-up
        for _ in range(reps):
            for name, fn in calls:
                res[name].append(once(fn))
        entry = {name: {"ms": sorted(round(r[0], 2) for r in runs), "peak_mib": round(max(r[1] for r in runs), 1)}
                 for name, runs in res.items()}
        entry["ratio"] = round(min(entry["marginals_fwd_bwd"]["ms"]) / min(entry["marginals"]["ms"]), 2)
        out["sizes"][str(ns)] = entry
        del xs0
    print(json.dumps(out))


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("time_sparse_predict_grad.py needs a CUDA device")
    main()
