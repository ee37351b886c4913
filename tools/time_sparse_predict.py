"""Time ``marginals()`` of a sparse posterior at BASELINE config 4 (n = 262144, m = 4096, d = 8, Matern52().stretch(2), noise
0.1, VFE, fp64), trained without grad, at n* = 262144 and 2^20 test points: the streamed call (``gpk_sparse_posterior_marginals``)
against the composition it replaces (``PosteriorMean.dev`` + the ``SumKernel`` element-wise evaluation: three K1 passes and
three solves over every test point at once).  The two alternate in one process after a warm-up of each; per call: ms, and the
peak device memory above the level before the call.  A composition that runs out of device memory is recorded as such.
Prints one JSON line with the card's name and power limit read in the same run."""
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
    """(ms, peak MiB above the pre-call level) of one call, or (None, "OOM")."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    try:
        out = fn()
        torch.cuda.synchronize()
    except torch.OutOfMemoryError:
        gc.collect()
        torch.cuda.empty_cache()
        return None, "OOM"
    ms = (time.perf_counter() - t0) * 1e3
    del out
    return ms, (torch.cuda.max_memory_allocated() - base) / 2**20


def main(n=262144, m=4096, d=8, sizes=(262144, 2**20), reps=3):
    S.B.epsilon = 1e-12
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    y = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    z = torch.randn(m, d, dtype=torch.float64, device="cuda", generator=g)
    f = S.GP(S.Matern52().stretch(2.0))
    out = {"n": n, "m": m, "d": d, "card": card(), "sizes": {}}
    with torch.no_grad():
        post = f | S.PseudoObs(f(z), f(x, 0.1), y)
        post(z[:1]).marginals()  # the factors of K_z and A and L_z^-1 (mu - m_z): shared by both routes, not timed
        for ns in sizes:
            xs = torch.randn(ns, d, dtype=torch.float64, device="cuda", generator=g)
            xi = kernels.as_input(xs)  # its stretched copy is made by the first call and shared by both routes

            def streamed():
                return post(xi).marginals()

            def composition():
                return post.mean.dev(xi), kernels._elwise_any(post.kernel, xi, None, True)

            assert kernels._sparse_posterior(post.mean, post.kernel, xi)
            res = {"streamed": [], "composition": []}
            for name, fn in (("streamed", streamed), ("composition", composition)):
                once(fn)  # warm-up
            for _ in range(reps):
                for name, fn in (("streamed", streamed), ("composition", composition)):
                    res[name].append(once(fn))
            entry = {}
            for name, runs in res.items():
                ok = [r for r in runs if r[0] is not None]
                entry[name] = ({"ms": sorted(r[0] for r in ok), "peak_mib": max(r[1] for r in ok)} if len(ok) == len(runs)
                               else {"oom": True, "runs": len(runs), "oom_runs": len(runs) - len(ok)})
            out["sizes"][str(ns)] = entry
            del xs, xi
    print(json.dumps(out))


if __name__ == "__main__":
    main()
