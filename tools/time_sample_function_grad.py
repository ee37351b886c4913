"""Time gradients of pathwise function samples in their evaluation points, with the setup of ``time_sample_function.py``
(exact posterior of ``EQ().stretch(2)``, n = 16384, d = 8, noise 0.1, F = 4096 features, num = 16 samples, fp64):

* the evaluation under grad (the points require grad) at 2^16 and 2^20 points, and its backward at the same sizes (the
  upstream gradient is a fixed random ``[m, num]`` tensor);
* ``gpk_feature_eval_bwd`` alone against ``gpk_feature_eval`` alone at 2^20 points, with CUDA events;
* the peak device memory above the level before each call.

Each is warmed up once and then timed ``reps`` times (ms, sorted).  Prints one JSON line with the card's name and power limit
read in the same run."""
import gc
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stheno_b200 as S  # noqa: E402
from stheno_b200 import ops  # noqa: E402
from tools.time_sample_function import card  # noqa: E402


def timed(setup, fn, reps):
    """``fn(setup())`` ``reps`` times after one warm-up: ms per call (host clock around a device synchronise; ``setup`` is
    outside the window) and the peak MiB above the level before ``fn``."""
    runs = []
    for _ in range(reps + 1):
        arg = setup()
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        out = fn(arg)
        torch.cuda.synchronize()
        runs.append(((time.perf_counter() - t0) * 1e3, (torch.cuda.max_memory_allocated() - base) / 2**20))
        del out, arg
    runs = runs[1:]
    return {"ms": sorted(round(r[0], 3) for r in runs), "peak_mib": round(max(r[1] for r in runs), 1)}


def events(fn, reps):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / reps, 3)


def main(n=16384, d=8, features=4096, num=16, reps=3):
    S.B.epsilon = 1e-12
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    y = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    f = S.GP(S.EQ().stretch(2.0))
    out = {"n": n, "d": d, "features": features, "num": num, "card": card()}
    with torch.no_grad():
        post = f | (f(x, 0.1), y)
        post.mean.K_z.chol()
        fs = post.sample_function(num=num, features=features, state=torch.Generator(device="cuda").manual_seed(1))
    for m in (2**16, 2**20):
        xs = torch.randn(m, d, dtype=torch.float64, device="cuda", generator=g)
        up = torch.randn(m, num, dtype=torch.float64, device="cuda", generator=g)

        def forward(_):
            return fs(xs.requires_grad_())

        def backward(v):
            return torch.autograd.grad(v, xs, up)

        out[f"eval_grad_{m}"] = timed(lambda: None, forward, reps)
        out[f"backward_{m}"] = timed(lambda: forward(None), backward, reps)
        xs = xs.detach()
    omega, b, amp, W = fs.omega, fs.b, fs.amp, fs.W
    res = torch.empty(xs.shape[0], num, dtype=torch.float64, device="cuda")
    grad = torch.empty_like(xs)
    out["feature_kernel_2^20_ms"] = events(lambda: ops.feature_eval(xs, omega, b, amp, W, out=res), reps)
    out["feature_bwd_kernel_2^20_ms"] = events(lambda: ops.feature_eval_bwd(xs, omega, b, amp, W, up, out=grad), reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
