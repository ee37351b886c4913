"""Time pathwise function samples (``GP.sample_function``) of an exact posterior at n = 16384, d = 8, ``EQ().stretch(2)``,
noise 0.1, F = 4096 features, num = 16 samples, fp64:

* building the sample (prior draws, ``f~(X)``, the noise draw and the two solves through the factor of ``K``; the factor
  itself is formed before and reused, as every prediction of the posterior reuses it);
* evaluating it at 2^16 and 2^20 points;
* the prior part of the 2^20-point evaluation on its own (prior mean + one ``gpk_feature_eval`` launch over every point, as
  the evaluation runs it), and the feature kernel alone at 2^20 points, timed with CUDA events;
* for comparison, one exact joint sample ``f_post(x*).sample()`` at m = 4096.

Each is warmed up once and then timed ``reps`` times; per call: ms (sorted) and the peak device memory above the level before
the call.  Prints one JSON line with the card's name and power limit read in the same run."""
import gc
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stheno_b200 as S  # noqa: E402
from stheno_b200 import kernels, ops  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def once(fn):
    """(ms, peak MiB above the pre-call level) of one call, timed with a host clock around a device synchronise."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    del out
    return ms, (torch.cuda.max_memory_allocated() - base) / 2**20


def timed(fn, reps):
    once(fn)
    runs = [once(fn) for _ in range(reps)]
    return {"ms": sorted(round(r[0], 3) for r in runs), "peak_mib": round(max(r[1] for r in runs), 1)}


def main(n=16384, d=8, features=4096, num=16, reps=3):
    S.B.epsilon = 1e-12
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    y = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    f = S.GP(S.EQ().stretch(2.0))
    out = {"n": n, "d": d, "features": features, "num": num, "card": card()}
    with torch.no_grad():
        post = f | (f(x, 0.1), y)
        post.mean.K_z.chol()  # the factor: shared by every prediction of the posterior, not timed
        state = torch.Generator(device="cuda").manual_seed(1)
        out["build"] = timed(lambda: post.sample_function(num=num, features=features, state=state), reps)
        fs = post.sample_function(num=num, features=features, state=state)
        for m in (2**16, 2**20):
            xs = torch.randn(m, d, dtype=torch.float64, device="cuda", generator=g)
            out[f"eval_{m}"] = timed(lambda: fs(xs), reps)
        out["prior_part_2^20"] = timed(lambda: fs._prior(kernels.as_input(xs)), reps)
        # the feature kernel alone, at 2^20 points: CUDA events over `reps` launches after a warm-up
        omega, b, amp, W = fs.omega, fs.b, fs.amp, fs.W
        res = torch.empty(xs.shape[0], num, dtype=torch.float64, device="cuda")
        ops.feature_eval(xs, omega, b, amp, W, out=res)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.feature_eval(xs, omega, b, amp, W, out=res)
        e1.record()
        torch.cuda.synchronize()
        out["feature_kernel_2^20_ms"] = round(e0.elapsed_time(e1) / reps, 3)
        del xs, res
        xs = torch.randn(4096, d, dtype=torch.float64, device="cuda", generator=g)
        out["exact_joint_sample_4096"] = timed(lambda: post(xs).sample(num), reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
