"""Time the cost of RQ's alpha-gradient.  (1) The square K1-backward alone at n = 16384, d = 8 for RQ(0.7).stretch(1.5) with
and without param_sum, and for EQ().stretch(1.5); (2) a loss + gradient step of f(x, 0.1).logpdf(y) with f = GP(RQ(alpha)
.stretch(l)), alpha requiring grad and not (l always does).  Every case is warmed up first; the with / without runs
alternate, and the median of the CUDA-event (1) or host-clock (2) times is reported.  Prints one JSON line with the card's
name and power limit, read in the same run."""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stheno_b200 as S  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def median(v):
    v = sorted(v)
    return round(v[len(v) // 2], 3)


def kernel_times(n=16384, d=8, reps=7):
    from stheno_b200 import _lib, autograd, ops

    g = torch.Generator(device="cuda").manual_seed(0)
    xg = (torch.randn(1, 1, n, d, dtype=torch.float64, device="cuda", generator=g) / 1.5).contiguous()
    G = torch.randn(1, n, n, dtype=torch.float64, device="cuda", generator=g)
    G = 0.5 * (G + G.transpose(1, 2))
    rq = ops.FlatKernel([(1.0, [("rq", 0, 0.7)])], 1)
    eq = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    cases = {
        "rq_bwd_ms": lambda: autograd._bwd_kernel(rq, xg, G, n),
        "rq_bwd_param_sum_ms": lambda: autograd._bwd_kernel(
            rq, xg, G, n, torch.zeros(1, _lib.GPK_MAX_FACTORS, dtype=xg.dtype, device=xg.device)),
        "eq_bwd_ms": lambda: autograd._bwd_kernel(eq, xg, G, n),
    }
    times = {k: [] for k in cases}
    for r in range(reps + 1):
        for name, fn in cases.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            if r:  # the first round warms up
                times[name].append(a.elapsed_time(b))
    return {k: median(v) for k, v in times.items()}


def step_times(n=16384, d=8, reps=5):
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    y = torch.sin(x.sum(-1))
    S.B.epsilon = 1e-10

    def step(alpha_grad):
        alpha = torch.tensor(0.7, dtype=torch.float64, device="cuda", requires_grad=alpha_grad)
        ell = torch.tensor(1.5, dtype=torch.float64, device="cuda", requires_grad=True)
        lp = S.GP(S.RQ(alpha).stretch(ell))(x, 0.1).logpdf(y)
        lp.backward()

    cases = {"logpdf_step_alpha_fixed_ms": lambda: step(False), "logpdf_step_alpha_grad_ms": lambda: step(True)}
    times = {k: [] for k in cases}
    for r in range(reps + 1):
        for name, fn in cases.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if r:
                times[name].append((time.perf_counter() - t0) * 1e3)
    return {k: median(v) for k, v in times.items()}


def main():
    out = {"card": card(), "n": 16384, "d": 8}
    out.update(kernel_times())
    out.update(step_times())
    print(json.dumps(out))


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("time_rq_grad.py needs a CUDA device")
    main()
