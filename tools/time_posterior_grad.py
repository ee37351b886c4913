"""Time posterior marginals and their gradients at the C2 size (n = 16384, d = 8, EQ().stretch(2) + noise 0.1, m = 4096):
forward only, forward + backward with every parameter requiring grad, forward + backward with only x* requiring grad, and
torch eager fp64 autograd through cholesky / solve_triangular on the same inputs.  Prints one JSON line: ms per call, the
peak device memory of a call, and the card's name and power limit read in the same run."""
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


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3, (torch.cuda.max_memory_allocated() - base) / 2**20


def main(n=16384, m=4096, d=8, reps=5):
    S.B.epsilon = 1e-10
    g = torch.Generator(device="cuda").manual_seed(0)
    x0 = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    xs0 = torch.randn(m, d, dtype=torch.float64, device="cuda", generator=g)
    y0 = torch.sin(x0.sum(-1))
    w = torch.randn(m, dtype=torch.float64, device="cuda", generator=g)

    def ours(all_params, backward=True):
        var, scale, noise = (torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=all_params)
                             for v in (1.0, 2.0, 0.1))
        x, y = x0.clone().requires_grad_(all_params), y0.clone().requires_grad_(all_params)
        xs = xs0.clone().requires_grad_(backward)
        f = S.GP(var * S.EQ().stretch(scale))
        mu, v = (f | (f(x, noise), y))(xs).marginals()
        if backward:
            ((mu + w * v).sum()).backward()

    def eager():
        var, scale, noise = (torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True) for v in (1.0, 2.0, 0.1))
        x, y, xs = (t.clone().requires_grad_(True) for t in (x0, y0, xs0))
        kern = lambda a, b: var * torch.exp(-0.5 * torch.cdist(a / scale, b / scale) ** 2)
        L = torch.linalg.cholesky(kern(x, x) + (noise + S.B.epsilon) * torch.eye(n, dtype=x.dtype, device=x.device))
        A = torch.linalg.solve_triangular(L, kern(x, xs), upper=False)
        h = torch.linalg.solve_triangular(L, y[:, None], upper=False)
        mu, v = (A * h).sum(0), var - (A * A).sum(0)
        ((mu + w * v).sum()).backward()

    def fwd():
        with torch.no_grad():
            ours(False, backward=False)

    out = {"n": n, "m": m, "d": d, "card": card()}
    for name, fn in (("forward_ms", fwd), ("fwd_bwd_all_ms", lambda: ours(True)), ("fwd_bwd_xstar_ms", lambda: ours(False)),
                     ("torch_eager_fwd_bwd_ms", eager)):
        ms, mib = timed(fn, reps)
        out[name] = round(ms, 2)
        out[name.replace("_ms", "_peak_mib")] = round(mib, 1)
    out["backward_chunk_ms"] = chunk_split(x0, xs0, w)
    print(json.dumps(out))


def chunk_split(x0, xs0, w, reps=3):
    """CUDA-event times of the steps the backward runs per 4096-point chunk of test points (only x* requiring grad)."""
    from stheno_b200 import _lib, ops

    flat = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    xg, xsg = (t.reshape(1, 1, *t.shape) / 2.0 for t in (x0, xs0))
    ch = ops.chol_from_kernel(flat, xg.contiguous(), noise_scalar=0.1, jitter=S.B.epsilon, full_precision=True)
    m = xsg.shape[2]
    state = {}

    def rows():
        state["W"] = ops.kernel_rows_padded(flat, xsg, xg, ch)

    steps = [("k1_rows", rows), ("solve_L", lambda: ch.solve_rows_(state["W"])),
             ("solve_Lt", lambda: ch.solve_many_rows_t_(state["W"])),
             ("solve_Lt_by_substitution", lambda: ch.solve_rows_t_(state["W"])),
             ("cross_bwd_rows_pass", lambda: ops.kernel_cross_bwd(
                 flat, xsg, xg, W=state["W"], r=2.0 * w.reshape(1, m), grad_xsg=torch.zeros_like(xsg))),
             ("cross_bwd_both_passes", lambda: ops.kernel_cross_bwd(
                 flat, xsg, xg, W=state["W"], r=2.0 * w.reshape(1, m), grad_xsg=torch.zeros_like(xsg),
                 grad_xg=torch.zeros_like(xg),
                 term_sum=torch.zeros(1, _lib.GPK_MAX_TERMS, dtype=xg.dtype, device=xg.device)))]
    times = {k: [] for k, _ in steps}
    for _ in range(reps + 1):
        for name, fn in steps:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b))
    return {k: round(sorted(v[1:])[len(v[1:]) // 2], 2) for k, v in times.items()}


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("time_posterior_grad.py needs a CUDA device")
    main()
