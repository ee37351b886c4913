"""Time loss + gradient through a periodic kernel against the no-grad call, fp64:

* the exact posterior of ``(1.2 * EQ().stretch(0.8)).periodic(1.7)`` with n = 16384 observations in 2-D and m = 4096 test
  points: the marginals, and ``sum(mean + 2 sd)`` + backward with the variance, length scale, period, noise, x, x* and y
  requiring grad;
* the VFE ELBO of ``(Matern52().stretch(2)).periodic(3)`` at n = 262144, m = 4096, d = 8 (config 4's data with the periodic
  map): the ELBO, and ELBO + backward with the variance, length scale, period, noise and z requiring grad;
* the periodic map itself at the exact problem's points (forward + backward of its torch ops), to show its share.

Prints one JSON line: ms per call, the peak device memory of a call above the level after ``gc.collect()``, and the card's
name and power limit read in the same run."""
import gc
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
    gc.collect()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3, (torch.cuda.max_memory_allocated() - base) / 2**20


def leaves(vals, grad):
    return [torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=grad) for v in vals]


def exact(out, reps, n=16384, m=4096, d=2):
    g = torch.Generator(device="cuda").manual_seed(1)
    x0 = torch.rand(n, d, dtype=torch.float64, device="cuda", generator=g) * 3
    xs0 = torch.rand(m, d, dtype=torch.float64, device="cuda", generator=g) * 3
    y0 = torch.sin(2 * x0.sum(-1))

    def run(grad):
        v, ell, p, noise = leaves((1.2, 0.8, 1.7, 0.1), grad)
        x, xs, y = (t.clone().requires_grad_(grad) for t in (x0, xs0, y0))
        f = S.GP((v * S.EQ().stretch(ell)).periodic(p))
        mean, var = (f | (f(x, noise), y))(xs).marginals()
        if grad:
            (mean + 2 * var.sqrt()).sum().backward()

    def fwd():
        with torch.no_grad():
            run(False)

    def map_only():
        p = torch.tensor(1.7, dtype=torch.float64, device="cuda", requires_grad=True)
        x = x0.clone().requires_grad_()
        ang = x * (2 * torch.pi) / p
        torch.cat([torch.sin(ang), torch.cos(ang)], dim=-1).sum().backward()

    for name, fn in (("exact_marginals_ms", fwd), ("exact_marginals_bwd_ms", lambda: run(True)),
                     ("periodic_map_fwd_bwd_ms", map_only)):
        ms, mib = timed(fn, reps)
        out[name] = round(ms, 2)
        out[name.replace("_ms", "_peak_mib")] = round(mib, 1)


def sparse(out, reps, n=262144, m=4096, d=8):
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    y = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    z0 = torch.randn(m, d, dtype=torch.float64, device="cuda", generator=g)

    def run(grad):
        v, ell, p, noise = leaves((1.0, 2.0, 3.0, 0.1), grad)
        z = z0.clone().requires_grad_(grad)
        f = S.GP((v * S.Matern52().stretch(ell)).periodic(p))
        e = S.PseudoObs(f(z), f(x, noise), y).elbo(f.measure)
        if grad:
            e.backward()

    def fwd():
        with torch.no_grad():
            run(False)

    for name, fn in (("sparse_elbo_ms", fwd), ("sparse_elbo_bwd_ms", lambda: run(True))):
        ms, mib = timed(fn, reps)
        out[name] = round(ms, 1)
        out[name.replace("_ms", "_peak_mib")] = round(mib, 1)


def main(reps=3):
    S.B.epsilon = 1e-12
    out = {"card": card(), "chunk": S.B.sparse_chunk}
    exact(out, reps)
    sparse(out, reps)
    print(json.dumps(out))


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("time_mapped_grad.py needs a CUDA device")
    main()
