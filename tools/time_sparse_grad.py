"""Time the sparse ELBO and its gradient at BASELINE config 4 (n = 262144, m = 4096, d = 8, Matern52().stretch(2), noise 0.1,
VFE, fp64): the no-grad ELBO, ELBO + backward with every parameter (variance, length scale, noise, x, z, y) requiring grad,
and ELBO + backward with only z requiring grad.  Prints one JSON line: ms per call, the peak device memory of a call above
the level after ``gc.collect()``, and the card's name and power limit read in the same run."""
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


def main(n=262144, m=4096, d=8, reps=3):
    S.B.epsilon = 1e-12
    g = torch.Generator(device="cuda").manual_seed(4)
    x0 = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    y0 = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    z0 = torch.randn(m, d, dtype=torch.float64, device="cuda", generator=g)

    def run(all_params, z_grad):
        var, scale, noise = (torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=all_params)
                             for v in (1.0, 2.0, 0.1))
        x, y = x0.clone().requires_grad_(all_params), y0.clone().requires_grad_(all_params)
        z = z0.clone().requires_grad_(z_grad)
        f = S.GP(var * S.Matern52().stretch(scale))
        e = S.PseudoObs(f(z), f(x, noise), y).elbo(f.measure)
        if e.requires_grad:
            e.backward()

    def fwd():
        with torch.no_grad():
            run(False, False)

    out = {"n": n, "m": m, "d": d, "chunk": S.B.sparse_chunk, "card": card()}
    for name, fn in (("elbo_ms", fwd), ("elbo_bwd_all_ms", lambda: run(True, True)), ("elbo_bwd_z_ms", lambda: run(False, True))):
        ms, mib = timed(fn, reps)
        out[name] = round(ms, 1)
        out[name.replace("_ms", "_peak_mib")] = round(mib, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("time_sparse_grad.py needs a CUDA device")
    main()
