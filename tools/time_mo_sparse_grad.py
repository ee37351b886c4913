"""Time the sparse ELBO over several processes and its gradient: 4 observed processes x 65536 points, inducing points on each
of them (4 x 1024), d = 8, VFE, fp64 ``auto``.  Two independent latents with Matern52 kernels, observed as ``f1``, ``f2``,
``f1 + f2`` and ``f1 - f2 / 2``; noise 0.1, inducing noise 1e-3.  Prints one JSON line: ms per call of the no-grad ELBO and
of ELBO + backward with every parameter (coefficients, length scales, noise, x, z, y) requiring grad, the peak device memory
of a call above the level after ``gc.collect()``, and the card's name and power limit read in the same run."""
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


def main(n_p=65536, m_q=1024, d=8, reps=3):
    S.B.epsilon = 1e-12
    g = torch.Generator(device="cuda").manual_seed(4)
    xs0 = [torch.randn(n_p, d, dtype=torch.float64, device="cuda", generator=g) for _ in range(4)]
    ys0 = [torch.randn(n_p, dtype=torch.float64, device="cuda", generator=g) for _ in range(4)]
    zs0 = [torch.randn(m_q, d, dtype=torch.float64, device="cuda", generator=g) for _ in range(4)]

    def run(grad):
        p = [torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=grad) for v in (1.0, 2.0, 0.5, 3.0, 0.1)]
        xs = [x.clone().requires_grad_(grad) for x in xs0]
        ys = [y.clone().requires_grad_(grad) for y in ys0]
        zs = [z.clone().requires_grad_(grad) for z in zs0]
        f1 = S.GP(p[0] * S.Matern52().stretch(p[1]))
        f2 = S.GP(p[2] * S.Matern52().stretch(p[3]), measure=f1.measure)
        ps = [f1, f2, f1 + f2, f1 + f2 * -0.5]
        u = tuple(q(z, 1e-3) for q, z in zip(ps, zs))
        e = S.PseudoObs(u, *[(q(x, p[4]), y) for q, x, y in zip(ps, xs, ys)]).elbo(f1.measure)
        if e.requires_grad:
            e.backward()

    def fwd():
        with torch.no_grad():
            run(False)

    out = {"n": 4 * n_p, "m": 4 * m_q, "d": d, "chunk": S.B.sparse_chunk, "card": card()}
    for name, fn in (("elbo_ms", fwd), ("elbo_bwd_all_ms", lambda: run(True))):
        ms, mib = timed(fn, reps)
        out[name] = round(ms, 1)
        out[name.replace("_ms", "_peak_mib")] = round(mib, 1)
    out["ratio"] = round(out["elbo_bwd_all_ms"] / out["elbo_ms"], 2)
    print(json.dumps(out))


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("time_mo_sparse_grad.py needs a CUDA device")
    main()
