"""Time leave-one-out predictive marginals and LOO log densities at config 2 (n = 16384, d = 8, ``EQ().stretch(2)``, noise 0.1,
fp64 "auto"):

* ``loo_marginals`` without grad;
* ``loo_logpdf`` + backward with the variance, the length scale, the noise, ``x`` and ``y`` requiring grad;
* for comparison, ``logpdf`` and ``logpdf`` + backward on the same inputs;
* torch eager fp64 (``cholesky``, ``cholesky_inverse``, cuSOLVER / cuBLAS) forming the same LOO values, and the same with
  autograd for the loss + gradient step.

Each is warmed up once and then timed ``reps`` times: host-clock ms around a device synchronise (sorted) and the peak device
memory above the level before the call.  Prints one JSON line with the card's name and power limit read in the same run."""
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stheno_b200 as S  # noqa: E402
from tools.time_sample_function import card  # noqa: E402
from tools.time_sample_function_grad import timed  # noqa: E402


def torch_loo(K, r):
    L = torch.linalg.cholesky(K)
    alpha = torch.cholesky_solve(r, L)
    c = torch.diagonal(torch.cholesky_inverse(L))
    s = alpha / c[:, None]
    return r - s, 1.0 / c, 0.5 * ((torch.log(c)[:, None] - alpha * s).sum(0) - K.shape[0] * math.log(2 * math.pi))


def main(n=16384, d=8, reps=3):
    S.B.epsilon, S.B.precision = 1e-12, "auto"
    g = torch.Generator(device="cuda").manual_seed(0)
    x0 = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    y0 = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)

    def leaves():
        p = [torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True) for v in (1.0, 2.0, 0.1)]
        return p, x0.clone().requires_grad_(True), y0.clone().requires_grad_(True)

    def fdd(p, x):
        return S.GP(p[0] * S.EQ().stretch(p[1]))(x, p[2])

    def step(method):
        def run(a):
            p, x, y = a
            out = getattr(fdd(p, x), method)(y)
            out.backward()
            return out
        return run

    def no_grad(method):
        def run(_):
            with torch.no_grad():
                return getattr(S.GP(S.EQ().stretch(2.0))(x0, 0.1), method)(y0)
        return run

    def torch_fwd(_):
        with torch.no_grad():
            K = torch.cdist(x0 / 2.0, x0 / 2.0).pow_(2).mul_(-0.5).exp_()
            K.diagonal().add_(0.1 + 1e-12)
            return torch_loo(K, y0[:, None])

    def torch_step(a):
        p, x, y = a
        xs = x / p[1]
        sq = (xs * xs).sum(-1)
        K = p[0] * torch.exp(-0.5 * (sq[:, None] + sq[None, :] - 2 * xs @ xs.T))
        K = K + (p[2] + 1e-12) * torch.eye(n, dtype=K.dtype, device=K.device)
        lp = torch_loo(K, y[:, None])[2].sum()
        lp.backward()
        return lp

    out = {"card": card(), "n": n, "d": d, "precision": "auto"}
    out["loo_marginals"] = timed(lambda: None, no_grad("loo_marginals"), reps)
    out["logpdf"] = timed(lambda: None, no_grad("logpdf"), reps)
    out["loo_logpdf_step"] = timed(leaves, step("loo_logpdf"), reps)
    out["logpdf_step"] = timed(leaves, step("logpdf"), reps)
    out["torch_loo_marginals"] = timed(lambda: None, torch_fwd, reps)
    out["torch_loo_step"] = timed(leaves, torch_step, reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main(n=int(sys.argv[1]) if len(sys.argv) > 1 else 16384)
