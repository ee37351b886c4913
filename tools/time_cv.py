"""Time multi-fold cross-validation at config 2 (n = 16384, d = 8, ``EQ().stretch(2)``, noise 0.1, fp64 "auto"), for K = 5,
K = 10 (labels ``i % K``, shuffled) and scattered blocks of 64:

* ``cv_marginals`` without grad, and ``cv_logpdf`` + backward with the variance, the length scale, the noise, ``x`` and ``y``
  requiring grad;
* in the same run, ``loo_marginals`` and ``logpdf`` (no grad) for comparison;
* the split of the forward, each stage timed on its own: the full-precision factor with ``alpha``; ``CVFolds.blocks``, the
  fold-block product (chunked trailing solves of identity rows and lower-tile GEMMs); ``CVFolds.factor``, the fold
  factorisations (batched Cholesky, solves, inverse diagonals).

Each is warmed up once and then timed ``reps`` times: host-clock ms around a device synchronise (sorted) and the peak device
memory above the level before the call.  Prints one JSON line with the card's name and power limit read in the same run."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stheno_b200 as S  # noqa: E402
from stheno_b200 import ops  # noqa: E402
from tools.time_sample_function import card  # noqa: E402
from tools.time_sample_function_grad import timed  # noqa: E402


def main(n=16384, d=8, reps=3):
    S.B.epsilon, S.B.precision = 1e-12, "auto"
    g = torch.Generator(device="cuda").manual_seed(0)
    x0 = torch.randn(n, d, dtype=torch.float64, device="cuda", generator=g)
    y0 = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    rng = np.random.default_rng(0)
    layouts = {"K5": rng.permutation(np.arange(n) % 5), "K10": rng.permutation(np.arange(n) % 10),
               "blocks64": rng.permutation(n) // 64}

    def leaves():
        p = [torch.tensor(v, dtype=torch.float64, device="cuda", requires_grad=True) for v in (1.0, 2.0, 0.1)]
        return p, x0.clone().requires_grad_(True), y0.clone().requires_grad_(True)

    def fixed():
        return S.GP(S.EQ().stretch(2.0))(x0, 0.1)

    def no_grad(method, *args):
        def run(_):
            with torch.no_grad():
                return getattr(fixed(), method)(y0, *args)
        return run

    def step(lab):
        def run(a):
            p, x, y = a
            out = S.GP(p[0] * S.EQ().stretch(p[1]))(x, p[2]).cv_logpdf(y, lab)
            out.backward()
            return out
        return run

    flat = ops.FlatKernel([(1.0, [("eq", 0)])], 1)
    xg = (x0 / 2.0).reshape(1, 1, n, d)

    def factor(_):
        ch = ops.chol_from_kernel(flat, xg, noise_scalar=0.1, jitter=1e-12, rhs_t=y0.reshape(1, 1, n), full_precision=True)
        ar = ch.new_rows(1)
        ar[:, :1, :n] = ch.rhs_half()
        ch.solve_rows_t_(ar)
        return ch, ar[:, :1, :n]

    out = {"card": card(), "n": n, "d": d, "precision": "auto"}
    out["loo_marginals"] = timed(lambda: None, no_grad("loo_marginals"), reps)
    out["logpdf"] = timed(lambda: None, no_grad("logpdf"), reps)
    out["factor_and_alpha"] = timed(lambda: None, factor, reps)
    for name, lab in layouts.items():
        sizes = [int(s) for s in np.unique(lab, return_counts=True)[1]]
        out[f"cv_marginals_{name}"] = timed(lambda: None, no_grad("cv_marginals", lab), reps)
        out[f"cv_logpdf_step_{name}"] = timed(leaves, step(lab), reps)
        ch, alpha = factor(None)
        folds = ops.CVFolds(ch, sizes, alpha)
        out[f"fold_blocks_{name}"] = timed(lambda: None, lambda _: folds.blocks(ch), reps)
        out[f"fold_factors_{name}"] = timed(lambda: folds.blocks(ch), folds.factor, reps)
        del ch, alpha, folds
    print(json.dumps(out))


if __name__ == "__main__":
    main(n=int(sys.argv[1]) if len(sys.argv) > 1 else 16384)
