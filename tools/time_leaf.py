"""Leaf Cholesky: correctness against torch.linalg.cholesky and latency of the shipped leaf kernels (fp64: the recursive
kernel, fp32: the flat register-tiled one), and whole log-pdf steps around them.  python tools/time_leaf.py  ->  one JSON
line."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    import torch

    sys.path.insert(0, ROOT)
    from stheno_b200 import ops

    out = {}
    g = torch.Generator(device="cuda").manual_seed(0)
    for dtype, tol in ((torch.float64, 1e-12), (torch.float32, 2e-5)):
        for n, batch in ((128, 1), (128, 300), (512, 1), (1024, 3), (2000, 1)):
            M = torch.randn(batch, n, n, device="cuda", dtype=torch.float64, generator=g)
            K = (M @ M.transpose(1, 2) / n + torch.eye(n, device="cuda", dtype=torch.float64)).to(dtype)
            ch = ops.chol_from_dense(K, jitter=0.0)
            L = ch.L()
            ref = torch.linalg.cholesky(K.double())
            err = ((L.double() - ref).abs().max() / ref.abs().max()).item()
            ld = (ch.logdet.double() - 2 * torch.log(torch.diagonal(ref, dim1=1, dim2=2)).sum(-1)).abs().max().item()
            key = f"{str(dtype)[-7:]}_n{n}_b{batch}"
            out[key] = {"err": err, "logdet_err": ld, "info": int(ch.info.abs().max())}
            assert err < tol * 50 and ch.info.abs().max() == 0, (key, out[key])
    # non-PD: the pivot index must be reported
    K = torch.eye(256, device="cuda", dtype=torch.float64)
    K[200, 200] = -1.0
    ch = ops.chol_from_dense(K[None], jitter=0.0)
    out["info_non_pd"] = int(ch.info[0])
    assert out["info_non_pd"] == 201, out
    # latency of one 128-leaf: potrf on n_pad = 128 (one launch of the leaf kernel)
    for dtype in (torch.float64, torch.float32):
        W0 = (torch.eye(128, device="cuda", dtype=dtype) * 4 + 0.01).reshape(1, 128, 128).contiguous()
        reps = 200
        Ws = W0.repeat(reps, 1, 1)
        logdet = torch.zeros(1, device="cuda", dtype=dtype)
        info = torch.zeros(1, device="cuda", dtype=torch.int32)
        fn = ops._fn("gpk_potrf", dtype)

        def run():
            for i in range(reps):
                fn(ops._ptr(Ws[i]), 128, 128 * 128, 128, 0, ops._ptr(logdet), ops._ptr(info), 1, ops._stream())

        run()
        torch.cuda.synchronize()
        Ws.copy_(W0.repeat(reps, 1, 1))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        out[f"leaf_us_{str(dtype)[-7:]}"] = e0.elapsed_time(e1) * 1e3 / reps
    # n = 16384 logpdf (whole step), 5 reps
    import stheno_b200 as S

    x = torch.randn(16384, 8, device="cuda", dtype=torch.float64, generator=g)
    y = torch.randn(16384, device="cuda", dtype=torch.float64, generator=g)
    k = S.EQ().stretch(2.0) + 0.1 * S.Delta()
    for prec in ("auto", "fp64"):
        S.B.precision = prec
        for _ in range(3):
            lp = S.GP(k)(x).logpdf(y)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            lp = S.GP(k)(x).logpdf(y)
        e1.record()
        torch.cuda.synchronize()
        out[f"logpdf16384_ms_{prec}"] = e0.elapsed_time(e1) / 10
        out[f"logpdf16384_{prec}"] = float(lp)
    # batched fp32 (config 3 share): 64 x 2048
    S.B.precision = "auto"
    S.B.epsilon = 1e-6
    xb = torch.randn(64, 2048, 8, device="cuda", generator=g)
    yb = torch.randn(64, 2048, 1, device="cuda", generator=g)
    for _ in range(3):
        lpb = S.GP(S.EQ())(xb, 0.1).logpdf(yb)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        lpb = S.GP(S.EQ())(xb, 0.1).logpdf(yb)
    e1.record()
    torch.cuda.synchronize()
    out["c3_64x2048_ms"] = e0.elapsed_time(e1) / 10
    out["c3_sum"] = float(lpb.sum())
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
