"""K1: the specialised single-factor kernel against the generic descriptor kernel, agreement and time.  The generic kernel
runs the same kernel with a ``("one", 0)`` factor appended, which the specialised one does not take.
python tools/time_k1.py  ->  one JSON line per kernel."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_variant(variant):
    import torch

    sys.path.insert(0, ROOT)
    from stheno_b200 import ops

    out = {"variant": variant}
    g = torch.Generator(device="cuda").manual_seed(1)
    n, d = 16384, 8
    x = torch.randn(1, 1, n, d, device="cuda", dtype=torch.float64, generator=g) / 2.0
    extra = [("one", 0)] if variant == "generic" else []
    for kind in ("eq", "matern12", "matern32", "matern52"):
        flat = ops.FlatKernel([(1.3, [(kind, 0)] + extra)], 1)
        W = torch.empty(1, n, n, device="cuda", dtype=torch.float64)
        def run():
            ops._km_launch(flat, x, x, n, n, d, ops.KM_LOWER | ops.KM_SAME | ops.KM_PAD_IDENTITY, 0.1, None, 1e-12, W, n, n * n, 1)
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            run()
        e1.record()
        torch.cuda.synchronize()
        out[f"{kind}_lower_ms"] = e0.elapsed_time(e1) / 10
        # checksum + a sample against a float64 torch evaluation
        idx = torch.randint(0, n, (4096,), device="cuda", generator=g)
        jdx = (idx * 7919 + 13) % n
        lo = torch.maximum(idx, jdx), torch.minimum(idx, jdx)
        got = W[0, lo[0], lo[1]]
        d2 = ((x[0, 0, lo[0]] - x[0, 0, lo[1]]) ** 2).sum(-1)
        r = torch.sqrt(torch.clamp_min(d2, 1e-30))
        ref = {"eq": torch.exp(-0.5 * d2), "matern12": torch.exp(-r),
               "matern32": (1 + 3 ** 0.5 * r) * torch.exp(-(3 ** 0.5) * r),
               "matern52": (1 + 5 ** 0.5 * r + 5.0 / 3.0 * d2) * torch.exp(-(5 ** 0.5) * r)}[kind] * 1.3
        ref = ref + (lo[0] == lo[1]) * (0.1 + 1e-12)
        out[f"{kind}_max_rel_err_vs_torch"] = ((got - ref).abs() / ref.abs().clamp_min(1e-300)).max().item()
        out[f"{kind}_checksum"] = float(torch.tril(W[0]).sum())
    # fp32 full square
    xf = x.float()
    flat = ops.FlatKernel([(1.0, [("eq", 0)] + extra)], 1)
    Wf = torch.empty(1, n, n, device="cuda", dtype=torch.float32)
    for _ in range(3):
        ops._km_launch(flat, xf, xf, n, n, d, ops.KM_SAME, 0.1, None, 1e-6, Wf, n, n * n, 1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        ops._km_launch(flat, xf, xf, n, n, d, ops.KM_SAME, 0.1, None, 1e-6, Wf, n, n * n, 1)
    e1.record()
    torch.cuda.synchronize()
    out["eq_f32_full_ms"] = e0.elapsed_time(e1) / 10
    out["eq_f32_full_GBs"] = n * n * 4 / (out["eq_f32_full_ms"] * 1e-3) / 1e9
    out["eq_f64_lower_GBs"] = (n * n / 2 + 64 * n) * 8 / (out["eq_lower_ms"] * 1e-3) / 1e9
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    for variant in ("fast", "generic"):
        run_variant(variant)
