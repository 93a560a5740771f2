"""bench_dw.py — micro-benchmark of the Linear weight gradient (k_tc_linear_dw + k_splitk_reduce) alone (not a pytest
file).

dW = dY^T X, plain and on dropout(X) with the keep-mask fused into the operand load (how the training step runs it),
CUDA-event timed on HBM-resident operands larger than L2, with a sampled fp64 check of the plain dW so a fast wrong
kernel is caught here.  The default shapes are config 2's; the dW shapes of configs 3-5 are
    --shapes 100x256,256x256,256x47,602x128,602x256
    python tests/bench_dw.py [--rows 4194304] [--shapes 602x64,64x41] [--iters 5]
Prints one JSON line per (shape, op): ms, and GB/s over the algorithmic bytes (X and dY once, plus the mask).
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from roc_b200 import kernels as K  # noqa: E402


def timeit(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 22)
    ap.add_argument("--shapes", default="602x64,64x41")
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(1)
    for shp in a.shapes.split(","):
        i, o = (int(t) for t in shp.split("x"))
        n = a.rows
        x = K.padded(n, i, dev)
        x[:, :i] = torch.randn(n, i, device=dev, generator=g)
        w = torch.randn(o, i, device=dev, generator=g) * 0.1
        dy = K.padded(n, o, dev)
        dy[:, :o] = torch.randn(n, o, device=dev, generator=g)
        mask = K.dropout_mask(n, i, 0, 0.5, 5, 1, dev)
        dw = torch.zeros(o, i, device=dev)
        byt = n * (i + o) * 4

        def run_dw():
            dw.zero_()
            K.linear_bwd(x[:, :i], w, None, dy[:, :o], dw)

        def run_dw_mask():
            dw.zero_()
            K.linear_bwd_dropout(x[:, :i], w, None, dy[:, :o], dw, mask, 0.5)

        ms = timeit(run_dw, a.iters)
        m = min(n, 1 << 16)        # fp64 check on a prefix (exact function of the same kernel path)
        dw2 = torch.zeros(o, i, device=dev)
        K.linear_bwd(x[:m, :i], w, None, dy[:m, :o], dw2)
        ref = dy[:m, :o].double().t() @ x[:m, :i].double()
        err = ((dw2.double() - ref).abs().max() / ref.abs().max()).item()
        print(json.dumps({"op": "linear_dw", "shape": shp, "rows": n, "ms": round(ms, 4),
                          "GBps": round(byt / ms / 1e6, 1), "max_rel_err_prefix": err}), flush=True)
        ms = timeit(run_dw_mask, a.iters)
        mbyt = byt + n * mask.stride(0) * 4
        print(json.dumps({"op": "linear_dw+mask", "shape": shp, "rows": n, "ms": round(ms, 4),
                          "GBps": round(mbyt / ms / 1e6, 1)}), flush=True)
        del x, dy, mask, dw, dw2


if __name__ == "__main__":
    main()
