"""bench_dw_ab.py — the two dW kernels against each other (not a pytest file): k_tc_linear_dw_ws (the default at
outDim <= 128) and k_tc_linear_dw (ROC_B200_DW=sync), alternated call by call in one process on the same operands,
plain and with the fused dropout mask, as tests/bench_dw.py times them.

    python tests/bench_dw_ab.py [--rows 4194304] [--shapes 602x64,64x41,602x128,256x47] [--rounds 3] [--iters 5]
Prints one JSON line per (shape, op) with each kernel's per-round times and their range.  At outDim > 128 both
names run the synchronised kernel (a spread check).
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_dw import timeit  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402


def with_kernel(kernel, fn):
    def run():
        if kernel == "sync":
            os.environ["ROC_B200_DW"] = "sync"
        else:
            os.environ.pop("ROC_B200_DW", None)
        fn()
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 22)
    ap.add_argument("--shapes", default="602x64,64x41,602x128,256x47")
    ap.add_argument("--rounds", type=int, default=3)
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

        def run_dw():
            dw.zero_()
            K.linear_bwd(x[:, :i], w, None, dy[:, :o], dw)

        def run_dw_mask():
            dw.zero_()
            K.linear_bwd_dropout(x[:, :i], w, None, dy[:, :o], dw, mask, 0.5)

        for op, fn in (("linear_dw", run_dw), ("linear_dw+mask", run_dw_mask)):
            ms = {"sync": [], "ws": []}
            for _ in range(a.rounds):
                for kernel in ("sync", "ws"):
                    ms[kernel].append(round(timeit(with_kernel(kernel, fn), a.iters), 4))
            os.environ.pop("ROC_B200_DW", None)
            print(json.dumps({"op": op, "shape": shp, "rows": n, "sync_ms": ms["sync"], "ws_ms": ms["ws"],
                              "sync_range": [min(ms["sync"]), max(ms["sync"])],
                              "ws_range": [min(ms["ws"]), max(ms["ws"])]}), flush=True)
        del x, dy, mask, dw


if __name__ == "__main__":
    main()
