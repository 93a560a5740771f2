"""bench_linear_cfg2.py — the three k_tc_linear launches of bench.py config 2's step, each alone (not a pytest file).

    python tests/bench_linear_cfg2.py [--rows 4194304] [--rounds 3] [--iters 10]

fwd 602 -> 64 and 64 -> 41 with the dropout mask on the input and the indegree-norm epilogue, and dX 41 -> 64 with the
dropout-backward, relu-mask and norm epilogue (parts = ONLY_DX), CUDA-event timed on HBM-resident operands larger than
L2.  Bytes are what a launch must move at the padded leading dimensions: A, Y, mask words, reluOf and the row ends,
each once.  Prints the card (name, power limit, max SM clock), then one JSON line per launch and round: ms, GB/s and
the share of the H100 SXM data-sheet 3.35 TB/s, and roc_last_gemm_info of the launch.
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from roc_b200 import _lib  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402

_spec = importlib.util.spec_from_file_location("bench_linear", os.path.join(HERE, "bench_linear.py"))
_bl = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_bl)
timeit = _bl.timeit

PEAK_GBS = 3350.0


def pad4(h):
    return (h + 3) // 4 * 4


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        return torch.cuda.get_device_name(0)


def fwd_case(n, i, o, re, g, dev):
    x = K.padded(n, i, dev)
    x[:, :i] = torch.rand(n, i, device=dev, generator=g) * 2 - 1
    w = (torch.rand(o, i, device=dev, generator=g) - 0.5) * 0.2
    y = K.padded(n, o, dev)
    mask = K.dropout_mask(n, i, 0, 0.5, 5, 1, dev)
    byt = n * (pad4(i) * 4 + o * 4 + mask.stride(0) * 4 + 8)
    return ("fwd %d->%d mask+norm" % (i, o), byt,
            lambda: K.linear_fwd_dropout(x[:, :i], w, mask, 0.5, norm_row_end=re, out=y[:, :o]), _lib.GEMM_FWD)


def dx_case(n, i, o, re, g, dev):
    dy = K.padded(n, o, dev)
    dy[:, :o] = torch.rand(n, o, device=dev, generator=g) * 2 - 1
    ro = K.padded(n, i, dev)
    ro[:, :i] = torch.rand(n, i, device=dev, generator=g) - 0.5
    w = (torch.rand(o, i, device=dev, generator=g) - 0.5) * 0.2
    dx = K.padded(n, i, dev)
    dw = torch.zeros(o, i, device=dev)
    mask = K.dropout_mask(n, i, 0, 0.5, 5, 1, dev)
    byt = n * (pad4(o) * 4 + i * 4 + pad4(i) * 4 + mask.stride(0) * 4 + 8)
    return ("dX %d->%d omask+reluof+norm" % (o, i), byt,
            lambda: K.linear_bwd_fused(ro[:, :i], w, None, dy[:, :o], dw, dx[:, :i], mask=mask, rate=0.5,
                                       relu_of=ro[:, :i], norm_row_end=re, parts=_lib.LINEAR_BWD_ONLY_DX),
            _lib.GEMM_DX)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 22)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    dev = "cuda"
    n = a.rows
    print(json.dumps({"card": card(), "peak_GBps": PEAK_GBS,
                      "peak_source": "H100 SXM data sheet (3.35 TB/s HBM3)"}), flush=True)
    g = torch.Generator(device=dev).manual_seed(2)
    re = torch.cumsum(torch.randint(1, 30, (n,), device=dev, generator=g), 0)
    for make, i, o in ((fwd_case, 602, 64), (fwd_case, 64, 41), (dx_case, 64, 41)):
        name, byt, fn, which = make(n, i, o, re, g, dev)
        for _ in range(a.rounds):
            ms = timeit(fn, a.iters)
            gbs = byt / ms / 1e6
            print(json.dumps({"launch": name, "rows": n, "ms": round(ms, 4), "GB": round(byt / 1e9, 3),
                              "GBps": round(gbs, 1), "frac_of_peak": round(gbs / PEAK_GBS, 3),
                              "bound_ms": round(byt / PEAK_GBS / 1e6, 4), "info": _lib.last_gemm_info(which)}),
                  flush=True)
        del fn
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
