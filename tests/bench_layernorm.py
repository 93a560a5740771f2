"""bench_layernorm.py — layer normalisation's kernels against their bytes bound, beside batch normalisation's, and its
cost in a training step (not a pytest file).

    python tests/bench_layernorm.py kernels [--rounds 3] [--iters 5] [--widths 41,64,128,256]
    python tests/bench_layernorm.py model [--rounds 2] [--steps 3]

kernels: at N = 4,194,304 rows, per width H, every form alternating call by call, each timed alone with CUDA events
after a 256 MB write that flushes the 50 MB L2, --iters calls per form per round over --rounds rounds: layer norm's
forward with a fused relu (roc_layernorm_fwd), its backward (roc_layernorm_bwd with dX written) and its backward
accumulating into dX; and batch norm's training forward and backward.  Reports the median and the range, and the
matrix passes each form must make at N * round_up4(H) * 4 bytes each, as a bound at the 3.35 TB/s HBM3 of the H100
SXM data sheet: layer norm forward 2 (read x, write y), backward 3 (read x and dY, write dX), accumulating 4; batch
norm training forward 3, backward 5.
model: one training step of GCN 602-64-41 on R-MAT-22 (bench.py's config-2 graph) with norm=None, "batch" and
"layer_norm", and of DeeperGCN 602-64-41 at depth 2 with norm="batch" and "layer_norm", alternately in each of
--rounds rounds, --steps steps after one warm-up step, with the device memory each model holds.
Prints the card (name, power limit, max SM clock) read in the same run, then one JSON line per measurement.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from roc_b200 import _lib, datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402
from roc_b200.model import Host, Model, build_deepergcn, build_gcn  # noqa: E402
from bench_inputs import bench_module, node_inputs  # noqa: E402

PEAK_GBS = 3350.0
DEV = "cuda"
N = 4194304
PASSES = {"ln_fwd": 2, "ln_bwd": 3, "ln_bwd_acc": 4, "bn_train_fwd": 3, "bn_bwd": 5}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def timed(fn, flush):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    flush.zero_()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def kernels(rounds, iters, widths):
    flush = torch.empty(64 << 20, dtype=torch.float32, device=DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    for h in widths:
        ld = (h + 3) // 4 * 4
        x = K.padded(N, h, fill=torch.randn((N, h), generator=gen, device=DEV) * 2 + 1)
        dy = K.padded(N, h, fill=torch.randn((N, h), generator=gen, device=DEV))
        y, dx = K.padded(N, h), K.padded(N, h)
        gamma, beta = torch.rand(h, device=DEV) + 0.5, torch.randn(h, device=DEV)
        rm, rv = torch.zeros(h, device=DEV), torch.ones(h, device=DEV)
        st = K.BatchNormState(N, h)
        cases = {"ln_fwd": lambda: K.layernorm_fwd(x, gamma, beta, relu=True, out=y),
                 "ln_bwd": lambda: K.layernorm_bwd(x, dy, gamma, beta, relu=True, dx=dx),
                 "ln_bwd_acc": lambda: K.layernorm_bwd(x, dy, gamma, beta, relu=True, dx=dx, accumulate=True),
                 "bn_train_fwd": lambda: K.batchnorm_fwd(x, gamma, beta, rm, rv, relu=True, state=st, out=y),
                 "bn_bwd": lambda: K.batchnorm_bwd(x, dy, gamma, st, relu=True, dx=dx)}
        for fn in cases.values():
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in cases}
        for _ in range(rounds):
            for _ in range(iters):
                for k, fn in cases.items():
                    ms[k].append(timed(fn, flush))
        line = {"what": "layernorm_kernels", "N": N, "H": h, "ld": ld, "relu": True}
        for k in cases:
            med = statistics.median(ms[k])
            nbytes = PASSES[k] * N * ld * 4
            line[k] = {"median_ms": round(med, 4), "range_ms": [round(min(ms[k]), 4), round(max(ms[k]), 4)],
                       "bytes": nbytes, "bound_ms": round(nbytes / PEAK_GBS / 1e6, 4),
                       "over_bound": round(med / (nbytes / PEAK_GBS / 1e6), 3)}
        print(json.dumps(line), flush=True)
        del x, dy, y, dx, st
        torch.cuda.empty_cache()


def model(rounds, steps):
    B = bench_module()
    re_h, col_h, label = B.make_graph(datasets, 2, 1, DEV)
    n = re_h.shape[0]
    layers = B.CONFIGS[2]["layers"]
    feats, labels, mask = node_inputs(n, layers, DEV)
    runs = (("gcn", "none"), ("gcn", "batch"), ("gcn", "layer_norm"), ("deepergcn", "batch"),
            ("deepergcn", "layer_norm"))
    ms = {r: [] for r in runs}
    mem = {}
    for _ in range(rounds):
        for name, norm in runs:
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            host = Host(0, 0, 1)
            host.graph_from_arrays(re_h, col_h)
            m = Model(host, seed=1)
            kw = dict(lr=B.LR, weight_decay=B.WD, norm=None if norm == "none" else norm)
            if name == "gcn":
                h = build_gcn(m, layers, B.DROPOUT, **kw)
            else:
                h = build_deepergcn(m, layers, B.DROPOUT, 2, **kw)
            m.set_tensor_from_host_ptr(h["input"], feats.data_ptr())
            m.set_labels(h["label"], labels.numpy())
            m.set_tensor(h["mask"], mask.numpy())
            m.train_epoch()
            torch.cuda.synchronize()
            t0 = time.time()
            for _ in range(steps):
                m.train_epoch()
            host.synchronize()
            ms[(name, norm)].append((time.time() - t0) * 1e3 / steps)
            mem[(name, norm)] = round((free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30, 2)
            host.close()
            torch.cuda.empty_cache()
    for r in runs:
        print(json.dumps({"what": "train_step", "model": r[0], "norm": r[1], "layers": layers, "graph": label,
                          "depth": 2 if r[0] == "deepergcn" else None, "steps": steps,
                          "ms_per_step": [round(v, 2) for v in ms[r]], "median_ms": round(statistics.median(ms[r]), 2),
                          "device_GiB": mem[r]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=("kernels", "model"))
    ap.add_argument("--rounds", type=int, default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--widths", default="41,64,128,256")
    a = ap.parse_args()
    _lib.require_device()
    print(json.dumps({"card": card(), "peak_GBps": PEAK_GBS,
                      "peak_source": "H100 SXM data sheet (3.35 TB/s HBM3)"}), flush=True)
    if a.mode == "kernels":
        kernels(a.rounds or 3, a.iters, [int(x) for x in a.widths.split(",")])
    else:
        model(a.rounds or 2, a.steps)


if __name__ == "__main__":
    main()
