"""bench_batchnorm.py — batch normalisation's kernels against their bytes bound, and its cost in a training step (not a
pytest file).

    python tests/bench_batchnorm.py kernels [--rounds 3] [--iters 5] [--widths 64,128,256]
    python tests/bench_batchnorm.py model [--rounds 2] [--steps 3]

kernels: at N = 4,194,304 rows, per width H, three calls alternating call by call, each timed alone with CUDA events
after a 256 MB write that flushes the 50 MB L2, --iters calls per form per round over --rounds rounds: the training
forward (roc_batchnorm_fwd, statistics + normalise), the inference forward (normalise from the running statistics)
and the backward (roc_batchnorm_bwd with dX, written not accumulated).  Reports the median and the range, and the
matrix passes each form must make — training forward 3 (read x twice, write y), inference 2, backward 5 (read x and
dY twice, write dX) — at N * round_up4(H) * 4 bytes each, as a bound at the 3.35 TB/s HBM3 of the H100 SXM data sheet.
model: one training step of GCN 602-64-41 on R-MAT-22 (bench.py's config-2 graph) and of GraphSAGE-mean with
config 3's layers (100-256-256-47) on its graph, each built with and without norm="batch", alternately in each of
--rounds rounds, --steps steps after one warm-up step.
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
from roc_b200.model import Host, Model, build_gcn, build_sage_mean  # noqa: E402
from bench_inputs import bench_module, node_inputs  # noqa: E402

PEAK_GBS = 3350.0
DEV = "cuda"
N = 4194304
PASSES = {"train_fwd": 3, "infer_fwd": 2, "bwd": 5}


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
        cases = {"train_fwd": lambda: K.batchnorm_fwd(x, gamma, beta, rm, rv, relu=True, state=st, out=y),
                 "infer_fwd": lambda: K.batchnorm_fwd(x, gamma, beta, rm, rv, training=False, relu=True, state=st,
                                                      out=y),
                 "bwd": lambda: K.batchnorm_bwd(x, dy, gamma, st, relu=True, dx=dx)}
        cases["train_fwd"]()
        for fn in cases.values():
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in cases}
        for _ in range(rounds):
            for _ in range(iters):
                for k, fn in cases.items():
                    ms[k].append(timed(fn, flush))
        line = {"what": "batchnorm_kernels", "N": N, "H": h, "ld": ld, "relu": True}
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
    for name, cfg, build in (("gcn", 2, build_gcn), ("sage_mean", 3, build_sage_mean)):
        re_h, col_h, label = B.make_graph(datasets, cfg, 1, DEV)
        n = re_h.shape[0]
        layers = B.CONFIGS[cfg]["layers"]
        feats, labels, mask = node_inputs(n, layers, DEV)
        ms = {"none": [], "batch": []}
        for _ in range(rounds):
            for norm in ("none", "batch"):
                host = Host(0, 0, 1)
                host.graph_from_arrays(re_h, col_h)
                m = Model(host, seed=1)
                h = build(m, layers, B.DROPOUT, lr=B.LR, weight_decay=B.WD, norm=None if norm == "none" else norm)
                m.set_tensor_from_host_ptr(h["input"], feats.data_ptr())
                m.set_labels(h["label"], labels.numpy())
                m.set_tensor(h["mask"], mask.numpy())
                m.train_epoch()
                torch.cuda.synchronize()
                t0 = time.time()
                for _ in range(steps):
                    m.train_epoch()
                host.synchronize()
                ms[norm].append((time.time() - t0) * 1e3 / steps)
                host.close()
                torch.cuda.empty_cache()
        print(json.dumps({"what": "train_step", "model": name, "layers": layers, "graph": label, "steps": steps,
                          "ms_per_step": {k: [round(v, 2) for v in vs] for k, vs in ms.items()},
                          "median_ms": {k: round(statistics.median(vs), 2) for k, vs in ms.items()},
                          "batch_over_none": round(statistics.median(ms["batch"]) / statistics.median(ms["none"]), 3)}),
              flush=True)
        del feats, labels, mask
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=("kernels", "model"))
    ap.add_argument("--rounds", type=int, default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--widths", default="64,128,256")
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
