"""bench_minmax.py — measurements of the max / min aggregation (not a pytest file).  Prints one JSON line per case.

    python tests/bench_minmax.py kernels [--scale 22] [--hs 41,64,128,256] [--iters 10]
        the max forward and backward next to the sum ScatterGather on an R-MAT graph, CUDA events, L2 flushed
    python tests/bench_minmax.py model [--shrink 2] [--steps 10] [--warmup 3] [--aggr max]
        ms per training step of GraphSAGE-pool (build_sage_pool) next to GraphSAGE-mean (build_sage_mean) with
        layers 100-256-256-47 on the products-shaped power-law graph (2.45 M vertices / shrink), dropout 0.5, Adam;
        host clock around steps that end in a device synchronise, models alternated

Writes nothing to the tree.  Every record carries the GPU name and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from roc_b200 import _lib, datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def sum_bytes(n, e, h):
    return e * (4 * h + 4) + n * (4 * h + 8)


def max_fwd_bytes(n, e, h):
    return e * (4 * h + 4) + n * (8 * h + 8)


def max_bwd_bytes(n, e, h):
    return e * (8 * h + 4) + n * (4 * h + 8)


def timeit(fn, iters, flush):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters


def kernels(a):
    dev = "cuda"
    re, col = datasets.rmat_graph(a.scale, 1 << (a.scale + 3), seed=1, device=dev)
    n, e = re.shape[0], col.shape[0]
    plan = K.SgPlan(0, n - 1, 0, re, col)
    gpu = gpu_info()
    print(json.dumps({"graph": "R-MAT scale %d" % a.scale, "N": n, "E": e, "gpu": gpu}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # 256 MB > 50 MB L2
    for h in [int(v) for v in a.hs.split(",")]:
        x = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
        out, gin = K.padded(n, h, dev), K.padded(n, h, dev)
        arg = K.padded(n, h, dev, dtype=torch.int32)
        plan.reserve(h)
        ms_s = timeit(lambda: plan.forward(x, out=out), a.iters, flush)
        ms_f = timeit(lambda: plan.minmax_forward(x, _lib.AGGR_MAX, out=out, arg=arg), a.iters, flush)
        ms_b = timeit(lambda: plan.minmax_backward(x, arg, 0, out=gin), a.iters, flush)
        print(json.dumps({"H": h, "sum_ms": round(ms_s, 4), "max_fwd_ms": round(ms_f, 4), "max_bwd_ms": round(ms_b, 4),
                          "fwd_over_sum": round(ms_f / ms_s, 3), "bwd_over_sum": round(ms_b / ms_s, 3),
                          "sum_GBps": round(sum_bytes(n, e, h) / ms_s / 1e6, 1),
                          "max_fwd_GBps": round(max_fwd_bytes(n, e, h) / ms_f / 1e6, 1),
                          "max_bwd_GBps": round(max_bwd_bytes(n, e, h) / ms_b / 1e6, 1), "gpu": gpu}), flush=True)


def model(a):
    from roc_b200.model import Host, Model, build_sage_mean, build_sage_pool
    layers, dropout, lr, wd = [100, 256, 256, 47], 0.5, 0.01, 0.0001
    re_t, col_t = datasets.powerlaw_graph(2449029 // a.shrink, 30_000_000 // a.shrink, alpha=1.6, seed=1, device="cuda")
    row_end, col = re_t.cpu().numpy().astype(np.uint64), col_t.cpu().numpy().astype(np.uint32)
    del re_t, col_t
    torch.cuda.empty_cache()
    n, e = row_end.shape[0], col.shape[0]
    feats, labels, mask = datasets.node_data(n, layers[0], layers[-1], seed=1)
    aggr = _lib.AGGR_MAX if a.aggr == "max" else _lib.AGGR_MIN
    builders = {"sage-pool-%s" % a.aggr: lambda m: build_sage_pool(m, layers, dropout, aggr=aggr, lr=lr,
                                                                    weight_decay=wd),
                "sage-mean": lambda m: build_sage_mean(m, layers, dropout, lr=lr, weight_decay=wd)}
    gpu = gpu_info()
    times = {k: [] for k in builders}
    for rnd in range(a.rounds):
        for name, build in builders.items():
            host = Host(0, 0, 1)
            host.graph_from_arrays(row_end, col)
            m = Model(host, seed=1)
            h = build(m)
            m.set_tensor(h["input"], feats.numpy())
            m.set_labels(h["label"], labels.numpy())
            m.set_tensor(h["mask"], mask.numpy().astype(np.int32))
            for _ in range(a.warmup):
                m.train_epoch()
            host.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                m.train_epoch()
            host.synchronize()
            times[name].append(1e3 * (time.perf_counter() - t0) / a.steps)
            loss = m.metrics()["trainLoss"]
            host.close()
            print(json.dumps({"model": name, "round": rnd, "ms_per_step": round(times[name][-1], 2),
                              "train_loss": loss, "N": n, "E": e, "layers": layers, "gpu": gpu}), flush=True)
    print(json.dumps({"summary": {k: {"median_ms": round(float(np.median(v)), 2), "min_ms": round(min(v), 2),
                                      "max_ms": round(max(v), 2)} for k, v in times.items()},
                      "graph": "products-shaped power-law / %d (N=%d, E=%d)" % (a.shrink, n, e), "gpu": gpu}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="what", required=True)
    k = sub.add_parser("kernels")
    k.add_argument("--scale", type=int, default=22)
    k.add_argument("--hs", default="41,64,128,256")
    k.add_argument("--iters", type=int, default=10)
    m = sub.add_parser("model")
    m.add_argument("--shrink", type=int, default=2, help="divide the graph's vertices and edges by this")
    m.add_argument("--steps", type=int, default=10)
    m.add_argument("--warmup", type=int, default=3)
    m.add_argument("--rounds", type=int, default=2, help="times each model is built and timed, alternating")
    m.add_argument("--aggr", default="max", choices=["max", "min"])
    a = ap.parse_args()
    _lib.require_device()
    kernels(a) if a.what == "kernels" else model(a)


if __name__ == "__main__":
    main()
