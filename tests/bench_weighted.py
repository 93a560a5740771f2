"""bench_weighted.py — measurements of edge-weighted aggregation (not a pytest file).  Prints one JSON line per case.

    python tests/bench_weighted.py kernels [--scale 22] [--hs 41,64,128,256] [--iters 10] [--rounds 3]
        the weighted forward, its transposed backward (weight permutation + gather) and the edge dot next to the sum's
        forward and backward (the same gather over the same CSR, quirk Q1) on an R-MAT graph; CUDA events with L2
        flushed, the kernels alternated within each round; median and min-max over the rounds.  A torch.profiler run
        then splits the backward into its launches.  The transpose's build time and memory (measured with
        cudaMemGetInfo around its creation and its first backward) come first.
    python tests/bench_weighted.py model [--scale 22] [--steps 10] [--warmup 3] [--rounds 2]
        ms per training step of the weighted GCN 602-64-41 (build_gcn_weighted, gcn_edge_weights of all-ones weights,
        no edge gradient) next to GCN 602-64-41 (build_gcn) on the same R-MAT graph, dropout 0.5, Adam; host clock
        around steps that end in a device synchronise, models alternated

Algorithmic bytes: forward E(4H+8) + N(4H+8); backward E*12 (the permutation) plus the forward's bytes on the
transpose; edge dot E(4H+8) + N*4H (+ E*4 when accumulating); the sum E(4H+4) + N(4H+8).
Writes nothing to the tree.  Every record carries the GPU name and its power limit.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench_minmax import gpu_info, sum_bytes  # noqa: E402
from roc_b200 import _lib, datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402


def fwd_bytes(n, e, h):
    return e * (4 * h + 8) + n * (4 * h + 8)


def bwd_bytes(n, e, h):
    return e * 12 + fwd_bytes(n, e, h)


def dot_bytes(n, e, h):
    return e * (4 * h + 8) + n * 4 * h


def time_once(fn, flush):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def stats(v):
    return {"median_ms": round(float(np.median(v)), 4), "min_ms": round(min(v), 4), "max_ms": round(max(v), 4)}


def kernels(a):
    dev = "cuda"
    re, col = datasets.rmat_graph(a.scale, 1 << (a.scale + 3), seed=1, device=dev)
    n, e = re.shape[0], col.shape[0]
    plan = K.SgPlan(0, n - 1, 0, re, col)
    gpu = gpu_info()
    w = torch.rand(e, device=dev)
    gy0 = K.padded(n, 1, dev)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    tr = K.SgTranspose(re, col)
    torch.cuda.synchronize()
    build_ms = 1e3 * (time.perf_counter() - t0)
    free1 = torch.cuda.mem_get_info()[0]
    tr.backward(gy0, w)                                       # grows the permuted-weight buffer (and H = 1 carries)
    torch.cuda.synchronize()
    free2 = torch.cuda.mem_get_info()[0]
    # measured: device memory the transpose took (cudaMemGetInfo before and after; nothing else allocates between)
    print(json.dumps({"graph": "R-MAT scale %d" % a.scale, "N": n, "E": e, "transpose_build_ms": round(build_ms, 1),
                      "transpose_bytes": free0 - free1, "transpose_bytes_with_wT": free0 - free2,
                      "weights_bytes": 4 * e, "gpu": gpu}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # 256 MB > 50 MB L2
    for h in [int(v) for v in a.hs.split(",")]:
        x = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
        gy = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
        out, gin = K.padded(n, h, dev), K.padded(n, h, dev)
        dw = torch.empty(e, device=dev)
        plan.reserve(h)
        cases = {"sum_fwd": lambda: plan.forward(x, out=out),
                 "sum_bwd": lambda: plan.forward(gy, out=gin),
                 "wfwd": lambda: plan.weighted_forward(x, w, out=out),
                 "wbwd": lambda: tr.backward(gy, w, out=gin),
                 "edge_dot": lambda: plan.edge_dot(gy, x, dw=dw)}
        for fn in cases.values():
            fn(); fn()
        torch.cuda.synchronize()
        t = {k: [] for k in cases}
        for _ in range(a.rounds):
            for k, fn in cases.items():
                t[k].append(float(np.mean([time_once(fn, flush) for _ in range(a.iters)])))
        med = {k: float(np.median(v)) for k, v in t.items()}
        rec = {"H": h, "gpu": gpu}
        rec.update({k: stats(v) for k, v in t.items()})
        rec.update({"wfwd_over_sum": round(med["wfwd"] / med["sum_fwd"], 3),
                    "wbwd_over_sum_bwd": round(med["wbwd"] / med["sum_bwd"], 3),
                    "edge_dot_over_sum": round(med["edge_dot"] / med["sum_fwd"], 3),
                    "sum_GBps": round(sum_bytes(n, e, h) / med["sum_fwd"] / 1e6, 1),
                    "wfwd_GBps": round(fwd_bytes(n, e, h) / med["wfwd"] / 1e6, 1),
                    "wbwd_GBps": round(bwd_bytes(n, e, h) / med["wbwd"] / 1e6, 1),
                    "edge_dot_GBps": round(dot_bytes(n, e, h) / med["edge_dot"] / 1e6, 1)})
        # the backward's launches, split by a profiler run (kernel name -> mean device ms)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.iters):
                tr.backward(gy, w, out=gin)
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            if ev.device_type == torch.autograd.DeviceType.CUDA and ev.count:
                name = "permute" if "k_permute" in ev.key else "fixup" if "fixup" in ev.key else "gather"
                split[name] = split.get(name, 0.0) + ev.device_time_total / 1e3 / a.iters
        rec["wbwd_split_ms"] = {k: round(v, 4) for k, v in split.items()}
        print(json.dumps(rec), flush=True)
    tr.close()


def model(a):
    from roc_b200.model import Host, Model, build_gcn, build_gcn_weighted
    layers, dropout = [602, 64, 41], 0.5
    re_t, col_t = datasets.rmat_graph(a.scale, 1 << (a.scale + 3), seed=1)
    row_end, col = re_t.numpy().astype(np.uint64), col_t.numpy().astype(np.uint32)
    n, e = row_end.shape[0], col.shape[0]
    ew = datasets.gcn_edge_weights(row_end, col, np.ones(e))
    feats, labels, mask = datasets.node_data(n, layers[0], layers[-1], seed=1)
    builders = {"gcn-weighted": lambda m: build_gcn_weighted(m, layers, dropout, ew),
                "gcn": lambda m: build_gcn(m, layers, dropout)}
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
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({"summary": {k: {"median_ms": round(med[k], 2), "min_ms": round(min(v), 2),
                                      "max_ms": round(max(v), 2)} for k, v in times.items()},
                      "weighted_over_gcn": round(med["gcn-weighted"] / med["gcn"], 3),
                      "graph": "R-MAT scale %d (N=%d, E=%d)" % (a.scale, n, e), "gpu": gpu}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="what", required=True)
    k = sub.add_parser("kernels")
    k.add_argument("--scale", type=int, default=22)
    k.add_argument("--hs", default="41,64,128,256")
    k.add_argument("--iters", type=int, default=10)
    k.add_argument("--rounds", type=int, default=3)
    m = sub.add_parser("model")
    m.add_argument("--scale", type=int, default=22)
    m.add_argument("--steps", type=int, default=10)
    m.add_argument("--warmup", type=int, default=3)
    m.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    _lib.require_device()
    kernels(a) if a.what == "kernels" else model(a)


if __name__ == "__main__":
    main()
