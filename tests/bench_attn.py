"""bench_attn.py — measurements of the attention aggregation (not a pytest file).  Prints one JSON line per case.

    python tests/bench_attn.py kernels [--scale 22] [--hs 64,256] [--heads 1,8] [--iters 10] [--rounds 3]
        the attention forward and backward next to the sum ScatterGather on an R-MAT graph, CUDA events, L2 flushed,
        the three alternated in every round; then, in a separate profiled run, each direction's device time split
        by launch (pass 1 / pass 2 / fix-ups; records / B1 / B2 / fix-ups) from torch.profiler
    python tests/bench_attn.py model [--scale 22] [--steps 10] [--warmup 3] [--rounds 2]
        ms per training step of GAT 602-64-41 (one head, and 8 heads of 8) next to GCN 602-64-41 on the same R-MAT
        graph, dropout 0.5, Adam; host clock around steps that end in a device synchronise, models alternated

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


# Algorithmic bytes: what each launch must read or write once, by the kernels' own schedule (DESIGN §3.1).
def sum_bytes(n, e, h):
    return e * (4 * h + 4) + n * (4 * h + 8)


def attn_fwd_bytes(n, e, h, k):
    # pass 1: col + s_src per edge; s_dst, stats and rs per row.  pass 2: col, X[j] and s_src per edge; s_dst, stats,
    # out and rs per row.
    return e * (4 * h + 8 + 8 * k) + n * (4 * h + 16 + 24 * k)


def attn_bwd_bytes(n, e, h, k):
    # records: G, O, s_dst and stats in, the record out per node.  B1: col, X[j], s_src per edge; G[i], the record,
    # d s_dst and rs per row.  B2: col, G[j] and the record of j per edge; X[i], s_src, inGrad, d s_src and rs per row.
    return e * (8 * h + 8 + 20 * k) + n * (20 * h + 56 * k + 16)


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


# which part of an attention call a kernel is: sg_chunk_kernel's last template argument is its reduction
PARTS = {"4": "stats pass", "5": "weighted sum", "6": "B1 (d s_dst)", "7": "B2 (inGrad, d s_src)"}


def part_of(name):
    if "sg_attn_rec_kernel" in name:
        return "records"
    if "sg_attn_stat_fixup" in name or "sg_fixup" in name:
        return "fix-ups"
    if "sg_chunk_kernel<" in name:
        return PARTS.get(name.split(">(")[0].split(",")[-1].strip(), "other")
    return "other"


def split(fn, iters):
    """ms per call of each part of fn, from the CUDA kernels torch.profiler records."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    parts = {}
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = getattr(ev, "cuda_time_total", 0.0)
        if us:
            k = part_of(ev.key)
            parts[k] = parts.get(k, 0.0) + us / 1e3 / iters
    return {k: round(v, 4) for k, v in sorted(parts.items())}


def spread(v):
    return {"median": round(float(np.median(v)), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def kernels(a):
    dev = "cuda"
    re, col = datasets.rmat_graph(a.scale, 1 << (a.scale + 3), seed=1, device=dev)
    n, e = re.shape[0], col.shape[0]
    plan = K.SgPlan(0, n - 1, 0, re, col)
    gpu = gpu_info()
    print(json.dumps({"graph": "R-MAT scale %d" % a.scale, "N": n, "E": e, "gpu": gpu}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # 256 MB > 50 MB L2
    cases = []
    for h in [int(v) for v in a.hs.split(",")]:
        x = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
        g = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
        out, gin = K.padded(n, h, dev), K.padded(n, h, dev)
        plan.reserve(h)
        for k in [int(v) for v in a.heads.split(",")]:
            sc = torch.randn((n, 2 * k), device=dev)
            stats, sg = torch.empty((n, 2 * k), device=dev), torch.empty((n, 2 * k), device=dev)
            plan.attn_backward(x, sc, out, stats, g, k, in_grad=gin, score_grad=sg)   # the one-time id scan
            cases.append((h, k, lambda x=x, out=out: plan.forward(x, out=out),
                          lambda x=x, sc=sc, k=k, out=out, stats=stats: plan.attn_forward(x, sc, k, out=out, stats=stats),
                          lambda x=x, sc=sc, k=k, out=out, stats=stats, g=g, gin=gin, sg=sg:
                              plan.attn_backward(x, sc, out, stats, g, k, in_grad=gin, score_grad=sg)))
    times = {(h, k): {"sum": [], "fwd": [], "bwd": []} for h, k, *_ in cases}
    for rnd in range(a.rounds):
        for h, k, f_sum, f_fwd, f_bwd in cases:
            t = times[(h, k)]
            t["sum"].append(timeit(f_sum, a.iters, flush))
            t["fwd"].append(timeit(f_fwd, a.iters, flush))
            t["bwd"].append(timeit(f_bwd, a.iters, flush))
    for h, k, f_sum, f_fwd, f_bwd in cases:
        t = times[(h, k)]
        ms_s, ms_f, ms_b = (float(np.median(t[w])) for w in ("sum", "fwd", "bwd"))
        print(json.dumps({"H": h, "heads": k, "rounds": a.rounds, "iters": a.iters, "sum_ms": spread(t["sum"]),
                          "attn_fwd_ms": spread(t["fwd"]), "attn_bwd_ms": spread(t["bwd"]),
                          "fwd_over_sum": round(ms_f / ms_s, 3), "bwd_over_sum": round(ms_b / ms_s, 3),
                          "sum_GBps": round(sum_bytes(n, e, h) / ms_s / 1e6, 1),
                          "attn_fwd_GBps": round(attn_fwd_bytes(n, e, h, k) / ms_f / 1e6, 1),
                          "attn_bwd_GBps": round(attn_bwd_bytes(n, e, h, k) / ms_b / 1e6, 1), "gpu": gpu}),
              flush=True)
    for h, k, f_sum, f_fwd, f_bwd in cases:       # profiled separately: tracing slows the host
        print(json.dumps({"H": h, "heads": k, "split": "ms per call by launch (torch.profiler, L2 not flushed)",
                          "fwd": split(f_fwd, a.iters), "bwd": split(f_bwd, a.iters), "gpu": gpu}), flush=True)


def model(a):
    from roc_b200.model import Host, Model, build_gat, build_gcn
    layers, dropout, lr, wd = [602, 64, 41], 0.5, 0.01, 0.0001
    re_t, col_t = datasets.rmat_graph(a.scale, 1 << (a.scale + 3), seed=1, device="cuda")
    row_end, col = re_t.cpu().numpy().astype(np.uint64), col_t.cpu().numpy().astype(np.uint32)
    del re_t, col_t
    torch.cuda.empty_cache()
    n, e = row_end.shape[0], col.shape[0]
    feats, labels, mask = datasets.node_data(n, layers[0], layers[-1], seed=1)
    builders = {"gat-1-head": lambda m: build_gat(m, layers, dropout, heads=1, lr=lr, weight_decay=wd),
                "gat-8-heads": lambda m: build_gat(m, layers, dropout, heads=8, lr=lr, weight_decay=wd),
                "gcn": lambda m: build_gcn(m, layers, dropout, lr=lr, weight_decay=wd)}
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
                      "graph": "R-MAT scale %d (N=%d, E=%d)" % (a.scale, n, e), "gpu": gpu}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="what", required=True)
    k = sub.add_parser("kernels")
    k.add_argument("--scale", type=int, default=22)
    k.add_argument("--hs", default="64,256")
    k.add_argument("--heads", default="1,8")
    k.add_argument("--iters", type=int, default=10)
    k.add_argument("--rounds", type=int, default=3, help="times every case is timed, the cases alternating")
    m = sub.add_parser("model")
    m.add_argument("--scale", type=int, default=22)
    m.add_argument("--steps", type=int, default=10)
    m.add_argument("--warmup", type=int, default=3)
    m.add_argument("--rounds", type=int, default=2, help="times each model is built and timed, alternating")
    a = ap.parse_args()
    _lib.require_device()
    kernels(a) if a.what == "kernels" else model(a)


if __name__ == "__main__":
    main()
