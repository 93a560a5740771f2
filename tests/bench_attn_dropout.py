"""bench_attn_dropout.py — measurements of attention dropout (not a pytest file).  Prints one JSON line per case.

    python tests/bench_attn_dropout.py kernels [--scale 22] [--hs 64,256] [--heads 1,8] [--iters 10] [--rounds 3]
        on an R-MAT graph, CUDA events, L2 flushed, every case alternated in every round: the keep-mask generator in
        the forward and the reverse-pair order, and the attention forward and backward without and with dropout
        (rate 0.6); then, in a separate profiled run, each call's device time split by pass from torch.profiler, so
        each dropout pass can be set against the same pass without dropout
    python tests/bench_attn_dropout.py model [--scale 22] [--steps 10] [--warmup 3] [--rounds 2]
        ms per training step of the paper's GAT 602-(8x8)-41 (per-head scores, ELU, dropout 0.6) with attn_dropout 0.6
        and 0 on the same R-MAT graph; host clock around steps that end in a device synchronise, models alternated

Writes nothing to the tree.  Every record carries the GPU name and its power limit.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_attn import ROOT, gpu_info, spread, timeit  # noqa: E402,F401
from roc_b200 import _lib, datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402

RATE, SEED = 0.6, 7

# sg_chunk_kernel's last template argument is its reduction; 32 + r is pass r with dropout
PARTS = {"4": "stats pass", "5": "weighted sum", "6": "B1 (d s_dst)", "7": "B2 (inGrad, d s_src)",
         "37": "weighted sum", "38": "B1 (d s_dst)", "39": "B2 (inGrad, d s_src)"}


def part_of(name):
    if "k_attn_keep" in name:
        return "keep mask"
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


def kernels(a):
    dev = "cuda"
    re, col = datasets.rmat_graph(a.scale, 1 << (a.scale + 3), seed=1, device=dev)
    n, e = re.shape[0], col.shape[0]
    plan = K.SgPlan(0, n - 1, 0, re, col)
    gpu = gpu_info()
    print(json.dumps({"graph": "R-MAT scale %d" % a.scale, "N": n, "E": e, "rate": RATE, "gpu": gpu}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # 256 MB > 50 MB L2
    keep = plan.attn_keep_mask(RATE, SEED, 1)
    keep_rev = plan.attn_keep_mask(RATE, SEED, 1, row_is_source=True)
    gen = {"gen_forward_order": lambda: plan.attn_keep_mask(RATE, SEED, 1, out=keep),
           "gen_reverse_order": lambda: plan.attn_keep_mask(RATE, SEED, 1, row_is_source=True, out=keep_rev)}
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
            fns = {
                "fwd": lambda x=x, sc=sc, k=k, out=out, stats=stats: plan.attn_forward(x, sc, k, out=out, stats=stats),
                "fwd_drop": lambda x=x, sc=sc, k=k, out=out, stats=stats:
                    plan.attn_forward_dropout(x, sc, keep, RATE, k, out=out, stats=stats),
                "bwd": lambda x=x, sc=sc, k=k, out=out, stats=stats, g=g, gin=gin, sg=sg:
                    plan.attn_backward(x, sc, out, stats, g, k, in_grad=gin, score_grad=sg),
                "bwd_drop": lambda x=x, sc=sc, k=k, out=out, stats=stats, g=g, gin=gin, sg=sg:
                    plan.attn_backward_dropout(x, sc, out, stats, g, keep, keep_rev, RATE, k, in_grad=gin,
                                               score_grad=sg)}
            cases.append((h, k, fns))
    gtimes = {w: [] for w in gen}
    times = {(h, k): {w: [] for w in fns} for h, k, fns in cases}
    for rnd in range(a.rounds):
        for w, f in gen.items():
            gtimes[w].append(timeit(f, a.iters, flush))
        for h, k, fns in cases:
            for w, f in fns.items():
                times[(h, k)][w].append(timeit(f, a.iters, flush))
    print(json.dumps({"E": e, "generator_ms": {w: spread(v) for w, v in gtimes.items()}, "gpu": gpu}), flush=True)
    for h, k, fns in cases:
        t = times[(h, k)]
        med = {w: float(np.median(v)) for w, v in t.items()}
        print(json.dumps({"H": h, "heads": k, "rounds": a.rounds, "iters": a.iters,
                          **{w + "_ms": spread(v) for w, v in t.items()},
                          "fwd_drop_over_fwd": round(med["fwd_drop"] / med["fwd"], 3),
                          "bwd_drop_over_bwd": round(med["bwd_drop"] / med["bwd"], 3), "gpu": gpu}), flush=True)
    for h, k, fns in cases:       # profiled separately: tracing slows the host
        parts = {w: split(f, a.iters) for w, f in fns.items()}
        ratio = {}
        for plain, drop in (("fwd", "fwd_drop"), ("bwd", "bwd_drop")):
            for p, ms in parts[drop].items():
                if p in parts[plain] and p in ("weighted sum", "B1 (d s_dst)", "B2 (inGrad, d s_src)"):
                    ratio[p] = round(ms / parts[plain][p], 3)
        print(json.dumps({"H": h, "heads": k, "split": "ms per call by launch (torch.profiler, L2 not flushed)",
                          **parts, "pass_drop_over_plain": ratio, "gpu": gpu}), flush=True)


def model(a):
    from roc_b200.model import Host, Model, build_gat
    layers, dropout, lr, wd = [602, 64, 41], 0.6, 0.005, 0.0005
    re_t, col_t = datasets.rmat_graph(a.scale, 1 << (a.scale + 3), seed=1, device="cuda")
    row_end, col = re_t.cpu().numpy().astype(np.uint64), col_t.cpu().numpy().astype(np.uint32)
    del re_t, col_t
    torch.cuda.empty_cache()
    n, e = row_end.shape[0], col.shape[0]
    feats, labels, mask = datasets.node_data(n, layers[0], layers[-1], seed=1)
    paper = dict(heads=8, scores="per_head", activation="elu", lr=lr, weight_decay=wd)
    builders = {"attn_dropout=0.6": lambda m: build_gat(m, layers, dropout, attn_dropout=RATE, **paper),
                "attn_dropout=0": lambda m: build_gat(m, layers, dropout, **paper)}
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
            print(json.dumps({"model": "GAT 602-(8x8)-41 " + name, "round": rnd,
                              "ms_per_step": round(times[name][-1], 2), "train_loss": loss, "N": n, "E": e,
                              "gpu": gpu}), flush=True)
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({"summary": {k: {"median_ms": round(float(np.median(v)), 2), "min_ms": round(min(v), 2),
                                      "max_ms": round(max(v), 2)} for k, v in times.items()},
                      "drop_over_plain": round(med["attn_dropout=0.6"] / med["attn_dropout=0"], 3),
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
