"""bench_exact.py — measurements of the exact backwards over the transpose (not a pytest file).  Prints one JSON line
per case.

    python tests/bench_exact.py kernels [--scale 22] [--hs 41,64,128,256] [--iters 10] [--rounds 3]
        on a symmetric R-MAT graph (rmat_graph(scale, 2^(scale+3)), as the other benchmarks) and a directed one
        (rmat_graph(scale, 2^(scale+4), directed=True): twice the pairs, as no reverse edges are added, for a similar
        edge count): each exact backward next to its gather over the same CSR (quirk Q1) — the sum with the NORM
        epilogue, the max backward, and attention with 1 and 8 heads.  CUDA events with L2 flushed, each exact call
        alternated with its gather call by call; median and min-max over the rounds.  A torch.profiler run then splits each exact
        call into its launches.  The transpose's build time and memory (cudaMemGetInfo around its creation) come first.
    python tests/bench_exact.py model [--scale 22] [--steps 10] [--warmup 3] [--rounds 2]
        ms per training step of GCN 602-64-41, GraphSAGE-pool 602-64-41 (max) and GAT 602-64-41 (one head) on the
        directed graph, with the gather backward and with the exact one (set_exact_backward); dropout 0.5, Adam; host
        clock around steps that end in a device synchronise, the variants alternated

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
from bench_minmax import gpu_info  # noqa: E402
from bench_weighted import stats, time_once  # noqa: E402
from roc_b200 import _lib, datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402


def graph(scale, directed, device="cpu"):
    if directed:
        return datasets.rmat_graph(scale, 1 << (scale + 4), seed=1, device=device, directed=True)
    return datasets.rmat_graph(scale, 1 << (scale + 3), seed=1, device=device)


def launch_split(fn, iters):
    """kernel family -> mean device ms per call, from a profiler run."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.count:
            k = ev.key
            name = ("record" if "rec_kernel" in k else "big_fixup" if "fixup_big" in k else "fixup" if "fixup" in k
                    else "ring" if "kernel_t" in k else "main" if "sg_chunk" in k else "other")
            split[name] = split.get(name, 0.0) + ev.device_time_total / 1e3 / iters
    return {k: round(v, 4) for k, v in split.items()}


def kernels(a):
    dev = "cuda"
    gpu = gpu_info()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # 256 MB > 50 MB L2
    for directed in (False, True):
        re, col = graph(a.scale, directed, dev)
        n, e = re.shape[0], col.shape[0]
        name = "R-MAT scale %d %s" % (a.scale, "directed" if directed else "symmetric")
        plan = K.SgPlan(0, n - 1, 0, re, col)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        t0 = time.perf_counter()
        tr = K.SgTranspose(re, col)
        torch.cuda.synchronize()
        build_ms = 1e3 * (time.perf_counter() - t0)
        free1 = torch.cuda.mem_get_info()[0]
        # measured: device memory the transpose took (cudaMemGetInfo before and after; nothing else allocates between)
        print(json.dumps({"graph": name, "N": n, "E": e, "transpose_build_ms": round(build_ms, 1),
                          "transpose_bytes": free0 - free1, "gpu": gpu}), flush=True)
        for h in [int(v) for v in a.hs.split(",")]:
            x = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
            gy = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
            gin = K.padded(n, h, dev)
            _, arg = plan.minmax_forward(x, _lib.AGGR_MAX)
            plan.reserve(h)
            tr.sum_backward(gy, _lib.SG_EPI_NORM, re, out=gin)             # grows the transposed plan's carries
            cases = {"sum_q1": lambda: plan.forward(gy, out=gin, epilogue=_lib.SG_EPI_NORM),
                     "sum_exact": lambda: tr.sum_backward(gy, _lib.SG_EPI_NORM, re, out=gin),
                     "max_q1": lambda: plan.minmax_backward(gy, arg, out=gin),
                     "max_exact": lambda: tr.minmax_backward(gy, arg, out=gin)}
            for heads in (1, 8):
                if h % heads or (heads > 1 and ((h // heads) < 4 or (h // heads) & (h // heads - 1))):
                    continue
                sc = torch.randn((n, 2 * heads), device=dev)
                ao, st = plan.attn_forward(x, sc, heads)
                sg = torch.empty((n, 2 * heads), device=dev)
                cases["attn%d_q1" % heads] = (lambda sc=sc, ao=ao, st=st, heads=heads, sg=sg: plan.attn_backward(
                    x, sc, ao, st, gy, heads, in_grad=gin, score_grad=sg))
                cases["attn%d_exact" % heads] = (lambda sc=sc, ao=ao, st=st, heads=heads, sg=sg: tr.attn_backward(
                    plan, x, sc, ao, st, gy, heads, in_grad=gin, score_grad=sg))
            for fn in cases.values():
                fn(); fn()
            torch.cuda.synchronize()
            # each exact call is timed right after its gather, pair by pair, so that both see the same clocks
            t = {k: [] for k in cases}
            for _ in range(a.rounds):
                for base in [k[:-len("_q1")] for k in cases if k.endswith("_q1")]:
                    pair = {base + "_q1": [], base + "_exact": []}
                    for _ in range(a.iters):
                        for k in pair:
                            pair[k].append(time_once(cases[k], flush))
                    for k, v in pair.items():
                        t[k].append(float(np.mean(v)))
            med = {k: float(np.median(v)) for k, v in t.items()}
            rec = {"graph": name, "H": h, "gpu": gpu}
            rec.update({k: stats(v) for k, v in t.items()})
            for k in cases:
                if k.endswith("_exact"):
                    base = k[:-len("_exact")]
                    rec[base + "_exact_over_q1"] = round(med[k] / med[base + "_q1"], 3)
                    rec[base + "_split_ms"] = {"q1": launch_split(cases[base + "_q1"], a.iters),
                                               "exact": launch_split(cases[k], a.iters)}
            print(json.dumps(rec), flush=True)
        tr.close()
        plan.close()
        del re, col
        torch.cuda.empty_cache()


def model(a):
    from roc_b200.model import Host, Model, build_gat, build_gcn, build_sage_pool
    layers, dropout = [602, 64, 41], 0.5
    re_t, col_t = graph(a.scale, True)
    row_end, col = re_t.numpy().astype(np.uint64), col_t.numpy().astype(np.uint32)
    n, e = row_end.shape[0], col.shape[0]
    feats, labels, mask = datasets.node_data(n, layers[0], layers[-1], seed=1)
    builders = {"gcn": lambda m, ex: build_gcn(m, layers, dropout, exact_backward=ex),
                "sage-pool": lambda m, ex: build_sage_pool(m, layers, dropout, exact_backward=ex),
                "gat": lambda m, ex: build_gat(m, layers, dropout, exact_backward=ex)}
    gpu = gpu_info()
    times = {(k, ex): [] for k in builders for ex in (False, True)}
    for rnd in range(a.rounds):
        for (name, ex) in times:
            host = Host(0, 0, 1)
            host.graph_from_arrays(row_end, col)
            m = Model(host, seed=1)
            h = builders[name](m, ex)
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
            times[(name, ex)].append(1e3 * (time.perf_counter() - t0) / a.steps)
            loss = m.metrics()["trainLoss"]
            host.close()
            print(json.dumps({"model": name, "backward": "exact" if ex else "q1", "round": rnd,
                              "ms_per_step": round(times[(name, ex)][-1], 2), "train_loss": loss, "N": n, "E": e,
                              "layers": layers, "gpu": gpu}), flush=True)
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({"summary": {"%s/%s" % (k, "exact" if ex else "q1"): {
                          "median_ms": round(med[(k, ex)], 2), "min_ms": round(min(v), 2), "max_ms": round(max(v), 2)}
                      for (k, ex), v in times.items()},
                      "exact_over_q1": {k: round(med[(k, True)] / med[(k, False)], 3) for k in builders},
                      "graph": "R-MAT scale %d directed (N=%d, E=%d)" % (a.scale, n, e), "gpu": gpu}), flush=True)


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
