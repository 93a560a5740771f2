"""bench_appnp.py — measurements of the APPNP / GCNII hop (not a pytest file).  Prints one JSON line per case.

    python tests/bench_appnp.py kernels [--scale 22] [--hs 41,47,64,112] [--iters 10] [--rounds 3]
        on bench.py's R-MAT graph, CUDA events, L2 flushed, the two alternated in every round: the teleport sum with
        NORM | NORM_OUT (roc_sg_forward_teleport_planned) against the unfused chain roc_sg_forward_planned(NORM) ->
        roc_scaled_add_fwd -> roc_indegree_norm, with each one's algorithmic bytes
    python tests/bench_appnp.py model [--scale 22] [--steps 5] [--warmup 2] [--rounds 2]
        ms per training step of APPNP 602-64-41 (K = 10), GCNII 602-64-41 (depth 16), fused and with set_fusion(False),
        and GCN 602-64-41, on bench.py's config-2 graph; host clock around steps that end in a device synchronise,
        models alternated; --cases picks some (one process per case keeps each model's device memory to itself)

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
from bench_attn import ROOT, gpu_info, spread, sum_bytes, timeit  # noqa: E402,F401
from roc_b200 import _lib, datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402
from roc_b200.model import Host, Model, build_appnp, build_gcn, build_gcnii  # noqa: E402

PAIRS = 1 << 25      # bench.py's BASE_PAIRS at scale 22
NORM, NORM_OUT = _lib.SG_EPI_NORM, _lib.SG_EPI_NORM_OUT


def r4(h):
    return (h + 3) // 4 * 4


def graph(scale, dev):
    return datasets.rmat_graph(scale, PAIRS if scale == 22 else 1 << (scale + 3), seed=1, device=dev)


def kernels(a):
    dev = "cuda"
    re, col = graph(a.scale, dev)
    n, e = re.shape[0], col.shape[0]
    plan = K.SgPlan(0, n - 1, 0, re, col)
    gpu = gpu_info()
    print(json.dumps({"graph": "R-MAT scale %d" % a.scale, "N": n, "E": e, "gpu": gpu}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # 256 MB > 50 MB L2
    alpha, beta = float(np.float32(0.9)), float(np.float32(0.1))
    for h in [int(v) for v in a.hs.split(",")]:
        plan.reserve(h)
        x = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
        t = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
        out, s, y = K.padded(n, h, dev), K.padded(n, h, dev), K.padded(n, h, dev)

        def fused():
            plan.teleport_forward(x, t, alpha, beta, NORM | NORM_OUT, out=out)

        def chain():
            plan.forward(x, out=s, epilogue=NORM)
            K.scaled_add_fwd(s, t, alpha, beta, out=y)
            K.indegree_norm(0, n - 1, 0, re, y, out=out)

        fused(); ref = out.clone(); chain()
        assert torch.equal(ref.view(torch.int32), out.view(torch.int32)), "the teleport's bytes differ from the chain's"
        ts = {"fused": [], "chain": []}
        for _ in range(a.rounds):
            ts["fused"].append(timeit(fused, a.iters, flush))
            ts["chain"].append(timeit(chain, a.iters, flush))
        row = 4 * r4(h)
        # the teleport also reads t and the row ends once; the chain writes s, reads s and t, writes y, reads y
        fb = sum_bytes(n, e, r4(h)) + n * row
        cb = sum_bytes(n, e, r4(h)) + 5 * n * row + n * 16
        print(json.dumps({"case": "hop", "H": h, "gpu": gpu,
                          "teleport_ms": spread(ts["fused"]), "chain_ms": spread(ts["chain"]),
                          "teleport_bytes": fb, "chain_bytes": cb,
                          "teleport_bytes_bound_ms": round(fb / 3.35e9, 4),
                          "chain_bytes_bound_ms": round(cb / 3.35e9, 4)}), flush=True)
        del x, t, out, s, y
        torch.cuda.empty_cache()


def step_ms(m, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        m.train_epoch()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def model(a):
    dev = "cuda"
    re_t, col_t = graph(a.scale, dev)
    row_end, col = re_t.cpu().numpy().astype(np.uint64), col_t.cpu().numpy().astype(np.uint32)
    n = row_end.shape[0]
    gpu = gpu_info()
    print(json.dumps({"graph": "R-MAT scale %d" % a.scale, "N": n, "E": int(col.shape[0]), "gpu": gpu}), flush=True)
    feats, labels, mask = (t.numpy() for t in datasets.node_data(n, 602, 41, seed=1))
    cases = {
        "appnp K=10": (lambda m: build_appnp(m, [602, 64, 41], 0.5, K=10, weight_decay=1e-4), True),
        "appnp K=10 unfused": (lambda m: build_appnp(m, [602, 64, 41], 0.5, K=10, weight_decay=1e-4), False),
        "gcnii depth=16": (lambda m: build_gcnii(m, [602, 64, 41], 0.5, 16, weight_decay=1e-4), True),
        "gcnii depth=16 unfused": (lambda m: build_gcnii(m, [602, 64, 41], 0.5, 16, weight_decay=1e-4), False),
        "gcn": (lambda m: build_gcn(m, [602, 64, 41], 0.5, weight_decay=1e-4), True),
    }
    if a.cases:
        cases = {k: v for k, v in cases.items() if k in a.cases.split(",")}
    ts = {k: [] for k in cases}
    for _ in range(a.rounds):
        for name, (build, fuse) in cases.items():
            host = Host(0, 0, 1)
            host.graph_from_arrays(row_end, col)
            m = Model(host, seed=1)
            m.set_fusion(fuse)
            h = build(m)
            m.set_tensor(h["input"], feats)
            m.set_labels(h["label"], labels)
            m.set_tensor(h["mask"], mask.astype(np.int32))
            step_ms(m, a.warmup)
            ts[name].append(step_ms(m, a.steps))
            host.close()
    for name, v in ts.items():
        print(json.dumps({"case": "step", "model": name, "gpu": gpu, "ms": spread(v)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["kernels", "model"])
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--hs", default="41,47,64,112")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cases", default="", help="model: a comma list of case names (default: all)")
    a = ap.parse_args()
    _lib.require_device()
    kernels(a) if a.what == "kernels" else model(a)


if __name__ == "__main__":
    main()
