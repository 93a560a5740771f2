"""bench_edge_dropout.py — measurements of edge dropout on the sum ScatterGather (not a pytest file).  Prints one JSON
line per case, each with the GPU name and its power limit.

    python tests/bench_edge_dropout.py [kernels|model|all] [--scale 22] [--hs 41,64,256] [--rates 0,0.1,0.5]
        kernels: on bench.py's R-MAT graph, CUDA events with L2 flushed, at every (H, rate): the forward
        (roc_sg_forward_dropout_planned, NORM), the backward over the same CSR (the same call on the gradient with the
        reverse pairs' bytes, NORM), the teleport hop (roc_sg_forward_teleport_dropout_planned, NORM | NORM_OUT) and the
        keep-mask pass (roc_sg_attn_keep_mask) alone, alternated in every round.  Rate 0 is the plain calls.  Each
        case carries its algorithmic bytes; the gathered rows are counted at (1 - rate) of the edges, which is what the
        kernel asks for, not what reaches DRAM (R-MAT's neighbour rows hit L2 heavily).
        model: ms per training step of APPNP 602-64-41 (K = 10) and GCN 602-64-41, each with and without
        edge_dropout=0.5, on bench.py's config-2 graph; host clock around steps that end in a device synchronise,
        models alternated.

Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_attn import gpu_info, spread, timeit  # noqa: E402
from roc_b200 import _lib, datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402
from roc_b200.model import Host, Model, build_appnp, build_gcn  # noqa: E402

PAIRS = 1 << 25      # bench.py's BASE_PAIRS at scale 22
NORM, NORM_OUT = _lib.SG_EPI_NORM, _lib.SG_EPI_NORM_OUT
KEY = (1 << 32) | 5


def r4(h):
    return (h + 3) // 4 * 4


def graph(scale, dev):
    return datasets.rmat_graph(scale, PAIRS if scale == 22 else 1 << (scale + 3), seed=1, device=dev)


def drop_bytes(n, e, h, rate):
    """the dropped sum: col and the keep byte per edge, the kept edges' rows, the row starts and the output row"""
    return int(e * 5 + (1.0 - rate) * e * 4 * h + n * (4 * h + 8)) if rate else e * (4 * h + 4) + n * (4 * h + 8)


def mask_bytes(n, e):
    """the keep-mask pass: col in and one byte out per edge, the row starts it searches"""
    return e * 5 + n * 4


def kernels(a, gpu):
    dev = "cuda"
    re, col = graph(a.scale, dev)
    n, e = re.shape[0], col.shape[0]
    plan = K.SgPlan(0, n - 1, 0, re, col)
    print(json.dumps({"graph": "R-MAT scale %d" % a.scale, "N": n, "E": e, "gpu": gpu}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # 256 MB > 50 MB L2
    alpha, beta = float(np.float32(0.9)), float(np.float32(0.1))
    keep = torch.empty(e, dtype=torch.uint8, device=dev)
    rev = torch.empty(e, dtype=torch.uint8, device=dev)
    for h in [int(v) for v in a.hs.split(",")]:
        plan.reserve(h)
        x = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
        t = K.padded(n, h, dev, fill=torch.rand((n, h), device=dev) - 0.5)
        out, ws = K.padded(n, h, dev), K.padded(n, h, dev)
        for rate in [float(v) for v in a.rates.split(",")]:
            if rate:
                plan.attn_keep_mask(rate, KEY, 3, out=keep)
                plan.attn_keep_mask(rate, KEY, 3, row_is_source=True, out=rev)
                # the bytes are the weighted chain's (checked here at size, at every rate)
                s = float(np.float32(1.0) / (np.float32(1.0) - np.float32(rate)))
                w = torch.where((keep & 1).bool(), torch.tensor(s, device=dev), torch.tensor(0.0, device=dev))
                plan.forward_dropout(x, keep, rate, out=out)
                plan.weighted_forward(x, w.float(), out=ws)
                assert torch.equal(out.view(torch.int32), ws.view(torch.int32)), "the dropped sum differs"
            k, kr = (keep, rev) if rate else (None, None)
            fns = {
                "forward": lambda: plan.forward_dropout(x, k, rate, out=out, epilogue=NORM),
                "backward": lambda: plan.forward_dropout(x, kr, rate, out=out, epilogue=NORM),
                "teleport": lambda: plan.teleport_forward_dropout(x, t, alpha, beta, k, rate, NORM | NORM_OUT,
                                                                  out=out),
            }
            if rate:
                fns["keep_mask"] = lambda: plan.attn_keep_mask(rate, KEY, 3, out=keep)
            ts = {name: [] for name in fns}
            for _ in range(a.rounds):
                for name, fn in fns.items():
                    ts[name].append(timeit(fn, a.iters, flush))
            b = drop_bytes(n, e, r4(h), rate)
            nbytes = {"forward": b, "backward": b, "teleport": b + n * 4 * r4(h), "keep_mask": mask_bytes(n, e)}
            for name, v in ts.items():
                print(json.dumps({"case": name, "H": h, "rate": rate, "gpu": gpu, "ms": spread(v),
                                  "bytes": nbytes[name], "bytes_bound_ms": round(nbytes[name] / 3.35e9, 4)}),
                      flush=True)
        del x, t, out, ws
        torch.cuda.empty_cache()


def step_ms(m, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        m.train_epoch()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def model(a, gpu):
    dev = "cuda"
    re_t, col_t = graph(a.scale, dev)
    row_end, col = re_t.cpu().numpy().astype(np.uint64), col_t.cpu().numpy().astype(np.uint32)
    del re_t, col_t
    n = row_end.shape[0]
    print(json.dumps({"graph": "R-MAT scale %d" % a.scale, "N": n, "E": int(col.shape[0]), "gpu": gpu}), flush=True)
    feats, labels, mask = (t.numpy() for t in datasets.node_data(n, 602, 41, seed=1))
    cases = {
        "appnp K=10": lambda m: build_appnp(m, [602, 64, 41], 0.5, K=10, weight_decay=1e-4),
        "appnp K=10 edge_dropout=0.5": lambda m: build_appnp(m, [602, 64, 41], 0.5, K=10, weight_decay=1e-4,
                                                             edge_dropout=0.5),
        "gcn": lambda m: build_gcn(m, [602, 64, 41], 0.5, weight_decay=1e-4),
        "gcn edge_dropout=0.5": lambda m: build_gcn(m, [602, 64, 41], 0.5, weight_decay=1e-4, edge_dropout=0.5),
    }
    ts = {k: [] for k in cases}
    for _ in range(a.model_rounds):
        for name, build in cases.items():
            host = Host(0, 0, 1)
            host.graph_from_arrays(row_end, col)
            m = Model(host, seed=1)
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
    ap.add_argument("what", nargs="?", default="all", choices=["kernels", "model", "all"])
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--hs", default="41,64,256")
    ap.add_argument("--rates", default="0,0.1,0.5")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--model-rounds", type=int, default=2)
    a = ap.parse_args()
    _lib.require_device()
    gpu = gpu_info()
    if a.what in ("kernels", "all"):
        kernels(a, gpu)
    if a.what in ("model", "all"):
        model(a, gpu)


if __name__ == "__main__":
    main()
