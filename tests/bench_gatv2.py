"""bench_gatv2.py — GATv2's dynamic attention against GAT's attention_gather (not a pytest file).  No speed target is
set: these are measurements, for a reader to compare.

    python tests/bench_gatv2.py kernels [--rounds 3] [--iters 5]
    python tests/bench_gatv2.py model [--rounds 2] [--steps 3]

kernels: on R-MAT scale 22 (2^25 generated edges, datasets.rmat_graph seed 1, as tests/bench_attn.py) at H = 64, with
1 head and with 8 heads of 8: the forward, the backward over the same CSR and the exact backward over the transposed
plan, of GATv2 (roc_sg_attn_v2_*) and of GAT (roc_sg_attn_*), each call timed alone with CUDA events after a 256 MB
write that flushes the 50 MB L2, alternating call by call, --iters calls per form per round over --rounds rounds.
model: one training step of GATv2 and of GAT, 602-64-41 with 1 head and 602-(8x8)-41, on bench.py's config-2 graph
(R-MAT-22), alternately in each of --rounds rounds, --steps steps after one warm-up step.
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
from roc_b200.model import Host, Model, build_gat, build_gatv2  # noqa: E402
from bench_inputs import bench_module, node_inputs  # noqa: E402

DEV = "cuda"
SHAPES = [(64, 1), (64, 8)]


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


def kernels(rounds, iters):
    re_, col = datasets.rmat_graph(22, 1 << 25, seed=1, device=DEV)
    n, e = re_.shape[0], col.shape[0]
    plan, tr = K.SgPlan(0, n - 1, 0, re_, col), K.SgTranspose(re_, col)
    print(json.dumps({"graph": "R-MAT scale 22", "N": n, "E": e}), flush=True)
    flush = torch.empty(64 << 20, dtype=torch.float32, device=DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    for h, heads in SHAPES:
        def rows():
            return K.padded(n, h, fill=torch.rand((n, h), generator=gen, device=DEV) - 0.5)
        xl, xr, g = rows(), rows(), rows()
        a = torch.rand((heads, h // heads), generator=gen, device=DEV) - 0.5
        sc = torch.randn((n, 2 * heads), generator=gen, device=DEV)
        out, out1 = K.padded(n, h), K.padded(n, h)
        dxl, dxr, gin = K.padded(n, h), K.padded(n, h), K.padded(n, h)
        stats, stats1 = torch.empty((n, 2 * heads), device=DEV), torch.empty((n, 2 * heads), device=DEV)
        sg = torch.empty((n, 2 * heads), device=DEV)
        plan.attn_v2_forward(xl, xr, a, heads, out=out, stats=stats)
        plan.attn_forward(xl, sc, heads, out=out1, stats=stats1)
        cases = {
            "gatv2_fwd": lambda: plan.attn_v2_forward(xl, xr, a, heads, out=out, stats=stats),
            "gat_fwd": lambda: plan.attn_forward(xl, sc, heads, out=out1, stats=stats1),
            "gatv2_bwd": lambda: plan.attn_v2_backward(xl, xr, a, out, stats, g, heads, dxl=dxl, dxr=dxr),
            "gat_bwd": lambda: plan.attn_backward(xl, sc, out1, stats1, g, heads, in_grad=gin, score_grad=sg),
            "gatv2_bwd_exact": lambda: tr.attn_v2_backward(plan, xl, xr, a, out, stats, g, heads, dxl=dxl, dxr=dxr),
            "gat_bwd_exact": lambda: tr.attn_backward(plan, xl, sc, out1, stats1, g, heads, in_grad=gin,
                                                      score_grad=sg)}
        for fn in cases.values():
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in cases}
        for _ in range(rounds):
            for _ in range(iters):
                for k, fn in cases.items():
                    ms[k].append(timed(fn, flush))
        line = {"what": "attention_kernels", "N": n, "E": e, "H": h, "heads": heads}
        for k in cases:
            line[k] = {"median_ms": round(statistics.median(ms[k]), 3),
                       "range_ms": [round(min(ms[k]), 3), round(max(ms[k]), 3)]}
        for p in ("fwd", "bwd", "bwd_exact"):
            line["gatv2_over_gat_" + p] = round(line["gatv2_" + p]["median_ms"] / line["gat_" + p]["median_ms"], 3)
        print(json.dumps(line), flush=True)
        del xl, xr, g, out, out1, dxl, dxr, gin
        torch.cuda.empty_cache()


def model(rounds, steps):
    B = bench_module()
    re_h, col_h, label = B.make_graph(datasets, 2, 1, DEV)
    n = re_h.shape[0]
    for layers, heads in (([602, 64, 41], 1), ([602, 64, 41], 8)):
        feats, labels, mask = node_inputs(n, layers, DEV)
        forms = {"gatv2": build_gatv2, "gat": build_gat}
        ms = {k: [] for k in forms}
        for _ in range(rounds):
            for name, build in forms.items():
                host = Host(0, 0, 1)
                host.graph_from_arrays(re_h, col_h)
                m = Model(host, seed=1)
                h = build(m, layers, B.DROPOUT, heads=heads, lr=B.LR, weight_decay=B.WD)
                m.set_tensor_from_host_ptr(h["input"], feats.data_ptr())
                m.set_labels(h["label"], labels.numpy())
                m.set_tensor(h["mask"], mask.numpy())
                m.train_epoch()
                torch.cuda.synchronize()
                t0 = time.time()
                for _ in range(steps):
                    m.train_epoch()
                host.synchronize()
                ms[name].append((time.time() - t0) * 1e3 / steps)
                host.close()
                torch.cuda.empty_cache()
        print(json.dumps({"what": "train_step", "layers": layers, "heads": heads, "graph": label, "steps": steps,
                          "ms_per_step": {k: [round(v, 2) for v in vs] for k, vs in ms.items()},
                          "median_ms": {k: round(statistics.median(vs), 2) for k, vs in ms.items()},
                          "gatv2_over_gat": round(statistics.median(ms["gatv2"]) / statistics.median(ms["gat"]), 3)}),
              flush=True)
        del feats, labels, mask
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=("kernels", "model"))
    ap.add_argument("--rounds", type=int, default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    _lib.require_device()
    print(json.dumps({"card": card()}), flush=True)
    if a.mode == "kernels":
        kernels(a.rounds or 3, a.iters)
    else:
        model(a.rounds or 2, a.steps)


if __name__ == "__main__":
    main()
