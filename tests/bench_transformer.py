"""bench_transformer.py — the graph transformer's dot-product attention against the sum and GAT's attention_gather (not
a pytest file).  Measurements for a reader to compare; the goals it is read against are in DESIGN.md §3.9.

    python tests/bench_transformer.py kernels [--rounds 3] [--iters 5]
    python tests/bench_transformer.py split [--iters 5]
    python tests/bench_transformer.py model [--rounds 2] [--steps 3]

kernels: on R-MAT scale 22 (2^25 generated edges, datasets.rmat_graph seed 1, as tests/bench_attn.py) at H = 41, 64
and 128 with 1 head and at H = 64 with 8 heads of 8: the forward, the backward over the same CSR and the exact backward
over the transposed plan of the dot-product attention (roc_sg_attn_dot_*) and of GAT (roc_sg_attn_*), and the sum's
forward, each call timed alone with CUDA events after a 256 MB write that flushes the 50 MB L2, alternating call by
call, --iters calls per form per round over --rounds rounds.  Each line also gives the algorithmic bytes of the dot
forward, E(8H + 4) + N(8H + 8 heads), and backward, about twice that (DESIGN.md §3.9), over the median time.
split: the same calls at H = 64, 1 head and 8 x 8, each call's device time by launch from torch.profiler (a run of its
own, L2 not flushed).
model: one training step of the graph transformer and of GAT, 602-64-41 with 1 head and 602-(8x8)-41, on bench.py's
config-2 graph (R-MAT-22), alternately in each of --rounds rounds, --steps steps after one warm-up step.
Prints the card (name, power limit, max SM clock) read in the same run, then one JSON line per measurement.
"""
import argparse
import json
import os
import re
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
from roc_b200.model import Host, Model, build_gat, build_graph_transformer  # noqa: E402
from bench_inputs import bench_module, node_inputs  # noqa: E402

DEV = "cuda"
SHAPES = [(41, 1), (64, 1), (128, 1), (64, 8)]


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


def dot_bytes(n, e, h, heads):
    """algorithmic bytes: forward E(8H+4) + N(8H + 8 heads) (q and out rows, stats); backward the record pass
    N(8H + 24 heads), the destination pass E(8H+4) + N(12H + 16 heads), the source pass E(8H + 16 heads + 4) + N(16H)"""
    fwd = e * (8 * h + 4) + n * (8 * h + 8 * heads)
    bwd = n * (8 * h + 24 * heads) + e * (8 * h + 4) + n * (12 * h + 16 * heads) + e * (8 * h + 16 * heads + 4) + \
        n * 16 * h
    return fwd, bwd


def setup(n, h, heads, gen):
    def rows():
        return K.padded(n, h, fill=torch.rand((n, h), generator=gen, device=DEV) - 0.5)
    t = dict(q=rows(), k=rows(), v=rows(), g=rows(), out=K.padded(n, h), out1=K.padded(n, h), outs=K.padded(n, h),
             dq=K.padded(n, h), dk=K.padded(n, h), dv=K.padded(n, h), gin=K.padded(n, h))
    t["sc"] = torch.randn((n, 2 * heads), generator=gen, device=DEV)
    t["stats"], t["stats1"], t["sg"] = (torch.empty((n, 2 * heads), device=DEV) for _ in range(3))
    return t


def cases(plan, tr, t, heads):
    return {
        "dot_fwd": lambda: plan.attn_dot_forward(t["q"], t["k"], t["v"], heads, out=t["out"], stats=t["stats"]),
        "gat_fwd": lambda: plan.attn_forward(t["v"], t["sc"], heads, out=t["out1"], stats=t["stats1"]),
        "sum_fwd": lambda: plan.forward(t["v"], out=t["outs"]),
        "dot_bwd": lambda: plan.attn_dot_backward(t["q"], t["k"], t["v"], t["out"], t["stats"], t["g"], heads,
                                                  dq=t["dq"], dk=t["dk"], dv=t["dv"]),
        "gat_bwd": lambda: plan.attn_backward(t["v"], t["sc"], t["out1"], t["stats1"], t["g"], heads, in_grad=t["gin"],
                                              score_grad=t["sg"]),
        "dot_bwd_exact": lambda: tr.attn_dot_backward(plan, t["q"], t["k"], t["v"], t["out"], t["stats"], t["g"],
                                                      heads, dq=t["dq"], dk=t["dk"], dv=t["dv"]),
        "gat_bwd_exact": lambda: tr.attn_backward(plan, t["v"], t["sc"], t["out1"], t["stats1"], t["g"], heads,
                                                  in_grad=t["gin"], score_grad=t["sg"])}


def graph():
    re_, col = datasets.rmat_graph(22, 1 << 25, seed=1, device=DEV)
    n, e = re_.shape[0], col.shape[0]
    print(json.dumps({"graph": "R-MAT scale 22", "N": n, "E": e}), flush=True)
    return K.SgPlan(0, n - 1, 0, re_, col), K.SgTranspose(re_, col), n, e


def kernels(rounds, iters):
    plan, tr, n, e = graph()
    flush = torch.empty(64 << 20, dtype=torch.float32, device=DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    for h, heads in SHAPES:
        t = setup(n, h, heads, gen)
        cs = cases(plan, tr, t, heads)
        for fn in cs.values():
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in cs}
        for _ in range(rounds):
            for _ in range(iters):
                for k, fn in cs.items():
                    ms[k].append(timed(fn, flush))
        line = {"what": "attention_kernels", "N": n, "E": e, "H": h, "heads": heads}
        for k in cs:
            line[k] = {"median_ms": round(statistics.median(ms[k]), 3),
                       "range_ms": [round(min(ms[k]), 3), round(max(ms[k]), 3)]}
        for p in ("fwd", "bwd", "bwd_exact"):
            line["dot_over_gat_" + p] = round(line["dot_" + p]["median_ms"] / line["gat_" + p]["median_ms"], 3)
        line["dot_fwd_over_sum_fwd"] = round(line["dot_fwd"]["median_ms"] / line["sum_fwd"]["median_ms"], 3)
        fb, bb = dot_bytes(n, e, h, heads)
        line["dot_fwd_GBps"] = round(fb / line["dot_fwd"]["median_ms"] / 1e6, 1)
        line["dot_bwd_GBps"] = round(bb / line["dot_bwd"]["median_ms"] / 1e6, 1)
        print(json.dumps(line), flush=True)
        del t, cs
        torch.cuda.empty_cache()


def part_of(name):
    m = re.search(r"sg_dot_kernel<(\d+), (\d+)>", name)
    if m:
        return ("fwd", "dst", "src")[int(m.group(2))]
    if "sg_dot_fixup" in name:
        return "fwd_fixups"
    if "sg_v2_rec_kernel" in name:
        return "record"
    if "fixup" in name:
        return "sum_fixups"
    return "other"


def split(iters):
    """ms per call of each launch of the dot forward and backwards, from the CUDA kernels torch.profiler records"""
    plan, tr, n, e = graph()
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    for h, heads in ((64, 1), (64, 8)):
        t = setup(n, h, heads, gen)
        cs = cases(plan, tr, t, heads)
        line = {"what": "dot_split", "H": h, "heads": heads,
                "split": "ms per call by launch (torch.profiler, L2 not flushed)"}
        for k in ("dot_fwd", "dot_bwd", "dot_bwd_exact"):
            cs[k]()
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(iters):
                    cs[k]()
                torch.cuda.synchronize()
            parts = {}
            for ev in prof.key_averages():
                us = getattr(ev, "device_time_total", None)
                if us is None:
                    us = getattr(ev, "cuda_time_total", 0.0)
                if us:
                    p = part_of(ev.key)
                    parts[p] = parts.get(p, 0.0) + us / 1e3 / iters
            line[k] = {p: round(v, 3) for p, v in sorted(parts.items())}
        print(json.dumps(line), flush=True)
        del t, cs
        torch.cuda.empty_cache()


def model(rounds, steps):
    B = bench_module()
    re_h, col_h, label = B.make_graph(datasets, 2, 1, DEV)
    n = re_h.shape[0]
    for layers, heads in (([602, 64, 41], 1), ([602, 64, 41], 8)):
        feats, labels, mask = node_inputs(n, layers, DEV)
        forms = {"transformer": build_graph_transformer, "gat": build_gat}
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
                          "transformer_over_gat": round(statistics.median(ms["transformer"]) /
                                                        statistics.median(ms["gat"]), 3)}), flush=True)
        del feats, labels, mask
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=("kernels", "split", "model"))
    ap.add_argument("--rounds", type=int, default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    _lib.require_device()
    print(json.dumps({"card": card()}), flush=True)
    if a.mode == "kernels":
        kernels(a.rounds or 3, a.iters)
    elif a.mode == "split":
        split(a.iters)
    else:
        model(a.rounds or 2, a.steps)


if __name__ == "__main__":
    main()
