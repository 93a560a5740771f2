"""bench_bf16_aggr_ops.py — the bf16 forms of the weighted, max / min and attention ScatterGathers (not a pytest file).

    python tests/bench_bf16_aggr_ops.py kernels [--rounds 3] [--iters 5] [--widths 41,64,128,256]
    python tests/bench_bf16_aggr_ops.py model [--rounds 2] [--steps 3]

kernels: on R-MAT-22 (config 2's graph), each call in its fp32 form (widened rows) and its bf16 form, alternating call
by call, each call timed alone with CUDA events after a 256 MB write that flushes the 50 MB L2, --iters calls per form
per round over --rounds rounds: the weighted forward, the edge dot, the max forward, and the attention forward and
backward with one head (and with 8 heads at H = 64).  Reports the median and the range, the algorithmic bytes per call
and their share of the 3.35 TB/s HBM3 bound of the H100 SXM data sheet at the median:
  weighted forward  E (s H + 8) + N (4 H + 8)        edge dot      E (s H + 8) + N 4 H
  max forward       E (s H + 4) + N (8 H + 8)        (s = 4 bytes per gathered fp32 value, 2 per bf16 one)
  attention forward E (s H + 12) + N (4 H + 24)      backward      E (s H + 4 H + 24) + N (s H + 12 H + 48)
(the attention counts take each gathered feature row and score once per edge, and each per-row input and output
once per row and pass; at one head.)
model: one training step of GAT, the weighted GCN and GraphSAGE-pool, 602-64-41 on R-MAT-22, with aggregation
"float32" and "bfloat16" built alternately in each of --rounds rounds, --steps steps after one warm-up step.
Prints the card (name, power limit, max SM clock) read in the same run, then one JSON line per measurement.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from roc_b200 import _lib, datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402
from roc_b200.model import Host, Model, build_gat, build_gcn_weighted, build_sage_pool  # noqa: E402
from bench_inputs import bench_module, node_inputs  # noqa: E402

PEAK_GBS = 3350.0
B = bench_module()
DEV = "cuda"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def graph():
    re_h, col_h, label = B.make_graph(datasets, 2, 1, DEV)
    return re_h, col_h, label


def timed(fn, flush):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    flush.zero_()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def report(what, h, heads, n, e, ms, nbytes, kinds):
    line = {"what": what, "H": h, "heads": heads, "N": n, "E": e, "bf16_kernels": kinds}
    for k in ("fp32", "bf16"):
        med = statistics.median(ms[k])
        line[k] = {"median_ms": round(med, 4), "range_ms": [round(min(ms[k]), 4), round(max(ms[k]), 4)],
                   "bytes": nbytes[k], "share_of_hbm_bound": round(nbytes[k] / med / 1e6 / PEAK_GBS, 3)}
    line["bf16_over_fp32"] = round(statistics.median(ms["bf16"]) / statistics.median(ms["fp32"]), 3)
    print(json.dumps(line), flush=True)


def kernels(rounds, iters, widths):
    re_h, col_h, label = graph()
    n, e = re_h.shape[0], col_h.shape[0]
    print(json.dumps({"graph": label, "N": n, "E": e}), flush=True)
    plan = K.SgPlan(0, n - 1, 0, torch.from_numpy(re_h.astype(np.int64)).to(DEV),
                    torch.from_numpy(col_h.astype(np.int32)).to(DEV))
    flush = torch.empty(64 << 20, dtype=torch.float32, device=DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    w = torch.rand(e, device=DEV, generator=gen)
    for h in widths:
        xb = torch.empty((n, (h + 7) // 8 * 8), device=DEV, dtype=torch.bfloat16)
        xb.copy_(torch.rand(xb.shape, device=DEV, generator=gen) * 2 - 1)
        xb = xb[:, :h]
        xf = K.bf16_to_f32(xb, out=K.padded(n, h))
        gy = K.padded(n, h, fill=torch.randn((n, h), device=DEV, generator=gen))
        out = K.padded(n, h)
        arg = K.padded(n, h, dtype=torch.int32)
        dw = torch.empty(e, device=DEV)
        cases = [("weighted_forward", 1, lambda x, f: (plan.weighted_forward_bf16 if f else plan.weighted_forward)(
                      x, w, out=out), lambda s: e * (s * h + 8) + n * (4 * h + 8)),
                 ("edge_dot", 1, lambda x, f: (plan.edge_dot_bf16 if f else plan.edge_dot)(gy, x, dw=dw),
                  lambda s: e * (s * h + 8) + n * 4 * h),
                 ("max_forward", 1, lambda x, f: (plan.minmax_forward_bf16 if f else plan.minmax_forward)(
                     x, _lib.AGGR_MAX, out=out, arg=arg), lambda s: e * (s * h + 4) + n * (8 * h + 8))]
        for heads in ((1, 8) if h == 64 else (1,)):
            sc = torch.randn((n, 2 * heads), device=DEV, generator=gen) * 0.5
            ao, st = plan.attn_forward(xf, sc, heads)
            ig, sg = K.padded(n, h), torch.empty((n, 2 * heads), device=DEV)
            cases += [("attn_forward", heads, lambda x, f, sc=sc, heads=heads, ao=ao, st=st:
                       (plan.attn_forward_bf16 if f else plan.attn_forward)(x, sc, heads, out=ao, stats=st),
                       lambda s: e * (s * h + 12) + n * (4 * h + 24)),
                      ("attn_backward", heads, lambda x, f, sc=sc, heads=heads, ao=ao, st=st, ig=ig, sg=sg:
                       (plan.attn_backward_bf16 if f else plan.attn_backward)(x, sc, ao, st, gy, heads, in_grad=ig,
                                                                              score_grad=sg),
                       lambda s: e * (s * h + 4 * h + 24) + n * (s * h + 12 * h + 48))]
        for what, heads, call, nbytes in cases:
            call(xf, 0)
            call(xb, 1)
            kinds = sorted({(l["kind"], l["red"]) for l in K.sg_launches()})
            ms = {"fp32": [], "bf16": []}
            for _ in range(rounds):
                for _ in range(iters):
                    ms["fp32"].append(timed(lambda: call(xf, 0), flush))
                    ms["bf16"].append(timed(lambda: call(xb, 1), flush))
            report(what, h, heads, n, e, ms, {"fp32": nbytes(4), "bf16": nbytes(2)}, kinds)
        del xb, xf, gy, out, arg, dw, cases
        torch.cuda.empty_cache()
    plan.close()


def model(rounds, steps):
    re_h, col_h, label = graph()
    n, e = re_h.shape[0], col_h.shape[0]
    layers = [602, 64, 41]
    feats, labels, mask = node_inputs(n, layers, DEV)
    ew = np.random.RandomState(1).uniform(0.05, 0.6, size=e).astype(np.float32)
    builders = {"gat": lambda m, a: build_gat(m, layers, B.DROPOUT, lr=B.LR, weight_decay=B.WD, aggregation=a),
                "gcn_weighted": lambda m, a: build_gcn_weighted(m, layers, B.DROPOUT, ew, lr=B.LR, weight_decay=B.WD,
                                                                aggregation=a),
                "sage_pool": lambda m, a: build_sage_pool(m, layers, B.DROPOUT, lr=B.LR, weight_decay=B.WD,
                                                          aggregation=a)}
    for name, build in builders.items():
        ms = {"float32": [], "bfloat16": []}
        loss = {}
        for _ in range(rounds):
            for aggr in ("float32", "bfloat16"):
                host = Host(0, 0, 1)
                host.graph_from_arrays(re_h, col_h)
                m = Model(host, seed=1)
                h = build(m, aggr)
                m.set_tensor_from_host_ptr(h["input"], feats.data_ptr())
                m.set_labels(h["label"], labels.numpy())
                m.set_tensor(h["mask"], mask.numpy())
                m.train_epoch()
                torch.cuda.synchronize()
                t0 = time.time()
                for _ in range(steps):
                    m.train_epoch()
                host.synchronize()
                ms[aggr].append((time.time() - t0) * 1e3 / steps)
                loss[aggr] = m.metrics()["trainLoss"]
                host.close()
                torch.cuda.empty_cache()
        print(json.dumps({"what": "train_step", "model": name, "layers": layers, "graph": label, "steps": steps,
                          "ms_per_step": {k: [round(x, 2) for x in v] for k, v in ms.items()},
                          "median_ms": {k: round(statistics.median(v), 2) for k, v in ms.items()},
                          "bf16_over_fp32": round(statistics.median(ms["bfloat16"]) / statistics.median(ms["float32"]), 3),
                          "last_loss": loss}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=("kernels", "model"))
    ap.add_argument("--rounds", type=int, default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--widths", default="41,64,128,256")
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
