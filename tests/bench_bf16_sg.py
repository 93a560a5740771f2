"""bench_bf16_sg.py — bf16 aggregation inputs on bench.py's graphs (not a pytest file).

    python tests/bench_bf16_sg.py [--configs 2,3,4,5] [--rounds 3] [--iters 10] [--steps 3] [--no-steps]

1. The sum ScatterGather forward at each config's aggregation widths, fp32 rows (roc_sg_forward_planned) against bf16
   rows (roc_sg_forward_planned_bf16), alternating within each of --rounds rounds, CUDA-event timed over --iters
   launches on HBM-resident operands.  Algorithmic bytes per launch: E * (s * H + 4) + N * (4 * H + 8) with s = 4 bytes
   per gathered fp32 value and 2 per bf16 one; the share of the HBM bound is those bytes at 3.35 TB/s (H100 SXM data
   sheet) over the kernel time.
2. The training step of configs 2 and 3 at full size, built as bench.py builds them, with and without
   aggregation="bfloat16": --steps steps between one pair of events after one warm-up step, alternating per round.
Prints the card (name, power limit, max SM clock) read in the same run, then one JSON line per measurement.
"""
import argparse
import importlib.util
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from roc_b200 import datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402
from roc_b200.model import Host, Model, build_gcn, build_sage_mean  # noqa: E402
from bench_inputs import bench_module, node_inputs  # noqa: E402

_spec = importlib.util.spec_from_file_location("bench_linear_cfg2", os.path.join(HERE, "bench_linear_cfg2.py"))
_b2 = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_b2)
card, PEAK_GBS = _b2.card, _b2.PEAK_GBS
B = bench_module()


def sg_bytes(n, e, h, elem):
    return e * (elem * h + 4) + n * (4 * h + 8)


def event_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def widths(cfg):
    """the widths config cfg aggregates: GCN's hidden and output widths, GraphSAGE-mean's hidden and output widths"""
    return sorted(set(B.CONFIGS[cfg]["layers"][1:]))


def sg_launches(cfg, rounds, iters):
    dev = "cuda"
    re_h, col_h, label = B.make_graph(datasets, cfg, 1, dev)
    n, e = re_h.shape[0], col_h.shape[0]
    d_re = torch.from_numpy(re_h.astype(np.int64)).to(dev)
    d_col = torch.from_numpy(col_h.astype(np.int32)).to(dev)
    plan = K.SgPlan(0, n - 1, 0, d_re, d_col)
    plan.reserve(max(widths(cfg)))
    g = torch.Generator(device=dev)
    g.manual_seed(cfg)
    for h in widths(cfg):
        xb = torch.empty((n, (h + 7) // 8 * 8), device=dev, dtype=torch.bfloat16)
        xb.copy_(torch.rand(xb.shape, device=dev, generator=g) * 2 - 1)
        xb = xb[:, :h]
        xf = K.bf16_to_f32(xb)
        out = K.padded(n, h, dev)
        ms = {"fp32": [], "bf16": []}
        for _ in range(rounds):
            ms["fp32"].append(event_ms(lambda: plan.forward(xf, out=out), iters))
            ms["bf16"].append(event_ms(lambda: plan.forward_bf16(xb, out=out), iters))
        kinds = [l["kind"] for l in K.sg_launches()]
        line = {"what": "sg_forward", "config": cfg, "graph": label, "N": n, "E": e, "H": h, "bf16_kernels": kinds}
        for k, elem in (("fp32", 4), ("bf16", 2)):
            best = min(ms[k])
            byt = sg_bytes(n, e, h, elem)
            line[k] = {"ms": [round(x, 4) for x in ms[k]], "best_ms": round(best, 4), "bytes": byt,
                       "GBps": round(byt / best / 1e6, 1), "share_of_hbm_bound": round(byt / best / 1e6 / PEAK_GBS, 3)}
        line["bf16_over_fp32"] = round(min(ms["bf16"]) / min(ms["fp32"]), 3)
        print(json.dumps(line), flush=True)
        del xb, xf, out
    plan.close()
    del d_re, d_col
    torch.cuda.empty_cache()


def step_times(cfg, rounds, steps):
    dev = "cuda"
    c = B.CONFIGS[cfg]
    re_h, col_h, label = B.make_graph(datasets, cfg, 1, dev)
    n = re_h.shape[0]
    feats, labels, mask = node_inputs(n, c["layers"], dev)
    ms = {"float32": [], "bfloat16": []}
    for _ in range(rounds):
        for aggr in ("float32", "bfloat16"):
            host = Host(0, 0, 1)
            host.graph_from_arrays(re_h, col_h)
            m = Model(host, seed=1)
            build = build_gcn if c["kind"] == "gcn" else build_sage_mean
            h = build(m, c["layers"], B.DROPOUT, lr=B.LR, weight_decay=B.WD, aggregation=aggr)
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
            loss = m.metrics()["trainLoss"]
            host.close()
            torch.cuda.empty_cache()
    print(json.dumps({"what": "train_step", "config": cfg, "graph": label, "steps": steps,
                      "ms_per_step": {k: [round(x, 2) for x in v] for k, v in ms.items()},
                      "best_ms": {k: round(min(v), 2) for k, v in ms.items()},
                      "bf16_over_fp32": round(min(ms["bfloat16"]) / min(ms["float32"]), 3), "last_loss": loss}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="2,3,4,5")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--no-steps", action="store_true")
    a = ap.parse_args()
    print(json.dumps({"card": card(), "peak_GBps": PEAK_GBS,
                      "peak_source": "H100 SXM data sheet (3.35 TB/s HBM3)"}), flush=True)
    for cfg in (int(x) for x in a.configs.split(",")):
        sg_launches(cfg, a.rounds, a.iters)
    if not a.no_steps:
        for cfg in (2, 3):
            step_times(cfg, a.rounds, a.steps)


if __name__ == "__main__":
    main()
