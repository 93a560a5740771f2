"""bench_softmax_aggr.py — the softmax aggregation against the sum and max aggregations, and a DeeperGCN training step
against GCN (not a pytest file).  No speed target is set: these are measurements, for a reader to compare.

    python tests/bench_softmax_aggr.py kernels [--rounds 3] [--iters 5]
    python tests/bench_softmax_aggr.py model [--rounds 2] [--steps 3] [--depth 2] [--hidden 64]

kernels: on R-MAT scale 22 (2^25 generated edges, datasets.rmat_graph seed 1, bench.py's config-2 graph) at H = 41, 64
and 128: the softmax forward (training, with stats), its backward over the same CSR and its exact backward over the
transposed plan, each with and without dt, beside the sum forward and the max forward and backward.  Each call is
timed alone with CUDA events after a 256 MB write that flushes the 50 MB L2, alternating call by call, --iters calls
per form per round over --rounds rounds.  Each line also gives the softmax passes' algorithmic bytes (DESIGN.md §3.7)
over their median time.
model: one training step of build_deepergcn (602-hidden-41, --depth layers, learned t, batch norm, expansion 2) and
of build_gcn with --depth hidden layers of the same width, on the config-2 graph, alternately in each of --rounds rounds, --steps steps after one
warm-up step, with the device memory each model holds after its first step.
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
from roc_b200.model import Host, Model, build_deepergcn, build_gcn  # noqa: E402
from bench_inputs import bench_module, node_inputs  # noqa: E402

DEV = "cuda"
HS = [41, 64, 128]


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


def smx_bytes(n, e, h):
    """the algorithmic bytes of DESIGN.md §3.7: forward, backward without dt, backward with dt"""
    fwd = e * (4 * h + 4) + n * 12 * h + n * 4 * h              # gathers and ids; y, m, 1/Z out; x is the gathered row
    rec = n * (12 * h) + n * 12 * h                             # m, 1/Z, gy, y in (3 of 4 rows); {m | r | y} out
    src = e * (12 * h + 4) + n * 8 * h                          # record gathers and ids; x in, dx out
    return fwd, rec + src, rec + src + n * 4 * h + n * 4 * h    # with dt: R out, then R in


def kernels(rounds, iters):
    re_, col = datasets.rmat_graph(22, 1 << 25, seed=1, device=DEV)
    n, e = re_.shape[0], col.shape[0]
    plan, tr = K.SgPlan(0, n - 1, 0, re_, col), K.SgTranspose(re_, col)
    print(json.dumps({"graph": "R-MAT scale 22", "N": n, "E": e}), flush=True)
    flush = torch.empty(64 << 20, dtype=torch.float32, device=DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    t = torch.ones((1,), device=DEV)
    for h in HS:
        def rows():
            return K.padded(n, h, fill=torch.rand((n, h), generator=gen, device=DEV) - 0.5)
        x, g = rows(), rows()
        y, ys, ym, dx, dm = (K.padded(n, h) for _ in range(5))
        stats = torch.empty((n, 2 * h), device=DEV)
        arg = K.padded(n, h, dtype=torch.int32)
        plan.softmax_forward(x, t, out=y, stats=stats)
        plan.minmax_forward(x, _lib.AGGR_MAX, out=ym, arg=arg)
        cases = {
            "softmax_fwd": lambda: plan.softmax_forward(x, t, out=y, stats=stats),
            "sum_fwd": lambda: plan.forward(x, out=ys),
            "softmax_bwd": lambda: plan.softmax_backward(x, t, y, stats, g, dx=dx),
            "softmax_bwd_no_dt": lambda: plan.softmax_backward(x, t, y, stats, g, dx=dx, want_dt=False),
            "max_fwd": lambda: plan.minmax_forward(x, _lib.AGGR_MAX, out=ym, arg=arg),
            "softmax_bwd_exact": lambda: tr.softmax_backward(plan, x, t, y, stats, g, dx=dx),
            "softmax_bwd_exact_no_dt": lambda: tr.softmax_backward(plan, x, t, y, stats, g, dx=dx, want_dt=False),
            "max_bwd": lambda: plan.minmax_backward(g, arg, out=dm)}
        for fn in cases.values():
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in cases}
        for _ in range(rounds):
            for _ in range(iters):
                for k, fn in cases.items():
                    ms[k].append(timed(fn, flush))
        line = {"what": "softmax_aggr_kernels", "N": n, "E": e, "H": h}
        for k in cases:
            line[k] = {"median_ms": round(statistics.median(ms[k]), 3),
                       "range_ms": [round(min(ms[k]), 3), round(max(ms[k]), 3)]}
        bf, bb, bbt = smx_bytes(n, e, h)
        for k, b in (("softmax_fwd", bf), ("softmax_bwd_no_dt", bb), ("softmax_bwd", bbt),
                     ("softmax_bwd_exact_no_dt", bb), ("softmax_bwd_exact", bbt)):
            line[k]["algorithmic_GBps"] = round(b / (line[k]["median_ms"] * 1e6), 1)
        line["softmax_fwd_over_sum_fwd"] = round(line["softmax_fwd"]["median_ms"] / line["sum_fwd"]["median_ms"], 3)
        print(json.dumps(line), flush=True)
        del x, g, y, ys, ym, dx, dm, stats, arg
        torch.cuda.empty_cache()


def model(rounds, steps, depth, hidden):
    B = bench_module()
    re_h, col_h, label = B.make_graph(datasets, 2, 1, DEV)
    n = re_h.shape[0]
    layers = [602, hidden, 41]
    feats, labels, mask = node_inputs(n, layers, DEV)
    forms = {"deepergcn": lambda m: build_deepergcn(m, layers, B.DROPOUT, depth, lr=B.LR, weight_decay=B.WD),
             "gcn": lambda m: build_gcn(m, [602] + [hidden] * depth + [41], B.DROPOUT, lr=B.LR, weight_decay=B.WD)}
    ms = {k: [] for k in forms}
    mem = {}
    for _ in range(rounds):
        for name, build in forms.items():
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            host = Host(0, 0, 1)
            host.graph_from_arrays(re_h, col_h)
            m = Model(host, seed=1)
            h = build(m)
            m.set_tensor_from_host_ptr(h["input"], feats.data_ptr())
            m.set_labels(h["label"], labels.numpy())
            m.set_tensor(h["mask"], mask.numpy())
            m.train_epoch()
            host.synchronize()
            mem[name] = round((free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30, 2)
            t0 = time.time()
            for _ in range(steps):
                m.train_epoch()
            host.synchronize()
            ms[name].append((time.time() - t0) * 1e3 / steps)
            host.close()
            torch.cuda.empty_cache()
    print(json.dumps({"what": "train_step", "layers": layers, "depth": depth, "graph": label, "steps": steps,
                      "ms_per_step": {k: [round(v, 2) for v in vs] for k, vs in ms.items()},
                      "median_ms": {k: round(statistics.median(vs), 2) for k, vs in ms.items()},
                      "device_memory_GiB": mem,
                      "deepergcn_over_gcn": round(statistics.median(ms["deepergcn"]) / statistics.median(ms["gcn"]),
                                                  3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=("kernels", "model"))
    ap.add_argument("--rounds", type=int, default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--depth", type=int, default=2)
    ap.add_argument("--hidden", type=int, default=64)
    a = ap.parse_args()
    _lib.require_device()
    print(json.dumps({"card": card()}), flush=True)
    if a.mode == "kernels":
        kernels(a.rounds or 3, a.iters)
    else:
        model(a.rounds or 2, a.steps, a.depth, a.hidden)


if __name__ == "__main__":
    main()
