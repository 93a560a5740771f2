"""bench_multilabel.py — the multi-label sigmoid cross-entropy head against the softmax head (not a pytest file).

    python tests/bench_multilabel.py kernels [--rounds 3] [--iters 5] [--widths 41,112]
    python tests/bench_multilabel.py model [--rounds 2] [--steps 3]

kernels: at N = 4,194,304 rows, per width C, four calls alternating call by call, each timed alone with CUDA events
after a 256 MB write that flushes the 50 MB L2, --iters calls per form per round over --rounds rounds: the sigmoid loss
plain and with the fused norm (roc_sigmoid_xent_bwd, with metrics, as the host calls it) and the softmax loss with
class-index labels plain and fused (roc_softmax_xent_bwd_idx / _norm).  Reports the median and the range, the bytes
each call must move and their share of the 3.35 TB/s HBM3 bound of the H100 SXM data sheet at the median:
  sigmoid  N (4 ldZ + 4 ldG + 4 W + 4) (+ 8 N fused)      softmax  N (4 ldZ + 4 ldG + 4 + 4) (+ 8 N fused)
with ld = C rounded up to 4 and W = ceil(C / 32) label words per row.
model: one training step of GCN 602-64-112 on R-MAT-22 (bench.py's config-2 graph) with each head, built alternately
in each of --rounds rounds, --steps steps after one warm-up step; the multi-labels are random at a 10 % positive rate.
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
from roc_b200.model import Host, Model, build_gcn  # noqa: E402
from bench_inputs import bench_module, node_inputs  # noqa: E402

PEAK_GBS = 3350.0
DEV = "cuda"
N = 4194304


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


def kernels(rounds, iters, widths):
    flush = torch.empty(64 << 20, dtype=torch.float32, device=DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    mask = torch.randint(0, 3, (N,), generator=gen, device=DEV, dtype=torch.int32)
    row_end = torch.cumsum(torch.randint(1, 40, (N,), generator=gen, device=DEV), 0)
    for c in widths:
        ld, w = (c + 3) // 4 * 4, (c + 31) // 32
        z = K.padded(N, c, fill=torch.randn((N, c), generator=gen, device=DEV) * 3)
        g = K.padded(N, c)
        bits = torch.randint(-(1 << 31), 1 << 31, (N, w), generator=gen, device=DEV, dtype=torch.int64).to(torch.int32)
        idx = torch.randint(0, c, (N,), generator=gen, device=DEV, dtype=torch.int32)
        ml = torch.zeros(18, dtype=torch.float64, device=DEV)
        perf = torch.zeros(7, dtype=torch.int32, device=DEV)
        st = K._stream()

        def sig(fused):
            _lib.lib.roc_sigmoid_xent_bwd(N, c, K._ptr(z), ld, K._ptr(bits), w, K._ptr(mask), K._ptr(g), ld,
                                          K._ptr(row_end) if fused else None, 0, K._ptr(ml), st)

        def soft(fused):
            if fused:
                _lib.lib.roc_softmax_xent_bwd_norm(N, c, K._ptr(z), ld, None, 0, K._ptr(idx), K._ptr(mask), K._ptr(g),
                                                   ld, K._ptr(row_end), 0, K._ptr(perf), st)
            else:
                _lib.lib.roc_softmax_xent_bwd_idx(N, c, K._ptr(z), ld, K._ptr(idx), K._ptr(mask), K._ptr(g), ld,
                                                  K._ptr(perf), st)

        base = {"sigmoid": N * (8 * ld + 4 * w + 4), "softmax": N * (8 * ld + 8)}
        cases = {"sigmoid": lambda: sig(False), "sigmoid_norm": lambda: sig(True),
                 "softmax": lambda: soft(False), "softmax_norm": lambda: soft(True)}
        nbytes = {k: base[k.split("_")[0]] + (8 * N if k.endswith("norm") else 0) for k in cases}
        for fn in cases.values():
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in cases}
        for _ in range(rounds):
            for _ in range(iters):
                for k, fn in cases.items():
                    ms[k].append(timed(fn, flush))
        line = {"what": "loss_kernel", "N": N, "C": c, "ld": ld}
        for k in cases:
            med = statistics.median(ms[k])
            line[k] = {"median_ms": round(med, 4), "range_ms": [round(min(ms[k]), 4), round(max(ms[k]), 4)],
                       "bytes": nbytes[k], "bound_ms": round(nbytes[k] / PEAK_GBS / 1e6, 4),
                       "share_of_hbm_bound": round(nbytes[k] / med / 1e6 / PEAK_GBS, 3)}
        print(json.dumps(line), flush=True)
        del z, g, bits, idx
        torch.cuda.empty_cache()


def model(rounds, steps):
    B = bench_module()
    re_h, col_h, label = B.make_graph(datasets, 2, 1, DEV)
    n = re_h.shape[0]
    layers = [602, 64, 112]
    feats, labels, mask = node_inputs(n, layers, DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(2)
    multi = (torch.rand((n, layers[-1]), generator=gen, device=DEV) < 0.1).cpu().numpy()
    ms = {"softmax": [], "sigmoid": []}
    last = {}
    for _ in range(rounds):
        for head in ("softmax", "sigmoid"):
            host = Host(0, 0, 1)
            host.graph_from_arrays(re_h, col_h)
            m = Model(host, seed=1)
            h = build_gcn(m, layers, B.DROPOUT, lr=B.LR, weight_decay=B.WD, loss=head)
            m.set_tensor_from_host_ptr(h["input"], feats.data_ptr())
            if head == "softmax":
                m.set_labels(h["label"], labels.numpy())
            else:
                m.set_multilabels(h["label"], multi)
            m.set_tensor(h["mask"], mask.numpy())
            m.train_epoch()
            torch.cuda.synchronize()
            t0 = time.time()
            for _ in range(steps):
                m.train_epoch()
            host.synchronize()
            ms[head].append((time.time() - t0) * 1e3 / steps)
            last[head] = m.metrics()["trainLoss"]
            host.close()
            torch.cuda.empty_cache()
    print(json.dumps({"what": "train_step", "model": "gcn", "layers": layers, "graph": label, "steps": steps,
                      "ms_per_step": {k: [round(x, 2) for x in v] for k, v in ms.items()},
                      "median_ms": {k: round(statistics.median(v), 2) for k, v in ms.items()},
                      "sigmoid_over_softmax": round(statistics.median(ms["sigmoid"]) / statistics.median(ms["softmax"]),
                                                    3),
                      "last_train_loss": last}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=("kernels", "model"))
    ap.add_argument("--rounds", type=int, default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--widths", default="41,112")
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
