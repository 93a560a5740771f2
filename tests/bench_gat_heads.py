"""bench_gat_heads.py — the per-head attention-score kernels and ELU against their bytes bounds, and GAT's training step
with scores="per_head", activation="elu" against the default (not a pytest file).

    python tests/bench_gat_heads.py kernels [--rounds 3] [--iters 5]
    python tests/bench_gat_heads.py model [--rounds 2] [--steps 3]

kernels: at N = 4,194,304 rows, for (H, heads) = (64, 1), (64, 8) and (256, 8), each call timed alone with CUDA events
after a 256 MB write that flushes the 50 MB L2, alternating call by call, --iters calls per form per round over
--rounds rounds.  The forms: roc_attn_scores_fwd (bytes: read X, write S) and roc_attn_scores_bwd with dX written
(read X and dS, write dX); next to them the dense score Linear H -> 2 * heads at the same shapes (its forward, its dX
alone and its dW alone); and at H = 64, ELU and relu forward (read x, write y) and backward (read y and dY, write dX).
Bytes count the rows' float4-padded widths, and the bound is bytes over the 3.35 TB/s HBM3 of the H100 SXM data sheet.
model: one training step of GAT 602-64-41 with 1 head and of 602-(8x8)-41 on R-MAT-22 (bench.py's config-2 graph),
built with the defaults and with scores="per_head", activation="elu", alternately in each of --rounds rounds, --steps
steps after one warm-up step.
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
from roc_b200.model import Host, Model, build_gat  # noqa: E402
from bench_inputs import bench_module, node_inputs  # noqa: E402

PEAK_GBS = 3350.0
DEV = "cuda"
N = 4194304
SHAPES = [(64, 1), (64, 8), (256, 8)]


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


def run_cases(cases, nbytes, rounds, iters, flush, line):
    for fn in cases.values():
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in cases}
    for _ in range(rounds):
        for _ in range(iters):
            for k, fn in cases.items():
                ms[k].append(timed(fn, flush))
    for k in cases:
        med = statistics.median(ms[k])
        bound = nbytes[k] / PEAK_GBS / 1e6
        line[k] = {"median_ms": round(med, 4), "range_ms": [round(min(ms[k]), 4), round(max(ms[k]), 4)],
                   "bytes": nbytes[k], "bound_ms": round(bound, 4), "over_bound": round(med / bound, 3)}
    print(json.dumps(line), flush=True)


def kernels(rounds, iters):
    flush = torch.empty(64 << 20, dtype=torch.float32, device=DEV)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    for h, heads in SHAPES:
        f, s4 = h // heads, (2 * heads + 3) // 4 * 4
        x = K.padded(N, h, fill=torch.randn((N, h), generator=gen, device=DEV))
        a = torch.randn((2 * heads, f), generator=gen, device=DEV)
        ds = K.padded(N, 2 * heads, fill=torch.randn((N, 2 * heads), generator=gen, device=DEV))
        s, dx = K.padded(N, 2 * heads), K.padded(N, h)
        w, dw = torch.randn((2 * heads, h), generator=gen, device=DEV), torch.empty((2 * heads, h), device=DEV)
        cases = {"scores_fwd": lambda: K.attn_scores_fwd(x, a, heads, out=s),
                 "scores_bwd": lambda: K.attn_scores_bwd(x, a, ds, heads, dx=dx),
                 "linear_fwd": lambda: K.linear_fwd(x, w, out=s),
                 "linear_dx": lambda: K.linear_bwd_fused(x, w, None, ds, dw, dx, parts=1),
                 "linear_dw": lambda: K.linear_bwd_fused(x, w, None, ds, dw, None, parts=2)}
        xb, sb = N * h * 4, N * s4 * 4
        nbytes = {"scores_fwd": xb + sb, "scores_bwd": 2 * xb + sb, "linear_fwd": xb + sb, "linear_dx": xb + sb,
                  "linear_dw": xb + sb}
        run_cases(cases, nbytes, rounds, iters, flush, {"what": "attn_scores_kernels", "N": N, "H": h, "heads": heads})
        del x, ds, s, dx
        torch.cuda.empty_cache()
    h = 64
    x = K.padded(N, h, fill=torch.randn((N, h), generator=gen, device=DEV) * 3)
    dy = K.padded(N, h, fill=torch.randn((N, h), generator=gen, device=DEV))
    ye, yr = K.activation_fwd(x, _lib.AC_MODE_ELU), K.activation_fwd(x, _lib.AC_MODE_RELU)
    dx = K.padded(N, h)
    cases = {"elu_fwd": lambda: K.activation_fwd(x, _lib.AC_MODE_ELU),
             "relu_fwd": lambda: K.activation_fwd(x, _lib.AC_MODE_RELU),
             "elu_bwd": lambda: K.activation_bwd(ye, dy, _lib.AC_MODE_ELU, dx=None),
             "relu_bwd": lambda: K.activation_bwd(yr, dy, _lib.AC_MODE_RELU, dx=None)}
    xb = N * h * 4
    run_cases(cases, {"elu_fwd": 2 * xb, "relu_fwd": 2 * xb, "elu_bwd": 3 * xb, "relu_bwd": 3 * xb}, rounds, iters,
              flush, {"what": "activation_kernels", "N": N, "H": h})


def model(rounds, steps):
    B = bench_module()
    re_h, col_h, label = B.make_graph(datasets, 2, 1, DEV)
    n = re_h.shape[0]
    for layers, heads in (([602, 64, 41], 1), ([602, 64, 41], 8)):
        feats, labels, mask = node_inputs(n, layers, DEV)
        forms = {"default": {}, "per_head_elu": dict(scores="per_head", activation="elu")}
        ms = {k: [] for k in forms}
        for _ in range(rounds):
            for name, kw in forms.items():
                host = Host(0, 0, 1)
                host.graph_from_arrays(re_h, col_h)
                m = Model(host, seed=1)
                h = build_gat(m, layers, B.DROPOUT, heads=heads, lr=B.LR, weight_decay=B.WD, **kw)
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
        print(json.dumps({"what": "train_step", "model": "gat", "layers": layers, "heads": heads, "graph": label,
                          "steps": steps, "ms_per_step": {k: [round(v, 2) for v in vs] for k, vs in ms.items()},
                          "median_ms": {k: round(statistics.median(vs), 2) for k, vs in ms.items()},
                          "per_head_elu_over_default": round(statistics.median(ms["per_head_elu"]) /
                                                             statistics.median(ms["default"]), 3)}), flush=True)
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
    print(json.dumps({"card": card(), "peak_GBps": PEAK_GBS,
                      "peak_source": "H100 SXM data sheet (3.35 TB/s HBM3)"}), flush=True)
    if a.mode == "kernels":
        kernels(a.rounds or 3, a.iters)
    else:
        model(a.rounds or 2, a.steps)


if __name__ == "__main__":
    main()
