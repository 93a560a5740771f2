"""bench_kernels.py — micro-benchmark of the ScatterGather kernel alone (not a pytest file).

For each (graph, H): our planned kernel vs the reference's aggre_coop_kernel (oracle/_ref, when
built) on the same HBM-resident buffers, CUDA-event timed, inputs >> L2 or L2 flushed between
iterations.  Prints one JSON line per case; used to pick kernel parameters and for profiles/.
    python tests/bench_kernels.py [--scale 22] [--hs 16,64,128,256] [--iters 10]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref  # noqa: E402
from roc_b200 import datasets  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402


def sg_bytes(n, e, h):
    return e * (4 * h + 4) + n * (4 * h + 8)


def timeit(fn, iters, flush):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--hs", default="16,41,64,128,256")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--graph", default="rmat", choices=["rmat", "reddit", "products"])
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--epi", type=int, default=0, help="ROC_SG_EPI_* flags for our kernel")
    ap.add_argument("--zero-rows", type=float, default=0.0, help="fraction of input rows set to zero")
    ap.add_argument("--scale-in", type=float, default=1.0, help="multiply the input (e.g. 1e-30 for tiny values)")
    a = ap.parse_args()
    dev = "cuda"
    if a.graph == "rmat":
        re, col = datasets.rmat_graph(a.scale, 1 << (a.scale + 3), seed=1, device=dev)
    elif a.graph == "reddit":      # BASELINE configs[4] shape: 233K vertices, ~114M edges
        re, col = datasets.powerlaw_graph(232965, 57_500_000, alpha=1.3, seed=1, device=dev)
    else:                          # configs[2] shape: 2.45M vertices, ~62M edges
        re, col = datasets.powerlaw_graph(2449029, 30_000_000, alpha=1.6, seed=1, device=dev)
    n, e = re.shape[0], col.shape[0]
    deg = torch.diff(re, prepend=torch.zeros(1, dtype=re.dtype, device=dev))
    plan = K.SgPlan(0, n - 1, 0, re, col)
    info = plan.info()
    print(json.dumps({"graph": a.graph, "N": n, "E": e, "max_deg": int(deg.max()), "plan": info}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)     # 256 MB > 50 MB L2
    use_ref = ref.available() and not a.no_ref
    if use_ref:
        rp, es = ref.edge_structs(col, re, 0, 0)
    for h in [int(v) for v in a.hs.split(",")]:
        x = K.padded(n, h, dev)
        x.copy_((torch.rand((n, h), device=dev) - 0.5) * a.scale_in)
        if a.zero_rows > 0:
            x[torch.rand(n, device=dev) < a.zero_rows] = 0
        out = K.padded(n, h, dev)
        plan.reserve(h)
        ms = timeit(lambda: plan.forward(x, out=out, epilogue=a.epi), a.iters, flush)
        rec = {"H": h, "ours_ms": ms, "ours_GBps": sg_bytes(n, e, h) / ms / 1e6, "ours_Gedges_s": e / ms / 1e6}
        if use_ref and h <= 512:
            xd = x.contiguous()
            od = torch.empty((n, h), device=dev)
            rms = timeit(lambda: ref.scatter_gather(0, n - 1, 0, rp, es, xd, out=od), max(2, a.iters // 3), flush)
            rec.update({"ref_ms": rms, "ref_GBps": sg_bytes(n, e, h) / rms / 1e6, "speedup": rms / ms})
            got = plan.forward(xd, out=torch.empty((n, h), device=dev))
            rec["max_rel_diff_vs_ref"] = float(((got - od).abs() / (od.abs() + 1e-3)).max())
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
