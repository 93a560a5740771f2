"""profile_step.py — device time per kernel of one bench.py training step (not a pytest file).

    python tests/profile_step.py [--config 2] [--steps 5] [--warmup 3] [--out DIR]

Builds the workload exactly as bench.py does (same graph, model and inputs), warms it up, then runs --steps training
steps under torch.profiler with CUDA activities and prints the device time of every kernel per step, summed over its
launches, one JSON line per kernel and a total.  Run it on its own: the tracer slows the host, so its step time is not
bench.py's.  With --out the per-kernel table is also written to DIR/profile_step_cfg<N>.json.
"""
import argparse
import importlib.util
import json
import os
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def bench_module():
    spec = importlib.util.spec_from_file_location("roc_bench", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def card():
    """name, power limit and max SM clock of GPU 0 (nvidia-smi), or what torch knows"""
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
        return q or torch.cuda.get_device_name(0)
    except Exception:
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    B = bench_module()
    from roc_b200 import _lib, datasets
    from roc_b200.model import Host, Model

    _lib.require_device()
    torch.cuda.set_device(0)
    dev = "cuda:0"
    layers = B.CONFIGS[a.config]["layers"]
    re_h, col_h, glabel = B.make_graph(datasets, a.config, 1, dev)
    host = Host(0, 0, 1)
    host.graph_from_arrays(re_h, col_h)
    info = host.graph_info()
    nloc = info["rowRight"] - info["rowLeft"] + 1
    m = Model(host, seed=1)
    hnd = B.build_model(m, a.config)
    # the inputs of bench.py's run_ours (rank 0)
    g = torch.Generator(device="cpu"); g.manual_seed(1000)
    feats = torch.empty((nloc, layers[0]), dtype=torch.float32, pin_memory=True)
    dg = torch.Generator(device=dev); dg.manual_seed(1000)
    chunk = 1 << 18
    for r0 in range(0, nloc, chunk):
        r1 = min(nloc, r0 + chunk)
        feats[r0:r1].copy_(torch.rand((r1 - r0, layers[0]), device=dev, generator=dg) * 2 - 1)
    labels = torch.randint(0, layers[-1], (nloc,), generator=g, dtype=torch.int32).pin_memory()
    u = torch.rand(nloc, generator=g)
    mask = torch.full((nloc,), 2, dtype=torch.int32)
    mask[u < 0.76] = 1
    mask[u < 0.66] = 0
    mask = mask.pin_memory()
    torch.cuda.synchronize()
    m.set_tensor_from_host_ptr(hnd["input"], feats.data_ptr())
    m.set_labels(hnd["label"], labels.numpy())
    m.set_tensor_from_host_ptr(hnd["mask"], mask.data_ptr())
    for _ in range(max(a.warmup, 1)):
        m.train_epoch()
    host.synchronize()
    torch.cuda.synchronize()

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            m.train_epoch()
        host.synchronize()
        torch.cuda.synchronize()
    tot, cnt = defaultdict(float), defaultdict(int)
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = getattr(ev, "device_time", None)
        if t is None:
            t = ev.cuda_time
        tot[ev.name] += t
        cnt[ev.name] += 1
    rows = sorted(tot, key=lambda k: -tot[k])
    meta = {"card": card(), "config": a.config, "graph": glabel, "rows": nloc, "steps": a.steps}
    print(json.dumps(meta), flush=True)
    table = []
    for k in rows:
        ent = {"kernel": k, "ms_per_step": round(tot[k] / 1e3 / a.steps, 4),
               "launches_per_step": cnt[k] / a.steps}
        table.append(ent)
        print(json.dumps(ent), flush=True)
    total = sum(tot.values()) / 1e3 / a.steps
    print(json.dumps({"kernel": "TOTAL", "ms_per_step": round(total, 4)}), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "profile_step_cfg%d.json" % a.config), "w") as f:
            json.dump({"meta": meta, "kernels": table, "total_ms_per_step": total}, f, indent=1)
    host.close()


if __name__ == "__main__":
    main()
