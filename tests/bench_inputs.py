"""bench.py's workload for tools that rebuild it outside bench.py (not a pytest file): bench.py loaded as a module, and
the synthetic node data of bench.run_ours, generated the same way from the same seeds."""
import importlib.util
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bench_module():
    spec = importlib.util.spec_from_file_location("roc_bench", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def node_inputs(nloc, layers, dev, rank=0):
    """The pinned host features [nloc][layers[0]] (uniform in [-1, 1), drawn on `dev`), the int32 class labels and the
    int32 0/1/2 mask (train / val / test, about 66 / 10 / 24 %) of bench.run_ours on rank `rank`."""
    g = torch.Generator(device="cpu"); g.manual_seed(1000 + rank)
    feats = torch.empty((nloc, layers[0]), dtype=torch.float32, pin_memory=True)
    dg = torch.Generator(device=dev); dg.manual_seed(1000 + rank)
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
    return feats, labels, mask
