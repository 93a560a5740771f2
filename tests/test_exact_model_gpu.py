"""Models trained with the exact backward (Model.set_exact_backward, the builders' exact_backward=True) on a small
directed multigraph with self loops, against torch fp64 autograd witnesses over three Adam steps (logits and every
dW at each step's weights), with the fusions on and off: GCN (2 and 3 layers, the latter with the residual branch),
GraphSAGE-mean, GraphSAGE-pool (max and min) and GAT (1 and 4 heads).  With the mode off the same case's dW misses
the witness, and max / min still refuse duplicate edges.  The mode refuses more than one partition."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, rel_close
from roc_b200 import _lib, datasets
from roc_b200.model import Host, Model, build_gat, build_gcn, build_sage_mean, build_sage_pool
from witness_exact import gcn_sage_witness
from witness_gat import gat_witness
from witness_pool import sage_pool_witness

pytestmark = pytest.mark.gpu

MODELS = {
    "gcn2": ((12, 16, 5), lambda m, l, ex: build_gcn(m, l, 0.0, exact_backward=ex)),
    "gcn3": ((12, 16, 16, 5), lambda m, l, ex: build_gcn(m, l, 0.0, exact_backward=ex)),
    "sage_mean": ((12, 16, 5), lambda m, l, ex: build_sage_mean(m, l, 0.0, exact_backward=ex)),
    "pool_max": ((12, 16, 5), lambda m, l, ex: build_sage_pool(m, l, 0.0, aggr=_lib.AGGR_MAX, exact_backward=ex)),
    "pool_min": ((12, 16, 5), lambda m, l, ex: build_sage_pool(m, l, 0.0, aggr=_lib.AGGR_MIN, exact_backward=ex)),
    "gat1": ((12, 16, 5), lambda m, l, ex: build_gat(m, l, 0.0, heads=1, exact_backward=ex)),
    "gat4": ((12, 16, 5), lambda m, l, ex: build_gat(m, l, 0.0, heads=4, exact_backward=ex)),
}


def directed_multigraph(layers, n=250, e=1800, seed=3):
    """Directed edges with duplicates, a heavy row, sources that feed many rows, and a self loop on every node (so
    every in-degree is at least 1)."""
    rng = np.random.RandomState(seed)
    dst = rng.randint(0, n, size=e)
    src = (rng.zipf(1.6, size=e) - 1) % n                  # a few sources with many out-edges
    src[1::4], dst[1::4] = src[0::4][:src[1::4].shape[0]], dst[0::4][:dst[1::4].shape[0]]   # duplicate edges
    dst[:120] = 9                                          # a heavy row
    dst, src = np.concatenate([dst, np.arange(n)]), np.concatenate([src, np.arange(n)])
    order = np.argsort(dst, kind="stable")                 # sources in random order within a row
    row_end = np.cumsum(np.bincount(dst[order], minlength=n)).astype(np.uint64)
    col = src[order].astype(np.uint32)
    pairs = dst.astype(np.int64) * n + src
    assert np.unique(pairs).shape[0] < pairs.shape[0]
    feats, labels, mask = datasets.node_data(n, layers[0], layers[-1], seed=seed)
    return row_end, col, feats.numpy(), labels.numpy(), mask.numpy()


def witness(kind, case, layers, w0, args):
    row_end, col, feats, labels, mask = case
    if kind.startswith("gcn") or kind == "sage_mean":
        return gcn_sage_witness("gcn" if kind.startswith("gcn") else "sage_mean", row_end, col, feats, labels, mask,
                                layers, w0)
    if kind.startswith("pool"):
        is_max = kind == "pool_max"
        _, _, chosen, pools = sage_pool_witness(row_end, col, feats, labels, mask, layers, w0, is_max)
        # where fp32 and fp64 pick different sources the candidates must tie to within rounding; the witness then
        # takes the product's choice
        for pa, wa, p64 in zip(args, chosen, pools):
            diff = pa.astype(np.int64) != wa
            if diff.any():
                cols = np.nonzero(diff)[1]
                a, b = p64[pa[diff].astype(np.int64), cols], p64[wa[diff], cols]
                assert np.abs(a - b).max() <= 1e-5 * np.abs(p64).max(), "argmax differs away from a tie"
        wl, wdw, _, _ = sage_pool_witness(row_end, col, feats, labels, mask, layers, w0, is_max,
                                          args=[a.astype(np.int64) for a in args])
        return wl, wdw
    return gat_witness(row_end, col, feats, labels, mask, layers, w0, [int(kind[3:])] * (len(layers) - 2))


def run_steps(kind, case, fuse, exact, steps=3):
    """Per Adam step: (weights before it, logits, dW, the max / min choices)."""
    layers, builder = MODELS[kind]
    row_end, col, feats, labels, mask = case
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    h = builder(m, list(layers), exact)
    m.set_tensor(h["input"], feats)
    m.set_labels(h["label"], labels)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    out = []
    for _ in range(steps):
        w0 = [m.get_parameter(p) for p in range(m.num_parameters())]
        m.train_mode(); m.zero_gradients(); m.forward()
        logits = m.get_tensor(h["logits"])
        args = [m.get_aggr_index(t) for t in h.get("pools", [])]
        m.backward()
        dw = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
        out.append((w0, logits, dw, args))
    host.close()
    return out


@pytest.mark.parametrize("fuse", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("kind", list(MODELS))
def test_exact_backward_against_torch_fp64_witness(kind, fuse):
    layers = MODELS[kind][0]
    case = directed_multigraph(layers)
    for step, (w0, logits, dw, args) in enumerate(run_steps(kind, case, fuse, exact=True)):
        wl, wdw = witness(kind, case, layers, w0, args)
        what = "%s step %d" % (kind, step)
        rel_close(logits, wl, what=what + " logits vs torch fp64")
        for p, (a, b) in enumerate(zip(dw, wdw)):
            rel_close(a, b, rtol=2e-4, atol_scale=2e-5, what=what + " dW[%d] vs torch autograd" % p)


@pytest.mark.parametrize("kind", ["gcn2", "gcn3", "sage_mean", "gat1", "gat4"])
def test_gather_backward_misses_the_witness(kind):
    """The default backward (the gather over the same CSR) trains the same case on a different gradient."""
    layers = MODELS[kind][0]
    case = directed_multigraph(layers)
    w0, logits, dw, args = run_steps(kind, case, True, exact=False, steps=1)[0]
    wl, wdw = witness(kind, case, layers, w0, args)
    rel_close(logits, wl, what=kind + " logits vs torch fp64")          # the forward is the same
    worst = max(np.abs(a - b).max() / np.abs(b).max() for a, b in zip(dw, wdw))
    assert worst > 1e-2, "%s: the gather's dW matches the directed graph's gradient (%.2e)" % (kind, worst)


def run_prog(lines):
    prog = "\n".join(["import sys; sys.path.insert(0, %r)" % ROOT, "import numpy as np",
                      "from roc_b200 import _lib",
                      "from roc_b200.model import Host, Model, build_sage_pool"] + lines)
    return subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True, timeout=300, cwd=ROOT,
                          env=dict(os.environ))


@pytest.mark.parametrize("aggr", [_lib.AGGR_MAX, _lib.AGGR_MIN])
def test_gather_backward_still_refuses_duplicate_edges(aggr):
    p = run_prog(["host = Host(0, 0, 1)",
                  "host.graph_from_arrays(np.array([3, 4, 5], dtype=np.uint64), "
                  "np.array([1, 1, 0, 1, 2], dtype=np.uint32))",
                  "m = Model(host, seed=1)",
                  "build_sage_pool(m, [4, 4, 2], 0.0, aggr=%d)" % aggr,
                  "print('built')"])
    assert p.returncode != 0 and "built" not in p.stdout
    assert "strictly increasing" in p.stderr, p.stderr[-2000:]
    p = run_prog(["host = Host(0, 0, 1)",
                  "host.graph_from_arrays(np.array([3, 4, 5], dtype=np.uint64), "
                  "np.array([1, 1, 0, 1, 2], dtype=np.uint32))",
                  "m = Model(host, seed=1)",
                  "build_sage_pool(m, [4, 4, 2], 0.0, aggr=%d, exact_backward=True)" % aggr,
                  "print('built')"])
    assert p.returncode == 0 and "built" in p.stdout, p.stderr[-2000:]


def test_exact_backward_refuses_more_than_one_partition():
    p = run_prog(["host = Host(0, 0, 2)",
                  "host.graph_from_arrays(np.array([2, 4, 6, 8], dtype=np.uint64), "
                  "np.array([0, 1, 0, 1, 2, 3, 2, 3], dtype=np.uint32))",
                  "m = Model(host, seed=1)",
                  "m.set_exact_backward(True)",
                  "print('built')"])
    assert p.returncode != 0 and "built" not in p.stdout
    assert "one partition only" in p.stderr, p.stderr[-2000:]
