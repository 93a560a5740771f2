"""Edge dropout of the sum ScatterGather without a GPU: the Python refusals (checked before the product is touched),
the builders' op graphs with and without edge_dropout, the restated keep mask, the fp64 witness of edge_dropout_witness
against torch autograd GCN and APPNP with PyG-style dropout of the normalised edge weights, and a check that the new
kernels of sg.cu compiled without local memory."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from edge_dropout_witness import drop_scale, edge_keep, witness
from opgraph import Recorder
from roc_b200 import _lib
from roc_b200.model import Model, build_appnp, build_gcn, fp32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class NoProduct:
    @property
    def h(self):
        raise AssertionError("touched the product")


# ----------------------------------------------------------------------------------------- the refusals ---
@pytest.mark.parametrize("kw", [dict(dropout=1.0), dict(dropout=-0.1), dict(dropout=float("nan")),
                                dict(dropout=1.5), dict(dropout=0.5, weights=3),
                                dict(dropout=0.5, aggr=_lib.AGGR_MAX), dict(dropout=0.5, aggr=_lib.AGGR_MIN),
                                dict(dropout=0.5, aggr=_lib.AGGR_AVG)])
def test_scatter_gather_refuses_before_the_product(kw):
    with pytest.raises(ValueError):
        Model.scatter_gather(NoProduct(), 0, **kw)


@pytest.mark.parametrize("rate", [1.0, -0.5, float("nan"), 2.0])
def test_builders_refuse_bad_edge_dropout(rate):
    with pytest.raises(ValueError):
        build_appnp(Recorder(None), [8, 4], 0.0, K=2, edge_dropout=rate)
    with pytest.raises(ValueError):
        build_gcn(Recorder(None), [8, 6, 4], 0.0, edge_dropout=rate)


def test_host_entry_points_are_declared():
    for name in ("roc_sg_forward_dropout_planned", "roc_sg_forward_teleport_dropout_planned",
                 "roc_sg_transpose_sum_backward_dropout", "roc_host_scatter_gather_dropout"):
        assert name in _lib.PROTOTYPES
    assert _lib.SG_RED_DROP == 32 and len(_lib.HOST_OPS) == 17


# ------------------------------------------------------------------------------------------ the builders ---
def _graph(ir):
    return [(n["kind"], n["ins"], n["out"], {k: v for k, v in n["attrs"].items()}) for n in ir.nodes]


def test_default_builders_are_unchanged():
    for build, args, kw in ((build_appnp, ([12, 8, 4], 0.5), dict(K=3)), (build_gcn, ([12, 8, 4], 0.5), {})):
        a, b = Recorder(None), Recorder(None)
        build(a, *args, **kw)
        build(b, *args, edge_dropout=0.0, **kw)
        assert _graph(a) == _graph(b)
        assert all("dropout" not in n["attrs"] for n in b.nodes if n["kind"] == "scatter_gather")


def test_every_hop_and_layer_draws_its_own_mask():
    ir = Recorder(None)
    h = build_appnp(ir, [12, 8, 4], 0.5, K=4, edge_dropout=0.3)
    sgs = [n for n in ir.nodes if n["kind"] == "scatter_gather"]
    assert len(sgs) == 4 and all(n["attrs"]["dropout"] == 0.3 for n in sgs)
    assert len({n["attrs"]["key"] for n in sgs}) == 4 and all(n["attrs"]["key"] == n["layer"] for n in sgs)
    # the same op sequence as without it
    plain = Recorder(None)
    build_appnp(plain, [12, 8, 4], 0.5, K=4)
    assert [n["kind"] for n in ir.nodes] == [n["kind"] for n in plain.nodes]
    assert h["coefficients"] == (fp32(0.9), fp32(0.1))
    ir = Recorder(None)
    build_gcn(ir, [12, 8, 6, 4], 0.5, edge_dropout=0.5)
    sgs = [n for n in ir.nodes if n["kind"] == "scatter_gather"]
    assert len(sgs) == 3 and len({n["attrs"]["key"] for n in sgs}) == 3


# --------------------------------------------------------------------------------------- the keep mask ---
def test_keep_fraction_and_independence():
    # distinct (destination, source) pairs: duplicate edges share one decision
    rng = np.random.RandomState(0)
    n = 3000
    pairs = np.unique(rng.randint(0, n * n, size=400000).astype(np.int64))
    dst, col = pairs // n, (pairs % n).astype(np.uint32)
    row_end = np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64)
    E = col.shape[0]
    for rate in (0.1, 0.5, 0.9):
        k = edge_keep(row_end, col, rate, 7, 3)
        p = 1.0 - float(np.float32(rate))
        assert abs(k.mean() - p) < 5 * np.sqrt(p * (1 - p) / E), (rate, k.mean())
    a, b, c = (edge_keep(row_end, col, 0.5, key, step) for key, step in ((7, 3), (8, 3), (7, 4)))
    assert 0.4 < (a != b).mean() < 0.6 and 0.4 < (a != c).mean() < 0.6
    assert drop_scale(0.5) == 2.0 and drop_scale(0.1) == float(np.float32(1) / np.float32(0.9))


# ------------------------------------------------------------------------------- the fp64 restatement ---
def small_graph(n=60, seed=3):
    """a symmetric graph with self loops, as CSR row ends and sources"""
    rng = np.random.RandomState(seed)
    a = rng.random_sample((n, n)) < 0.08
    a = a | a.T | np.eye(n, dtype=bool)
    rows = [np.nonzero(a[v])[0] for v in range(n)]
    return np.cumsum([len(r) for r in rows]).astype(np.uint64), np.concatenate(rows).astype(np.uint32)


def _weights(ir, rng):
    lins = [n for n in ir.nodes if n["kind"] == "linear"]
    return [rng.standard_normal((n["attrs"]["out_dim"], ir.width[n["ins"][0]])) * 0.3 for n in lins]


def _pyg_propagate(row_end, col, z, edge_mask, rate):
    """PyG's gcn_norm then F.dropout on the edge weights (with a given mask): sum over edges of w'_e z[src]"""
    n = row_end.shape[0]
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)])).astype(np.float64)
    dst = torch.from_numpy(np.repeat(np.arange(n), deg.astype(np.int64)))
    src = torch.from_numpy(col.astype(np.int64))
    w = torch.from_numpy(1.0 / np.sqrt(deg))[dst] * torch.from_numpy(1.0 / np.sqrt(deg))[src]
    w = w * torch.from_numpy(edge_mask.astype(np.float64)) * drop_scale(rate)
    return torch.zeros_like(z).index_add(0, dst, z[src] * w.unsqueeze(1))


@pytest.mark.parametrize("rate", [0.5, 0.1])
def test_witness_is_pyg_appnp(rate):
    row_end, col = small_graph()
    n, K, step = row_end.shape[0], 10, 2
    ir = Recorder(None)
    build_appnp(ir, [12, 9, 5], 0.0, K=K, alpha=0.1, edge_dropout=rate)
    rng = np.random.RandomState(1)
    x = rng.standard_normal((n, 12))
    ws = _weights(ir, rng)
    labels, mask = rng.randint(0, 5, size=n), np.zeros(n, np.int32)
    got = witness(ir, (row_end, col), x, labels, mask, ws, step=step)
    sgs = [nd for nd in ir.nodes if nd["kind"] == "scatter_gather"]
    assert sorted(got["masks"]) == [nd["layer"] for nd in sgs]
    wt = [torch.from_numpy(w).requires_grad_(True) for w in ws]
    hh = torch.relu(torch.from_numpy(x) @ wt[0].T) @ wt[1].T
    z = hh
    for nd in sgs:
        keep = edge_keep(row_end, col, rate, nd["attrs"]["key"], step)
        z = float(fp32(0.9)) * _pyg_propagate(row_end, col, z, keep, rate) + float(fp32(0.1)) * hh
    assert np.allclose(got["logits"], z.detach().numpy(), rtol=1e-12, atol=1e-12)
    torch.nn.functional.cross_entropy(z, torch.from_numpy(labels), reduction="sum").backward()
    for a, b in zip(got["dW"], wt):
        assert np.allclose(a, b.grad.numpy(), rtol=1e-10, atol=1e-12)
    # the masks of different hops differ, and infer mode drops nothing
    assert len({m.tobytes() for m in got["masks"].values()}) == K
    plain = witness(ir, (row_end, col), x, labels, mask, ws, step=step, training=False)
    assert not plain["masks"]


def test_witness_is_pyg_gcn():
    row_end, col = small_graph(seed=5)
    n, rate, step = row_end.shape[0], 0.5, 3
    ir = Recorder(None)
    build_gcn(ir, [12, 10, 4], 0.0, edge_dropout=rate)
    rng = np.random.RandomState(2)
    x = rng.standard_normal((n, 12))
    ws = _weights(ir, rng)
    labels, mask = rng.randint(0, 4, size=n), np.zeros(n, np.int32)
    got = witness(ir, (row_end, col), x, labels, mask, ws, step=step)
    sgs = [nd for nd in ir.nodes if nd["kind"] == "scatter_gather"]
    wt = [torch.from_numpy(w).requires_grad_(True) for w in ws]
    h = torch.from_numpy(x)
    for i, nd in enumerate(sgs):
        keep = edge_keep(row_end, col, rate, nd["attrs"]["key"], step)
        h = _pyg_propagate(row_end, col, h @ wt[i].T, keep, rate)
        if i != len(sgs) - 1:
            h = torch.relu(h)
    assert np.allclose(got["logits"], h.detach().numpy(), rtol=1e-12, atol=1e-12)
    torch.nn.functional.cross_entropy(h, torch.from_numpy(labels), reduction="sum").backward()
    for a, b in zip(got["dW"], wt):
        assert np.allclose(a, b.grad.numpy(), rtol=1e-10, atol=1e-12)


# ------------------------------------------------------------------------------------- the new kernels ---
def test_new_kernels_use_no_local_memory():
    """every sum, exact-sum-backward and teleport instantiation with edge dropout (reductions 32, 42, 45): no stack,
    no local memory"""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    lib = os.path.join(ROOT, "roc_b200", "lib", "libroc_b200.so")
    out = subprocess.run([cuobjdump, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    found = {}
    name = None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            found[name] = line
            name = None
    drop = [f for f in found if re.search(r"sg_chunk_kernelI.*Li(32|42|45)EEEvNS_8SgParamsE$", f)]
    assert len(drop) == 42, len(drop)
    for f in drop:
        assert re.search(r"STACK:0\b", found[f]) and re.search(r"LOCAL:0\b", found[f]), (f, found[f])
