"""APPNP and GCNII without a GPU: the builders' op sequences and fp32 coefficients, their ValueErrors, an fp64
dense-matrix restatement of both models against the recorded op graph run by the fp64 interpreter of
appnp_witness.py, and a check that the new kernels of sg.cu / elementwise.cu compiled without local memory."""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from appnp_witness import witness
from opgraph import Recorder
from roc_b200 import _lib
from roc_b200.model import Model, build_appnp, build_gcnii, fp32, gcnii_beta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def appnp_ir(K=3, alpha=0.1, layers=(24, 16, 12), **kw):
    ir = Recorder(None)
    h = build_appnp(ir, list(layers), 0.0, K=K, alpha=alpha, **kw)
    return ir, h


def gcnii_ir(depth=4, alpha=0.1, theta=0.5, layers=(24, 16, 12), rate=0.0, **kw):
    ir = Recorder(None)
    h = build_gcnii(ir, list(layers), rate, depth, alpha=alpha, theta=theta, **kw)
    return ir, h


def kinds(ir):
    return [n["kind"] for n in ir.nodes]


# ---------------------------------------------------------------------------------------------- the builders ---
def test_appnp_ops_and_coefficients():
    ir, h = appnp_ir(K=3, alpha=0.15)
    mlp = ["dropout", "linear", "relu", "dropout", "linear"]
    hop = ["indegree_norm", "scatter_gather", "indegree_norm", "scaled_add"]
    assert kinds(ir) == mlp + hop * 3 + ["softmax_cross_entropy"]
    c = (float(np.float32(1.0 - 0.15)), float(np.float32(0.15)))
    assert h["coefficients"] == c
    adds = [n for n in ir.nodes if n["kind"] == "scaled_add"]
    assert [n["out"] for n in adds] == h["hops"] and h["logits"] == h["hops"][-1]
    for n in adds:
        assert n["ins"][1] == h["h"] and (n["attrs"]["alpha"], n["attrs"]["beta"]) == c
    # each hop normalises the previous hop's output (the MLP's for the first)
    norms = [n for n in ir.nodes if n["kind"] == "indegree_norm"][::2]
    assert [n["ins"][0] for n in norms] == [h["h"]] + h["hops"][:-1]
    # a two-layer list is one Linear and no relu
    ir2, _ = appnp_ir(K=1, layers=(8, 4))
    assert kinds(ir2) == ["dropout", "linear"] + hop + ["softmax_cross_entropy"]


def test_gcnii_ops_and_coefficients():
    ir, h = gcnii_ir(depth=3, alpha=0.2, theta=1.5)
    head = ["dropout", "linear", "relu"]
    layer = ["dropout", "indegree_norm", "scatter_gather", "indegree_norm", "scaled_add", "linear", "scaled_add",
             "relu"]
    assert kinds(ir) == head + layer * 3 + ["dropout", "linear", "softmax_cross_entropy"]
    ca = (float(np.float32(0.8)), float(np.float32(0.2)))
    cb = [(float(np.float32(1.0 - math.log(1.5 / l + 1.0))), float(np.float32(math.log(1.5 / l + 1.0))))
          for l in (1, 2, 3)]
    assert h["coefficients"] == {"alpha": ca, "beta": cb}
    adds = [n for n in ir.nodes if n["kind"] == "scaled_add"]
    for l in range(3):
        p, r = adds[2 * l], adds[2 * l + 1]
        assert p["ins"][1] == h["x0"] and (p["attrs"]["alpha"], p["attrs"]["beta"]) == ca
        lin = ir.nodes[r["layer"] - 1]
        assert lin["kind"] == "linear" and lin["ins"] == [p["out"]] and lin["attrs"]["out_dim"] == 16
        assert r["ins"] == [p["out"], lin["out"]] and (r["attrs"]["alpha"], r["attrs"]["beta"]) == cb[l]
    assert [n["out"] for n in adds[::2]] == h["hops"]
    assert gcnii_beta(0.5, 4) == math.log(0.5 / 4 + 1.0) and fp32(0.1) == float(np.float32(0.1))


def test_builders_keep_the_other_options():
    ir, _ = appnp_ir(K=2, loss="sigmoid", exact_backward=True)
    assert ir.nodes[-1]["kind"] == "sigmoid_cross_entropy" and ir.exact
    ir, _ = gcnii_ir(depth=2, features="bfloat16", loss="sigmoid")
    assert ir.nodes[-1]["kind"] == "sigmoid_cross_entropy"
    for build in (build_appnp, build_gcnii):
        with pytest.raises(TypeError):
            build(Recorder(None), [8, 4, 2], 0.0, 2, norm="batch")
        with pytest.raises(TypeError):
            build(Recorder(None), [8, 4, 2], 0.0, 2, aggregation="bfloat16")


@pytest.mark.parametrize("bad", [dict(K=0), dict(K=-3), dict(K=2.0), dict(K=True), dict(alpha=-0.01),
                                 dict(alpha=1.01), dict(alpha=float("nan")), dict(alpha="0.1")])
def test_appnp_value_errors(bad):
    with pytest.raises(ValueError):
        build_appnp(Recorder(None), [8, 4], 0.0, **bad)


@pytest.mark.parametrize("bad", [dict(depth=0), dict(depth=1.5), dict(alpha=2.0), dict(theta=0.0), dict(theta=-1.0),
                                 dict(theta=float("inf")), dict(theta=float("nan")), dict(layers=[8, 4]),
                                 dict(layers=[8, 4, 4, 2])])
def test_gcnii_value_errors(bad):
    kw = dict(depth=2, alpha=0.1, theta=0.5)
    kw.update(bad)
    layers = kw.pop("layers", [8, 4, 2])
    with pytest.raises(ValueError):
        build_gcnii(Recorder(None), layers, 0.0, **kw)


def test_scaled_add_refuses_bad_coefficients_before_the_product():
    class NoProduct:
        @property
        def h(self):
            raise AssertionError("touched the product")

    for alpha, beta in ((float("inf"), 0.1), (0.1, float("nan")), (1e39, 0.1), (0.1, -1e39)):
        with pytest.raises(ValueError):
            Model.scaled_add(NoProduct(), 0, 1, alpha, beta)


def test_host_op_kind_table():
    assert _lib.HOST_OPS[16] == "scaled_add" and len(_lib.HOST_OPS) == 17
    assert _lib.SG_EPI_NORM_OUT == 4 and _lib.SG_RED_TELE == 13


# ------------------------------------------------------------------------------ the fp64 restatement ---
def small_graph(n=60, seed=3):
    """a symmetric graph with self loops, as CSR row ends and sources"""
    rng = np.random.RandomState(seed)
    a = rng.random_sample((n, n)) < 0.08
    a = a | a.T | np.eye(n, dtype=bool)
    rows = [np.nonzero(a[v])[0] for v in range(n)]
    return np.cumsum([len(r) for r in rows]).astype(np.uint64), np.concatenate(rows).astype(np.uint32), a


def dense_appnp(adj, x, ws, K, alpha):
    """APPNP from its definition: Z_0 = H = MLP(X); Z_{k+1} = (1 - a) D^-1/2 A D^-1/2 Z_k + a H."""
    d = adj.sum(1).astype(np.float64)
    ahat = adj / np.sqrt(d)[:, None] / np.sqrt(d)[None, :]
    h = x
    for i, w in enumerate(ws):
        h = h @ w.T
        if i != len(ws) - 1:
            h = np.maximum(h, 0)
    z = h
    for _ in range(K):
        z = np.float32(1 - alpha).astype(np.float64) * (ahat @ z) + np.float32(alpha).astype(np.float64) * h
    return z


def dense_gcnii(adj, x, ws, depth, alpha, theta):
    """GCNII from its definition: X0 = relu(X W0); H_l = relu(((1 - b) I + b W_l) P_l), P_l = (1 - a) Ahat H + a X0."""
    d = adj.sum(1).astype(np.float64)
    ahat = adj / np.sqrt(d)[:, None] / np.sqrt(d)[None, :]
    a1, a2 = (np.float32(1 - alpha).astype(np.float64), np.float32(alpha).astype(np.float64))
    x0 = h = np.maximum(x @ ws[0].T, 0)
    for l in range(1, depth + 1):
        b = math.log(theta / l + 1)
        b1, b2 = np.float32(1 - b).astype(np.float64), np.float32(b).astype(np.float64)
        p = a1 * (ahat @ h) + a2 * x0
        h = np.maximum(b1 * p + b2 * (p @ ws[l].T), 0)
    return h @ ws[-1].T


def _weights(ir, rng):
    lins = [n for n in ir.nodes if n["kind"] == "linear"]
    return [rng.standard_normal((n["attrs"]["out_dim"], ir.width[n["ins"][0]])) * 0.3 for n in lins]


def test_witness_is_appnp():
    row_end, col, adj = small_graph()
    ir, h = appnp_ir(K=10, alpha=0.1, layers=(12, 9, 5))
    rng = np.random.RandomState(1)
    x = rng.standard_normal((adj.shape[0], 12))
    ws = _weights(ir, rng)
    labels, mask = rng.randint(0, 5, size=adj.shape[0]), np.zeros(adj.shape[0], np.int32)
    got = witness(ir, (row_end, col), x, labels, mask, ws)
    want = dense_appnp(adj, x, ws, 10, 0.1)
    assert np.allclose(got["logits"], want, rtol=1e-12, atol=1e-12)
    # and its gradient is the dense model's, through torch on the dense form
    wt = [torch.from_numpy(w).requires_grad_(True) for w in ws]
    d = torch.from_numpy(adj.sum(1).astype(np.float64))
    ahat = torch.from_numpy(adj.astype(np.float64)) / d.sqrt()[:, None] / d.sqrt()[None, :]
    hh = torch.relu(torch.from_numpy(x) @ wt[0].T) @ wt[1].T
    z = hh
    for _ in range(10):
        z = float(np.float32(0.9)) * (ahat @ z) + float(np.float32(0.1)) * hh
    torch.nn.functional.cross_entropy(z, torch.from_numpy(labels), reduction="sum").backward()
    for a, b in zip(got["dW"], wt):
        assert np.allclose(a, b.grad.numpy(), rtol=1e-10, atol=1e-12)


def test_witness_is_gcnii():
    row_end, col, adj = small_graph(seed=5)
    ir, h = gcnii_ir(depth=8, alpha=0.1, theta=0.5, layers=(12, 10, 4))
    rng = np.random.RandomState(2)
    x = rng.standard_normal((adj.shape[0], 12))
    ws = _weights(ir, rng)
    labels, mask = rng.randint(0, 4, size=adj.shape[0]), np.zeros(adj.shape[0], np.int32)
    got = witness(ir, (row_end, col), x, labels, mask, ws)
    assert np.allclose(got["logits"], dense_gcnii(adj, x, ws, 8, 0.1, 0.5), rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------- the new kernels ---
def test_new_kernels_use_no_local_memory():
    """every teleport instantiation of sg.cu (reduction 13) and the scaled_add kernels: no stack, no local memory"""
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
    tele = [f for f in found if re.search(r"sg_(chunk|fixup|fixup_big)_kernelI.*Li13EEEvNS_8SgParamsE$", f)]
    sa = [f for f in found if "k_scaled_add" in f]
    assert len(tele) == 42 and len(sa) == 4, (len(tele), len(sa))
    for f in tele + sa:
        assert re.search(r"STACK:0\b", found[f]) and re.search(r"LOCAL:0\b", found[f]), (f, found[f])
