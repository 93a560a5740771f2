"""The graph transformer's dot-product attention without a GPU: the fp64 witness of tests/transformer_witness.py against
a per-edge numpy restatement of the formulas of include/roc_b200.h (forward and the three gradients, loops over rows,
edges and heads), shared and separate inputs; build_graph_transformer's op graph on a recorder and its ValueErrors; the
declared entry points; and a check that the new kernels of sg.cu compiled without local memory or a stack frame."""
import re
import shutil
import subprocess

import numpy as np
import pytest

from opgraph import Recorder
from roc_b200 import _lib
from roc_b200.model import build_graph_transformer
from transformer_witness import dot_scale, kernel_witness


def _loop_dot(row_end, col, q, k, v, gy, heads, scale):
    """out, dq, dk and dv from the formulas, one row, edge and head at a time"""
    n, h = q.shape
    f = h // heads
    out, dq, dk, dv = (np.zeros((n, h)) for _ in range(4))
    for r in range(n):
        s0, s1 = (int(row_end[r - 1]) if r else 0), int(row_end[r])
        if s0 == s1:
            continue
        for hd in range(heads):
            sl = slice(hd * f, (hd + 1) * f)
            us = [int(col[e]) for e in range(s0, s1)]
            s = np.array([scale * np.dot(q[r, sl], k[u, sl]) for u in us])
            p = np.exp(s - s.max())
            p /= p.sum()
            for pu, u in zip(p, us):
                out[r, sl] += pu * v[u, sl]
            c = np.dot(gy[r, sl], out[r, sl])
            for pu, u in zip(p, us):
                d = pu * (np.dot(gy[r, sl], v[u, sl]) - c)
                dq[r, sl] += scale * d * k[u, sl]
                dk[u, sl] += scale * d * q[r, sl]
                dv[u, sl] += pu * gy[r, sl]
    return out, dq, dk, dv


def _graph(n, edges, seed):
    """a directed multigraph with self loops, a duplicate edge and a row of degree 0 (the last)"""
    rng = np.random.RandomState(seed)
    pairs = sorted([(i, i) for i in range(n - 1)] + [tuple(rng.randint(0, n - 1, 2)) for _ in range(edges)] +
                   [(1, 2)] * 2)
    dst = np.array([p[0] for p in pairs])
    col = np.array([p[1] for p in pairs], dtype=np.uint32)
    return np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64), col


@pytest.mark.parametrize("h,heads,shared", [(1, 1, "none"), (6, 3, "none"), (8, 2, "qkv"), (5, 5, "none"),
                                            (12, 4, "kv"), (9, 1, "qk")])
def test_witness_matches_the_per_edge_formulas(h, heads, shared):
    row_end, col = _graph(9, 25, seed=h + heads)
    rng = np.random.RandomState(1)
    q, k, v, gy = (rng.standard_normal((9, h)) for _ in range(4))
    if shared == "qkv":
        k = v = q
    elif shared == "kv":
        v = k
    elif shared == "qk":
        k = q
    scale = dot_scale(h // heads)
    w = kernel_witness(row_end, col, q, k, v, gy, heads, scale)
    out, dq, dk, dv = _loop_dot(row_end, col, q, k, v, gy, heads, scale)
    np.testing.assert_allclose(w["out"], out, rtol=1e-12, atol=1e-12)
    assert not w["out"][-1].any() and not w["m"][-1].any() and not w["iz"][-1].any()
    # a shared input's gradient is the sum of its parts, held by its first name
    want = {"dq": dq, "dk": dk, "dv": dv}
    if shared == "qkv":
        want = {"dq": dq + dk + dv, "dk": None, "dv": None}
    elif shared == "kv":
        want["dk"], want["dv"] = dk + dv, None
    elif shared == "qk":
        want["dq"], want["dk"] = dq + dk, None
    for name, g in want.items():
        if g is None:
            assert w[name] is None
        else:
            np.testing.assert_allclose(w[name], g, rtol=1e-10, atol=1e-12)


def test_default_scale_is_one_rounding_of_the_double():
    for f in (1, 2, 3, 8, 41, 64, 128, 256):
        assert dot_scale(f) == float(np.float32(1.0 / np.sqrt(np.float64(f))))
    assert dot_scale(64) == 0.125 and dot_scale(3) != 1.0 / np.sqrt(3.0)


class DotRecorder(Recorder):
    """Recorder with Model.dot_attention_gather, recorded as the attention_gather it reports as, and Model.layer_norm"""

    def layer_norm(self, t, eps=1e-5):
        return self._node("layer_norm", [t], self._call("layer_norm", t, eps))

    def dot_attention_gather(self, q, k, v, heads=1, scale=None):
        return self._node("attention_gather", [q, k, v], self._call("dot_attention_gather", q, k, v, heads, scale),
                          width=self.width[q], heads=int(heads), scale=scale, dot=True)


@pytest.mark.parametrize("root_weight", [True, False])
@pytest.mark.parametrize("norm", [None, "batch", "layer_norm"])
def test_build_graph_transformer_op_graph(root_weight, norm):
    ir = DotRecorder(None)
    h = build_graph_transformer(ir, [12, 16, 6], 0.5, heads=4, root_weight=root_weight, norm=norm, activation="elu")
    kinds = [n["kind"] for n in ir.nodes]
    skip = ["linear", "add"] if root_weight else []
    hidden = ([] if norm is None else [{"batch": "batch_norm"}.get(norm, norm)]) + ["elu"]
    assert kinds == (["dropout", "linear", "linear", "linear", "attention_gather"] + skip + hidden +
                     ["dropout", "linear", "linear", "linear", "attention_gather"] + skip + ["softmax_cross_entropy"])
    attn = [n for n in ir.nodes if n["kind"] == "attention_gather"]
    assert [n["attrs"]["heads"] for n in attn] == [4, 1]
    assert [n["attrs"]["scale"] for n in attn] == [dot_scale(4), dot_scale(6)]
    for n, qkv in zip(attn, h["attn_ins"]):
        assert n["ins"] == list(qkv) and len(set(qkv)) == 3
        # q, k and v are three Linears of the same dropout output
        d = [m["ins"][0] for m in ir.nodes if m["out"] in qkv]
        assert len(d) == 3 and len(set(d)) == 1
    assert h["attn"] == [n["out"] for n in attn] and len(h["relu_outs"]) == 1
    assert len(h["bns"]) == (0 if norm is None else 1)
    if root_weight:   # the skip Linear reads the same dropout output as q, k and v
        adds = [n for n in ir.nodes if n["kind"] == "add"]
        for a, n in zip(adds, attn):
            assert a["ins"][0] == n["out"]
            skip_lin = [m for m in ir.nodes if m["out"] == a["ins"][1]][0]
            assert skip_lin["kind"] == "linear" and skip_lin["ins"] == [m["ins"][0] for m in ir.nodes
                                                                        if m["out"] == n["ins"][0]]


def test_build_graph_transformer_heads_per_layer():
    ir = DotRecorder(None)
    build_graph_transformer(ir, [12, 16, 24, 6], 0.0, heads=[2, 8])
    attn = [n for n in ir.nodes if n["kind"] == "attention_gather"]
    assert [n["attrs"]["heads"] for n in attn] == [2, 8, 1]
    assert [n["attrs"]["scale"] for n in attn] == [dot_scale(8), dot_scale(3), dot_scale(6)]


@pytest.mark.parametrize("kw", [dict(activation="tanh"), dict(norm="layer"), dict(heads=0), dict(heads=9),
                                dict(heads=3), dict(heads=2.0), dict(heads=[2, 2]), dict(heads=True)])
def test_build_graph_transformer_refusals(kw):
    with pytest.raises(ValueError):
        build_graph_transformer(DotRecorder(None), [12, 16, 6], 0.5, **kw)


def test_build_graph_transformer_refuses_wide_layers():
    with pytest.raises(ValueError):
        build_graph_transformer(DotRecorder(None), [12, 264, 6], 0.5, heads=8)


def test_entry_points_are_declared():
    for name in ("roc_sg_attn_dot_forward_planned", "roc_sg_attn_dot_backward_planned",
                 "roc_sg_attn_dot_backward_exact", "roc_host_dot_attention_gather"):
        assert name in _lib.PROTOTYPES
    # the op reports as attention_gather: no op kind is added
    assert len(_lib.HOST_OPS) == 17


def test_new_kernels_use_no_local_memory():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            found[name] = line
            name = None
    dot = [f for f in found if re.search(r"sg_dot_", f)]
    assert len(dot) == 8 * 3 + 8 * 2, len(dot)      # (J, pass) main kernels and (J, BIG) forward fix-ups
    for f in dot:
        assert re.search(r"STACK:0\b", found[f]) and re.search(r"LOCAL:0\b", found[f]), (f, found[f])
