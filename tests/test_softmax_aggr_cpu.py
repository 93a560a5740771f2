"""The softmax aggregation without a GPU: the fp64 witness of tests/softmax_aggr_witness.py against a per-edge numpy
restatement of the formulas in include/roc_b200.h, the dt identity included, at several temperatures; build_deepergcn's
op graph on a recorder and its ValueErrors; the entry points declared and bound; and a check that the new kernels of
sg.cu compiled without local memory or a stack frame."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from opgraph import Recorder
from roc_b200 import _lib
from roc_b200.model import build_deepergcn
from softmax_aggr_witness import kernel_witness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _graph(n, edges, seed):
    """a directed multigraph with self loops, duplicate edges and one row of degree 0 (the last)"""
    rng = np.random.RandomState(seed)
    pairs = sorted([(i, i) for i in range(n - 1)] + [tuple(rng.randint(0, n - 1, 2)) for _ in range(edges)] +
                   [(1, 2)] * 2)
    dst = np.array([p[0] for p in pairs])
    col = np.array([p[1] for p in pairs], dtype=np.uint32)
    return np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64), col


def _loop(row_end, col, x, t, gy):
    """the formulas of include/roc_b200.h, one edge at a time: y, dx and dt (dt in its sum-of-squares form)"""
    n, h = x.shape
    y, dx, dt = np.zeros((n, h)), np.zeros((n, h)), 0.0
    for v in range(n):
        s, e = (int(row_end[v - 1]) if v else 0), int(row_end[v])
        for f in range(h):
            if s == e:
                continue
            us = [int(col[i]) for i in range(s, e)]
            z = [t * x[u, f] for u in us]
            m = max(z)
            ex = [np.exp(zi - m) for zi in z]
            Z = sum(ex)
            p = [a / Z for a in ex]
            y[v, f] = sum(pi * x[u, f] for pi, u in zip(p, us))
            g = gy[v, f]
            for pi, u in zip(p, us):
                d = x[u, f] - y[v, f]
                dx[u, f] += g * pi * (1.0 + t * d)
                dt += g * pi * d * d
    return y, dx, dt


@pytest.mark.parametrize("t", [0.0, 0.5, 1.0, -1.0, 20.0])
@pytest.mark.parametrize("h", [1, 5])
def test_witness_matches_the_per_edge_formulas(t, h):
    row_end, col = _graph(10, 30, seed=h)
    rng = np.random.RandomState(3)
    x = rng.standard_normal((10, h))
    gy = rng.standard_normal((10, h))
    w = kernel_witness(row_end, col, x, t, gy)
    y, dx, dt = _loop(row_end, col, x, t, gy)
    np.testing.assert_allclose(w["out"], y, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(w["dx"], dx, rtol=1e-10, atol=1e-12)
    assert abs(w["dt"] - dt) <= 1e-10 * max(1.0, abs(dt))
    assert not w["out"][-1].any() and not w["iz"][-1].any()          # the row of degree 0
    # the cancelling form of dt, E_p[x^2] - y^2, agrees here where the spread is not small next to y
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dst = np.repeat(np.arange(10), deg)
    ex2 = np.zeros((10, h))
    p = np.exp(t * x[col.astype(np.int64)] - (w["m"][dst])) * w["iz"][dst]
    np.add.at(ex2, dst, p * x[col.astype(np.int64)] ** 2)
    assert abs(float((gy * (ex2 - w["out"] ** 2)).sum()) - dt) <= 1e-9 * max(1.0, abs(dt))


def test_witness_limits():
    """t = 0 is the mean; a large t approaches the max, a large negative one the min"""
    row_end, col = _graph(10, 30, seed=4)
    x = np.random.RandomState(5).standard_normal((10, 3))
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dst = np.repeat(np.arange(10), deg)
    src = col.astype(np.int64)
    mean = np.zeros((10, 3))
    np.add.at(mean, dst, x[src])
    mean[deg > 0] /= deg[deg > 0, None]
    mx, mn = np.full((10, 3), -np.inf), np.full((10, 3), np.inf)
    np.maximum.at(mx, dst, x[src])
    np.minimum.at(mn, dst, x[src])
    gy = np.zeros((10, 3))
    np.testing.assert_allclose(kernel_witness(row_end, col, x, 0.0, gy)["out"], mean, rtol=1e-12, atol=1e-12)
    has = deg > 0
    np.testing.assert_allclose(kernel_witness(row_end, col, x, 1e4, gy)["out"][has], mx[has], atol=1e-3)
    np.testing.assert_allclose(kernel_witness(row_end, col, x, -1e4, gy)["out"][has], mn[has], atol=1e-3)


class SmxRecorder(Recorder):
    """Recorder with Model.softmax_gather, recorded as the attention_gather it reports as"""

    def softmax_gather(self, t, temperature=1.0, learn_temperature=False):
        if learn_temperature:
            self.params += 1
        return self._node("attention_gather", [t], self._call("softmax_gather", t, temperature, learn_temperature),
                          softmax=True, temperature=float(temperature), learn=bool(learn_temperature),
                          param=self.params - 1 if learn_temperature else None)

    def num_parameters(self):
        return self.params


@pytest.mark.parametrize("norm", ["batch", None])
@pytest.mark.parametrize("learn", [True, False])
def test_build_deepergcn_op_graph(norm, learn):
    ir = SmxRecorder(None)
    h = build_deepergcn(ir, [12, 16, 6], 0.5, 3, temperature=0.5, learn_temperature=learn, norm=norm, expansion=3)
    kinds = [n["kind"] for n in ir.nodes]
    nr = ["batch_norm", "relu"] if norm else ["relu"]
    conv = ["relu", "attention_gather", "add", "linear"] + nr + ["linear"]
    want = ["linear"] + conv + 2 * (nr + ["dropout"] + conv + ["add"]) + nr + ["dropout", "linear",
                                                                               "softmax_cross_entropy"]
    assert kinds == want
    aggs = [n for n in ir.nodes if n["kind"] == "attention_gather"]
    assert h["aggs"] == [n["out"] for n in aggs]
    assert all(n["attrs"]["temperature"] == 0.5 and n["attrs"]["learn"] == learn for n in aggs)
    assert h["temperatures"] == [n["attrs"]["param"] for n in aggs]
    assert (None in h["temperatures"]) == (not learn)
    assert len(h["bns"]) == (3 + 2 + 1 if norm else 0)    # one per conv, before layers 2 and 3, before the head
    widths = [ir.width[n["out"]] for n in ir.nodes if n["kind"] == "linear"]
    assert widths == [16] + [48, 16] * 3 + [6]
    # each aggregation reads the relu of its conv's input, and the residual adds that input
    for n in aggs:
        relu = ir.nodes[n["layer"] - 1]
        assert relu["kind"] == "relu" and n["ins"] == [relu["out"]]
        add = ir.nodes[n["layer"] + 1]
        assert add["kind"] == "add" and add["ins"] == [n["out"], relu["ins"][0]]


@pytest.mark.parametrize("args,kw", [(([12, 16], 0.5, 3), {}), (([12, 16, 6, 4], 0.5, 3), {}),
                                     (([12, 0, 6], 0.5, 3), {}), (([12, 16.0, 6], 0.5, 3), {}),
                                     (([12, 16, 6], 0.5, 0), {}), (([12, 16, 6], 0.5, 2.0), {}),
                                     (([12, 16, 6], 0.5, True), {}), (([12, 16, 6], 1.0, 3), {}),
                                     (([12, 16, 6], -0.1, 3), {}), (([12, 16, 6], 0.5, 3), dict(norm="layer")),
                                     (([12, 16, 6], 0.5, 3), dict(expansion=0)),
                                     (([12, 16, 6], 0.5, 3), dict(temperature=float("nan"))),
                                     (([12, 16, 6], 0.5, 3), dict(temperature=float("inf")))])
def test_build_deepergcn_refusals(args, kw):
    with pytest.raises(ValueError):
        build_deepergcn(SmxRecorder(None), *args, **kw)


def test_entry_points_are_declared():
    names = ("roc_sg_softmax_forward_planned", "roc_sg_softmax_backward_planned", "roc_sg_softmax_backward_exact",
             "roc_host_softmax_gather")
    for name in names:
        assert name in _lib.PROTOTYPES
    with open(os.path.join(ROOT, "include", "roc_b200.h")) as f:
        text = f.read()
    for name in names[:3]:
        assert re.search(r"\bint %s\(" % name, text)
    for name in names:
        assert getattr(_lib.lib, name) is not None
    assert len(_lib.HOST_OPS) == 17     # a mode of attention_gather, not a new op kind


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
    smx = [f for f in found if re.search(r"sg_smx_", f)]
    # 8 J x (3 passes + 2 fix-ups + the record) + dt's two sums
    assert len(smx) == 8 * 6 + 2, len(smx)
    for f in smx:
        assert re.search(r"STACK:0\b", found[f]) and re.search(r"LOCAL:0\b", found[f]), (f, found[f])
