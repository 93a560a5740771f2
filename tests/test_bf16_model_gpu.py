"""GPU suite: models on bf16 input features.  Every builder with features="bfloat16" against its fp32 twin whose input
holds the same bf16-rounded values: the bf16 kernels widen X exactly, so three training steps must give byte-identical
logits, every dW, every weight after Adam and the metric counts (not the loss, an atomically ordered sum), with fusion
on and off, and in infer mode.  Then the data paths (set_tensor / get_tensor in fp32 and raw bits, a load_features
round trip) and the refusals: every op but linear and dropout refuses a bf16 input at init, naming itself."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from roc_b200 import _lib, bf16, datasets
from roc_b200.model import (Host, Model, build_gat, build_gcn, build_gcn_weighted, build_sage_mean,
                            build_sage_pool)

pytestmark = pytest.mark.gpu
N, PAIRS = 700, 3000
BUILDERS = {
    "gcn2": lambda m, f, d: build_gcn(m, [40, 24, 7], d, features=f),
    "gcn4_residual": lambda m, f, d: build_gcn(m, [40, 24, 16, 12, 7], d, features=f),
    "sage_mean": lambda m, f, d: build_sage_mean(m, [40, 24, 7], d, features=f),
    "sage_pool": lambda m, f, d: build_sage_pool(m, [40, 24, 7], d, features=f),
    "gat": lambda m, f, d: build_gat(m, [40, 24, 7], d, features=f),
    "gcn_weighted": lambda m, f, d: build_gcn_weighted(m, [40, 24, 7], d, EDGE_W, features=f),
}


def graph():
    row_end, col = datasets.uniform_graph(N, PAIRS, seed=3)
    return row_end.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


ROW_END, COL = graph()
EDGE_W = datasets.gcn_edge_weights(ROW_END, COL, np.random.RandomState(4).uniform(0.2, 3.0, size=COL.shape[0]))
FEATS, LABELS, MASK = (t.numpy() for t in datasets.node_data(N, 40, 7, seed=2))


def run(name, features, fuse, weights=None):
    """three training steps, then an infer-mode forward; returns everything to compare and the initial weights"""
    host = Host(0, 0, 1)
    host.graph_from_arrays(ROW_END, COL)
    m = Model(host, seed=1)
    if not fuse:
        m.set_fusion(False)
    hd = BUILDERS[name](m, features, 0.5)
    if weights is not None:
        for p, w in enumerate(weights):
            m.set_parameter(p, w)
    w0 = [m.get_parameter(p) for p in range(m.num_parameters())]
    if features == "bfloat16":
        assert m.is_bf16(hd["input"])
        m.set_tensor(hd["input"], FEATS)                 # rounded on the device
    else:
        m.set_tensor(hd["input"], bf16.round_f32(FEATS))  # the same values, rounded on the host
    m.set_labels(hd["label"], LABELS)
    m.set_tensor(hd["mask"], MASK.astype(np.int32))
    out = []
    for _ in range(3):
        m.train_mode(); m.zero_gradients(); m.forward()
        logits = m.get_tensor(hd["logits"])
        m.backward()
        dw = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
        w = [m.get_parameter(p) for p in range(m.num_parameters())]
        met = {k: v for k, v in m.metrics().items() if "Loss" not in k}
        out.append((logits, dw, w, met))
    m.infer_mode(); m.forward()
    out.append(m.get_tensor(hd["logits"]))
    ops = m.op_info()
    host.close()
    return out, w0, ops


def same_bytes(a, b):
    return np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


@pytest.mark.parametrize("fuse", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("name", list(BUILDERS))
def test_builder_matches_its_fp32_twin_bit_for_bit(name, fuse):
    got, w0, ops = run(name, "bfloat16", fuse)
    want, _, _ = run(name, "float32", fuse, weights=w0)
    for step in range(3):
        (lb, dwb, wb, mb), (lf, dwf, wf, mf) = got[step], want[step]
        assert same_bytes(lb, lf), "step %d: logits differ" % step
        for p in range(len(dwb)):
            assert same_bytes(dwb[p], dwf[p]), "step %d: dW[%d] differs" % (step, p)
            assert same_bytes(wb[p], wf[p]), "step %d: W[%d] after Adam differs" % (step, p)
        assert mb == mf, (step, mb, mf)
    assert same_bytes(got[3], want[3]), "infer-mode logits differ"
    drops = [o for o in ops if o["kind"] == "dropout"]
    if fuse and name in ("gcn2", "gat", "gcn_weighted"):   # the first dropout's one consumer is a linear
        assert drops[0]["fusedInto"] >= 0, drops       # the first dropout reads bf16 inside the linear's GEMM
    else:
        assert drops[0]["fusedInto"] < 0, drops        # roc_dropout_fwd_bf16 writes the dropped copy


# ------------------------------------------------------------------------------------------------- data paths ---
def small_model():
    host = Host(0, 0, 1)
    host.graph_from_arrays(ROW_END, COL)
    return host, Model(host, seed=1)


def test_set_and_get_tensor():
    host, m = small_model()
    x = m.create_node_tensor(13, dtype="bfloat16")
    assert m.tensor_shape(x) == (N, 13, 16)
    f = np.random.RandomState(0).standard_normal((N, 13)).astype(np.float32) * 100
    m.set_tensor(x, f)
    assert same_bytes(m.get_tensor(x), bf16.round_f32(f))
    assert np.array_equal(m.get_tensor(x, raw=True), bf16.to_bits(f))
    t = torch.from_numpy(-f).to(torch.bfloat16)                 # raw bf16 rows
    m.set_tensor(x, t)
    assert np.array_equal(m.get_tensor(x, raw=True), t.view(torch.int16).numpy().view(np.uint16))
    with pytest.raises(_lib.RocError):
        m.get_tensor(x, grad=True)
    host.close()


def test_load_features_round_trip(tmp_path):
    f = np.random.RandomState(1).uniform(-3, 3, (N, 40)).astype(np.float32)
    prefix = str(tmp_path / "g")
    f.tofile(prefix + ".feats.bin")
    host, m = small_model()
    x = m.create_node_tensor(40, dtype="bfloat16")
    m.load_features(x, prefix)
    assert np.array_equal(m.get_tensor(x, raw=True), bf16.to_bits(f))
    host.close()


# -------------------------------------------------------------------------------------------------- refusals ---
REFUSED = {
    "scatter_gather": "m.scatter_gather(x)",
    "scatter_gather(max)": "m.scatter_gather(x, _lib.AGGR_MAX)",
    "scatter_gather(min)": "m.scatter_gather(x, _lib.AGGR_MIN)",
    "scatter_gather(weighted)": "m.scatter_gather(x, weights=m.create_edge_tensor(1))",
    "attention_gather": "m.attention_gather(x, m.linear(x, 2), 1)",
    "indegree_norm": "m.indegree_norm(x)",
    "relu": "m.relu(x)",
    "sigmoid": "m.sigmoid(x)",
    "add": "m.add(x, m.linear(x, 8))",
    "softmax_cross_entropy": "m.softmax_cross_entropy(x, m.create_node_tensor(8), m.create_node_tensor(1, is_int=True))",
}


@pytest.mark.parametrize("op", list(REFUSED))
def test_other_ops_refuse_a_bf16_input(op):
    prog = "\n".join([
        "import sys; sys.path.insert(0, %r)" % ROOT, "import numpy as np",
        "from roc_b200 import _lib", "from roc_b200.model import Host, Model",
        "host = Host(0, 0, 1)",
        "host.graph_from_arrays(np.array([2, 4, 6, 8], dtype=np.uint64), "
        "np.array([0, 1, 0, 1, 2, 3, 2, 3], dtype=np.uint32))",
        "m = Model(host, seed=1)",
        "x = m.create_node_tensor(8, dtype='bfloat16')",
        REFUSED[op],
        "m.adam()",
        "m.init()",
        "print('initialised')"])
    p = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ))
    assert p.returncode != 0 and "initialised" not in p.stdout
    assert "%s cannot read a bf16 tensor" % op in p.stderr, p.stderr[-2000:]
