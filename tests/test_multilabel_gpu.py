"""The multi-label sigmoid cross-entropy on the GPU: roc_sigmoid_xent_bwd against the fp64 oracle of
tests/multilabel_oracle.py over a matrix of widths, row counts, pitches, masks and logits; the fused norm variant
against the plain call followed by roc_indegree_norm, bit for bit; the five model builders with loss="sigmoid" over
three Adam steps against the fp64 autograd interpreter of tests/opgraph.py (its loss node read as the sigmoid loss),
fused and unfused; the head with the other
model options; inference metrics; a learning sanity check; and the refusals."""
import ctypes as C
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from conftest import ROOT
from multilabel_oracle import micro_f1, sigmoid_xent
import opgraph
import test_opgraph_gpu as opgraph_cases
from opgraph import Recorder
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import (Host, Model, build_gat, build_gcn, build_gcn_weighted, build_sage_mean, build_sage_pool,
                            pack_multilabels)

pytestmark = pytest.mark.gpu
SPECIAL = np.array([0.0, -0.0, 1e-3, -1e-3, 1.0, -1.0, 20.0, -20.0, 100.0, -100.0, 1e30, -1e30], dtype=np.float32)
COUNTS = ("rows", "exact", "tp", "fp", "fn")


# ------------------------------------------------------------------------------------------------- the kernel ---
def _inputs(rows, c, ld, wide_bits, seed):
    """logits in a NaN-padded [rows][ld] buffer, labels packed into a [rows][W (+3)] int32 buffer, a mask over all
    four values, and a degree per row (some 0) with its rowEnd."""
    rng = np.random.RandomState(seed)
    z = (rng.randn(rows, c) * 3).astype(np.float32)
    pick = rng.rand(rows, c) < 0.25
    z[pick] = rng.choice(SPECIAL, size=int(pick.sum()))
    y = rng.rand(rows, c) < 0.3
    y[: rows // 3 + 1] = z[: rows // 3 + 1] > 0        # rows whose predictions all match, for `exact`
    mask = rng.randint(0, 4, size=rows).astype(np.int32)
    deg = rng.randint(0, 40, size=rows)
    zbuf = torch.full((rows, ld), float("nan"), device="cuda")
    zbuf[:, :c] = torch.from_numpy(z).cuda()
    bits = pack_multilabels(y)
    w = bits.shape[1]
    bbuf = torch.zeros((rows, w + (3 if wide_bits else 0)), dtype=torch.int32, device="cuda")
    bbuf[:, :w] = torch.from_numpy(bits.view(np.int32)).cuda()
    row_end = torch.from_numpy(np.cumsum(deg).astype(np.int64)).cuda()
    return z, y, mask, deg, zbuf[:, :c], bbuf, torch.from_numpy(mask).cuda(), row_end


def _grad_buf(rows, c, ld):
    return torch.full((rows, ld), float("nan"), device="cuda")[:, :c]


def _check_metrics(got, want, what):
    for k in COUNTS:
        assert got[k] == want[k], (what, k, got[k], want[k])
    for s in range(3):
        a, b = got["loss"][s], want["loss"][s]
        assert abs(a - b) <= 1e-6 * abs(b) + 1e-30, (what, s, a, b)


@pytest.mark.parametrize("c", [1, 3, 5, 8, 31, 32, 33, 41, 64, 112, 128, 129, 256, 500])
@pytest.mark.parametrize("pitch", ["round4", "wide"])
def test_kernel_matches_the_oracle(c, pitch):
    ld = (c + 3) // 4 * 4 + (0 if pitch == "round4" else 5)     # wide: not a multiple of 4, the scalar path
    for rows in (1, 7, 1000, 65537):
        what = "C=%d ld=%d rows=%d" % (c, ld, rows)
        z, y, mask, deg, dz, bits, dmask, row_end = _inputs(rows, c, ld, pitch == "wide", seed=rows + c)
        g = _grad_buf(rows, c, ld)
        g, m1 = K.sigmoid_xent_bwd(dz, bits, dmask, with_metrics=True, out=g)
        want_g, want_m = sigmoid_xent(z, y, mask)
        got = g.cpu().numpy().astype(np.float64)
        assert np.all(got[mask != 0] == 0.0), what
        assert np.abs(got - want_g).max() <= 1e-6, what
        _check_metrics(m1, want_m, what)
        # the same call twice: the same loss bits; the same gradient bits
        g2, m2 = K.sigmoid_xent_bwd(dz, bits, dmask, with_metrics=True, out=_grad_buf(rows, c, ld))
        assert np.array_equal(np.array(m1["loss"]).view(np.uint64), np.array(m2["loss"]).view(np.uint64)), what
        assert m1 == m2 and torch.equal(g.view(torch.int32), g2.view(torch.int32)), what
        # fused norm == plain then roc_indegree_norm, bit for bit (NaN bits included: rows of degree 0)
        gf, mf = K.sigmoid_xent_bwd(dz, bits, dmask, row_end=row_end, with_metrics=True, out=_grad_buf(rows, c, ld))
        gn = K.indegree_norm(0, rows - 1, 0, row_end, g, out=_grad_buf(rows, c, ld))
        assert torch.equal(gf.view(torch.int32), gn.view(torch.int32)), what
        assert mf == m1, what
        if rows == 1000:   # without metrics: the same gradient
            g3 = K.sigmoid_xent_bwd(dz, bits, dmask, out=_grad_buf(rows, c, ld))
            assert torch.equal(g3.view(torch.int32), g.view(torch.int32)), what


def test_kernel_refuses_bad_arguments():
    rows, c = 8, 40
    z = torch.zeros((rows, 40), device="cuda")
    b = torch.zeros((rows, 2), dtype=torch.int32, device="cuda")
    mk = torch.zeros(rows, dtype=torch.int32, device="cuda")
    g = torch.zeros((rows, 40), device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731
    ok = dict(rows=rows, C=c, z=p(z), ldZ=40, b=p(b), ldB=2, mk=p(mk), g=p(g), ldG=40)

    def call(**kw):
        a = dict(ok, **kw)
        rc = _lib.lib.roc_sigmoid_xent_bwd(a["rows"], a["C"], a["z"], a["ldZ"], a["b"], a["ldB"], a["mk"], a["g"],
                                           a["ldG"], None, 0, None, None)
        torch.cuda.synchronize()
        return rc

    assert call() == _lib.ROC_OK
    for bad in (dict(C=0), dict(C=-3), dict(ldZ=39), dict(ldG=39), dict(ldB=1), dict(rows=-1), dict(z=None),
                dict(b=None), dict(mk=None), dict(g=None)):
        assert call(**bad) == _lib.ROC_ERR_INVALID, bad
    assert call(C=32, ldB=1) == _lib.ROC_OK          # W = 1 at C = 32
    assert call(rows=0) == _lib.ROC_OK


def test_kernel_at_production_rows():
    """N = 4,194,304, C = 112 (ogbn-proteins' width): gradient, counts and loss against the oracle in row chunks;
    fused == plain + roc_indegree_norm; the loss bits repeat."""
    n, c = 4194304, 112
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    z = torch.randn((n, c), generator=g, device="cuda") * 3
    y = (torch.rand((n, c), generator=g, device="cuda") < 0.1).to(torch.uint8)
    mask = torch.randint(0, 4, (n,), generator=g, device="cuda", dtype=torch.int32)
    deg = torch.randint(1, 64, (n,), generator=g, device="cuda")
    row_end = torch.cumsum(deg, 0)
    yh, maskh = y.cpu().numpy(), mask.cpu().numpy()
    bits = torch.from_numpy(pack_multilabels(yh).view(np.int32)).cuda()
    grad, m1 = K.sigmoid_xent_bwd(z, bits, mask, with_metrics=True)
    _, m2 = K.sigmoid_xent_bwd(z, bits, mask, with_metrics=True, out=torch.empty_like(z))
    assert np.array_equal(np.array(m1["loss"]).view(np.uint64), np.array(m2["loss"]).view(np.uint64))
    want = {k: [0, 0, 0] for k in COUNTS}
    want["loss"] = [0.0, 0.0, 0.0]
    step = 1 << 18
    for r0 in range(0, n, step):
        gw, mw = sigmoid_xent(z[r0:r0 + step].cpu().numpy(), yh[r0:r0 + step], maskh[r0:r0 + step])
        assert np.abs(grad[r0:r0 + step].cpu().numpy() - gw).max() <= 1e-6, r0
        for k in want:
            want[k] = [a + b for a, b in zip(want[k], mw[k])]
    _check_metrics(m1, want, "production")
    gf = K.sigmoid_xent_bwd(z, bits, mask, row_end=row_end)
    gn = K.indegree_norm(0, n - 1, 0, row_end, grad)
    assert torch.equal(gf.view(torch.int32), gn.view(torch.int32))


# ------------------------------------------------------------------------------------------------- the models ---
class Rec(Recorder):
    """Recorder that also takes the builders' bf16 feature tensors (the witness reads them widened)."""

    def create_node_tensor(self, hidden, is_int=False, dtype="float32"):
        if dtype == "float32":
            return super().create_node_tensor(hidden, is_int)
        t = self.m.create_node_tensor(hidden, dtype=dtype)
        self.width[t] = hidden
        self.leaves.append(t)
        return t

    def sigmoid_cross_entropy(self, logits, labels, mask):
        self._call("sigmoid_cross_entropy", logits, labels, mask)
        return self._node("sigmoid_cross_entropy", [logits, labels, mask], None)


def _bce_train_loss(x, labels, mask):
    """The sigmoid head's loss in fp64: the sum of binary_cross_entropy_with_logits over the train rows and all
    classes, whose gradient is the product's sigmoid(z) - y on those rows (no averaging).  labels: [N][C] 0/1."""
    train = torch.from_numpy(np.asarray(mask) == _lib.MASK_TRAIN)
    y = torch.from_numpy(np.asarray(labels, dtype=np.float64))
    return torch.nn.functional.binary_cross_entropy_with_logits(x[train], y[train], reduction="sum")


def sigmoid_witness(ir, *args, **kw):
    """opgraph.witness for a graph that ends in the sigmoid loss.  witness interprets its one loss node through the
    module's train_loss; here the node is shown to it under the loss kind it knows, and train_loss is _bce_train_loss
    for the duration of the call.  Every other node is interpreted as for any op graph."""
    nodes = [dict(n, kind="softmax_cross_entropy") if n["kind"] == "sigmoid_cross_entropy" else n for n in ir.nodes]
    shadow = types.SimpleNamespace(nodes=nodes, leaves=ir.leaves)
    saved = opgraph.train_loss
    opgraph.train_loss = _bce_train_loss
    try:
        return opgraph.witness(shadow, *args, **kw)
    finally:
        opgraph.train_loss = saved


def sym_graph():
    re_, col = datasets.rmat_graph(9, 2500, seed=3)
    return re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


def directed_graph():
    re_, col = datasets.rmat_graph(9, 2500, seed=4, directed=True)
    return re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


BUILDERS = {
    "gcn": lambda ir, **kw: build_gcn(ir, [24, 16, 12], 0.5, loss="sigmoid", **kw),
    "gcn4": lambda ir, **kw: build_gcn(ir, [24, 16, 16, 12], 0.5, loss="sigmoid", **kw),
    "sage_mean": lambda ir, **kw: build_sage_mean(ir, [24, 16, 12], 0.5, loss="sigmoid", **kw),
    "sage_pool": lambda ir, **kw: build_sage_pool(ir, [24, 16, 12], 0.5, loss="sigmoid", **kw),
    "gat": lambda ir, **kw: build_gat(ir, [24, 16, 12], 0.5, heads=2, loss="sigmoid", **kw),
    "gcn_weighted": lambda ir, **kw: build_gcn_weighted(ir, [24, 16, 12], 0.5, ir.edge_w, edge_grad=True,
                                                        loss="sigmoid", **kw),
}


def train(name, graph, fuse, steps=3, **kw):
    row_end, col = graph
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    ir = Rec(m)
    ir.edge_w = np.random.RandomState(2).uniform(0.05, 0.6, size=col.shape[0]).astype(np.float32)
    h = BUILDERS[name](ir, **kw)
    feats, labels, mask = datasets.multilabel_node_data(n, 24, 12, seed=5)
    feats, labels, mask = feats.numpy(), labels.numpy(), mask.numpy()
    m.set_tensor(h["input"], feats)
    m.set_multilabels(h["label"], labels)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    relu_of = {nd["layer"]: nd["out"] for nd in ir.nodes
               if nd["kind"] == "relu" or (nd["kind"] == "linear" and nd["attrs"]["activation"] == _lib.AC_MODE_RELU)}
    minmax = {nd["layer"]: nd["out"] for nd in ir.nodes if nd["kind"] in ("scatter_gather_max", "scatter_gather_min")}
    out = dict(ir=ir, h=h, feats=feats, labels=labels, mask=mask, info=m.op_info(), steps=[], graph=graph)
    for _ in range(steps):
        st = dict(w0=[m.get_parameter(p) for p in range(m.num_parameters())])
        m.train_mode(); m.zero_gradients(); m.forward()
        st["logits"] = m.get_tensor(h["logits"])
        st["relu"] = {l: m.get_tensor(t) > 0 for l, t in relu_of.items()}
        st["args"] = {l: m.get_aggr_index(t) for l, t in minmax.items()}
        m.backward()
        st["dw"] = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        st["train_ml"] = m.multilabel_metrics()
        m.update()
        st["w1"] = [m.get_parameter(p) for p in range(m.num_parameters())]
        out["steps"].append(st)
    m.infer_mode(); m.forward()
    out["infer_logits"] = m.get_tensor(h["logits"])
    out["infer_ml"] = m.multilabel_metrics()
    out["infer_perf"] = m.metrics()
    out["dtypes"] = {t: m.tensor_dtype(t) for t in ir.width}
    host.close()
    return out


def close(name, got, want, rtol=2e-4, atol_scale=2e-5):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    bound = rtol * np.abs(want) + atol_scale * np.abs(want).max() + 1e-30
    r = float((np.abs(got - want) / bound).max())
    assert r <= 1.0, (name, r)


def check_witness(run, feats=None):
    ir = run["ir"]
    edges = {e: ir.edge_w for e in ir.edges}
    for k, st in enumerate(run["steps"]):
        wt = sigmoid_witness(ir, run["graph"], run["feats"] if feats is None else feats, run["labels"], run["mask"],
                             st["w0"], edge_values=edges, step=k + 1, relu_masks=st["relu"], aggr_args=st["args"])
        close("step %d logits" % k, st["logits"], wt["logits"])
        for p, (a, b) in enumerate(zip(st["dw"], wt["dW"])):
            close("step %d dW%d" % (k, p), a, b)


def check_infer(run):
    """infer-mode metrics == the oracle's counts from the returned logits; metrics() carries rows / exact."""
    _, want = sigmoid_xent(run["infer_logits"], run["labels"], run["mask"])
    got = run["infer_ml"]
    _check_metrics(got, want, "infer")
    assert np.allclose(got["micro_f1"], micro_f1(want), equal_nan=True)
    p = run["infer_perf"]
    assert [p["trainAll"], p["valAll"], p["testAll"]] == got["rows"]
    assert [p["trainCorrect"], p["valCorrect"], p["testCorrect"]] == got["exact"]
    assert p["trainLoss"] == np.float32(got["loss"][0])


def same_metrics(a, b):
    """every multi-label metric equal, the loss bit for bit (micro-F1 follows from the counts)"""
    assert {k: v for k, v in a.items() if k != "micro_f1"} == {k: v for k, v in b.items() if k != "micro_f1"}
    assert np.array_equal(np.array(a["loss"]).view(np.uint64), np.array(b["loss"]).view(np.uint64))


def check_schedules_identical(a, b):
    for sa, sb in zip(a["steps"], b["steps"]):
        assert np.array_equal(sa["logits"].view(np.int32), sb["logits"].view(np.int32))
        for k in ("dw", "w1"):
            for x, y in zip(sa[k], sb[k]):
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), k
        same_metrics(sa["train_ml"], sb["train_ml"])
    same_metrics(a["infer_ml"], b["infer_ml"])
    assert a["infer_perf"] == b["infer_perf"]


@pytest.mark.parametrize("name", list(BUILDERS))
def test_builder_with_sigmoid_loss_matches_the_witness(name):
    g = sym_graph()
    fused, unfused = train(name, g, True), train(name, g, False)
    check_witness(fused)
    check_schedules_identical(fused, unfused)
    check_infer(fused)
    ir = fused["ir"]
    # these graphs are witness-checked at test_opgraph_gpu.py's bars: its coverage ledger counts their op kinds
    # (the sigmoid loss among them) as reached
    opgraph_cases.note_widths(ir)
    assert ir.nodes[-1]["kind"] == "sigmoid_cross_entropy"
    assert [i["kind"] for i in unfused["info"]][-1] == "sigmoid_cross_entropy"
    if name == "gcn":
        # GCN's last norm: its backward is done by the loss, which writes the aggregation output's gradient
        norm = next(nd for nd in ir.nodes if nd["out"] == ir.nodes[-1]["ins"][0])
        assert norm["kind"] == "indegree_norm"
        assert fused["info"][norm["layer"]]["bwdFused"] == 1
        assert fused["info"][-1]["gradOut"] == norm["ins"][0]
        assert unfused["info"][-1]["gradOut"] == -1 and unfused["info"][norm["layer"]]["bwdFused"] == 0


def test_sigmoid_head_with_exact_backward_on_a_directed_graph():
    g = directed_graph()
    fused, unfused = train("gcn", g, True, exact_backward=True), train("gcn", g, False, exact_backward=True)
    check_witness(fused)
    check_schedules_identical(fused, unfused)
    check_infer(fused)


def test_sigmoid_head_with_bf16_features():
    run = train("gcn", sym_graph(), True, features="bfloat16")
    assert run["dtypes"][run["h"]["input"]] == "bfloat16"
    widened = torch.from_numpy(run["feats"]).bfloat16().float().numpy()
    check_witness(run, feats=widened)
    check_infer(run)


def test_sigmoid_head_with_bf16_aggregation():
    """The bf16 tensors round the aggregation inputs, so no fp32 witness applies: the model trains, the loss's
    fusion holds, the inference metrics agree with the logits, and the run repeats bit for bit."""
    a = train("gcn", sym_graph(), True, aggregation="bfloat16")
    b = train("gcn", sym_graph(), True, aggregation="bfloat16")
    assert "bfloat16" in a["dtypes"].values()
    assert a["info"][-1]["gradOut"] >= 0
    for st in a["steps"]:
        assert all(np.isfinite(d).all() and np.abs(d).max() > 0 for d in st["dw"])
    check_infer(a)
    check_schedules_identical(a, b)


def test_gcn_learns_multilabel_data():
    """GCN 64-32-16 on learnable multi-label data for 30 steps: the train loss falls and the train micro-F1 rises
    above the all-negative predictor's (0).  A sanity check, not a bar.  The labels depend on each vertex's own
    features, so the graph is sparse (mean degree about 3 with the self loop) to keep that signal in the mean."""
    re_, col = datasets.uniform_graph(4096, 4096, seed=9)
    row_end, col = re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32)
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    h = build_gcn(m, [64, 32, 16], 0.0, lr=0.03, loss="sigmoid")
    feats, labels, mask = datasets.multilabel_node_data(n, 64, 16, seed=2)
    m.set_tensor(h["input"], feats.numpy())
    m.set_multilabels(h["label"], labels.numpy())
    m.set_tensor(h["mask"], mask.numpy())
    losses, f1 = [], []
    for _ in range(30):
        m.train_epoch()
        ml = m.multilabel_metrics()
        losses.append(ml["loss"][0])
        f1.append(ml["micro_f1"][0])
    host.close()
    assert losses[-1] < 0.7 * losses[0], losses
    assert f1[-1] > 0.0, f1


REFUSALS = {
    "sigmoid_on_class_labels": ("build_gcn(m, [8, 8, 5], 0.0, loss='sigmoid'); m.set_labels(1, lab)",
                                "sigmoid_cross_entropy: the label tensor has no multi-labels"),
    "softmax_on_multilabels": ("build_gcn(m, [8, 8, 5], 0.0); m.set_multilabels(1, y)",
                               "softmax_cross_entropy: the label tensor holds multi-labels"),
    "width_mismatch": ("x = m.create_node_tensor(8); y6 = m.create_node_tensor(6); mk = m.create_node_tensor(1, True);"
                       " m.sigmoid_cross_entropy(m.linear(x, 5), y6, mk)",
                       "sigmoid_cross_entropy: the label tensor's width"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_refusals(name):
    body, message = REFUSALS[name]
    prog = "\n".join([
        "import numpy as np",
        "from roc_b200 import datasets",
        "from roc_b200.model import Host, Model, build_gcn",
        "re_, col = datasets.uniform_graph(100, 300, seed=1)",
        "host = Host(0, 0, 1); host.graph_from_arrays(re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32))",
        "m = Model(host, seed=1)",
        "lab = np.zeros(100, dtype=np.int32); y = np.zeros((100, 5), dtype=np.uint8)",
        body,
        "m.set_tensor(0, np.zeros((100, 8), dtype=np.float32)); m.set_tensor(2, np.zeros(100, dtype=np.int32))",
        "m.train_epoch(); host.synchronize()",
        "print('NO REFUSAL')",
    ])
    p = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ))
    assert p.returncode != 0, p.stdout + p.stderr
    assert message in p.stderr, p.stderr[-2000:]
    assert "NO REFUSAL" not in p.stdout
