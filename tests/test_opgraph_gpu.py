"""Model op graphs, fused and unfused, against the fp64 interpreter of tests/opgraph.py over three Adam steps.

Model::init decides which tensors need a gradient, who overwrites a gradient and who adds to it (resetInputGrads,
set in reverse layer order by Model::backward), and the peephole fusions that reroute where a gradient is written
and switch other ops' forward or backward off (the GCN block, batch_norm or layer_norm -> relu, dropout -> linear,
the backward epilogues, the teleport of a scaled_add into a sum scatter_gather, with or without edge dropout).  This
file builds op graphs over every op kind and every attention_gather mode (GAT, GATv2's dynamic attention, the softmax
aggregation, dot-product attention) through a Recorder and checks, per case:

- the fusion report (Model.op_info) of both schedules: the hand-listed cases state it exactly, the unfused schedule
  has none;
- against the witness at each step's weights: the logits at the parity bar, every dW and every edge gradient at
  rtol 2e-4 with atol_scale 2e-5 (the bars of test_exact_model_gpu.py); a learned temperature's gradient (family dt)
  and a GATv2 a's (family da), sums over every edge and column that cancel, at rtol 1e-3 with atol_scale 1e-4 (the
  bars of test_softmax_aggr_gpu.py and test_gatv2_gpu.py);
- the batch_norm running statistics after training against the fp64 recurrence over the witness's batch statistics
  (from 0 / 1, var scaled by N / (N - 1)), at the dW bars;
- after training, an infer-mode forward: its logits against witness(training=False) at the final weights and running
  statistics, at the parity bar; equal metrics in both schedules (except trainLoss, an atomic sum), and the *All
  counts equal to the mask's counts;
- between the schedules, bit for bit: logits, dW, edge gradients, the weights after each update, the running
  statistics and the infer logits.  With set_bf16_aggregation the two schedules may store different tensors in bf16
  (a Linear's fused norm output against its own output), so there each is held to the witness with its own bf16
  values, and bit for bit only where both chose the same tensors.

Wirings that break Q7 (below) run in a subprocess: both schedules must exit non-zero at the first backward() with
the same assertion.

The rules every generated graph obeys, derived from model.cc:
- Q7 as implemented.  ScatterGather::backward and InDegreeNorm::backward assert resetInputGrads[0] before they check
  requiresGrad, so each must be the last-created consumer of its input, even when that input is a leaf.
  Dropout::backward checks requiresGrad first: the rule binds a dropout only when its input needs a gradient.  Every
  other op (batch_norm, elu, attention_scores and scaled_add among them) adds into a gradient another op already
  wrote.
- Q7 amended (mark_scaled_add_readers): a norm or dropout whose input a scaled_add also reads need not be its
  input's last reader; it adds its part through scratch.  The generator builds that shape in both creation orders.
- bf16 leaves: only linear and dropout read them.  set_bf16_aggregation: the witness takes the values of the tensors
  tensor_dtype reports as bf16, with the gradient passed straight through.
- batch_norm on any fp32 tensor, sometimes read by a relu alone (the BN-relu fusion); elu on any fp32 tensor.
- attention scores from linear(t, 2 * heads) or attention_scores(t, heads); attention dropout at rate 0 or 0.6.
- scaled_add of two different same-width tensors, coefficients (1, 1), (0.9, 0.1), (1.5, -0.5) or (0, 1).
- The teleport hop norm(sg(norm(t))) -> scaled_add(., t0) [-> norm], t0 a leaf or a tensor produced before the sum
  scatter_gather (the fusion applies), or produced after it (refused).
- Q1: without set_exact_backward, the sum, max / min and attention backwards gather over the forward CSR, the true
  adjoint only on a symmetric graph; so only exact-mode cases run on the directed multigraph.
- Max / min without the exact mode need strictly increasing sources per row (the symmetric graphs have them).
- attention_gather: scores of 2 * heads columns; heads 1, 2, 4 or 8; with heads > 1 the width is heads * F with F a
  power of two >= 4; width <= 512.
- dynamic_attention_gather and dot_attention_gather: width <= 256, heads <= 8 and heads divides the width; xr (of q,
  k and v, any) another open tensor of the same width or the first input itself.  Their backward, and
  softmax_gather's, writes an input gradient another op already wrote (or a repeated input's) through scratch and adds
  it, so they close nothing.  A dynamic gather's output and a learned temperature's gather's need a gradient even over
  leaves (their own parameter); a dot gather's only when an input does.
- softmax_gather: temperature 0, 1, -0.5 or 3, learned or constant.
- layer_norm on any fp32 tensor, sometimes read by a relu alone (the norm-relu fusion).
- Edge dropout at rate 0.1 or 0.5 on a sum scatter_gather (plain or a teleport hop's), which closes its input as
  every ScatterGather does (Q7).
- None of the five reads a bf16 tensor: only linear and dropout read a bf16 leaf, and set_bf16_aggregation keeps the
  inputs of a dropped sum and of the dynamic, softmax and dot gathers in fp32.
- One loss, softmax or sigmoid (labels from datasets.node_data / datasets.multilabel_node_data)."""
import atexit
import itertools
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import pytest

from conftest import ROOT
from opgraph import INNER, Recorder, witness
from roc_b200 import _lib, datasets
from roc_b200.model import Host, Model

pytestmark = pytest.mark.gpu
NONE, RELU = _lib.AC_MODE_NONE, _lib.AC_MODE_RELU
SEEN = set()               # what the cases reached: op kinds, fusions, near-misses, width classes
WORST = {}                 # output family -> worst |error| / bound
T0 = time.time()


# ------------------------------------------------------------------------------------------------------ graphs ---
def symmetric(n, pairs, seed, hub=False):
    """Symmetric, deduplicated, a self loop on every node, sources strictly increasing per row.  hub: node 0 is
    joined to every node, so its row has n > 2,112 in-edges (cut rows and the big-row fix-up)."""
    rng = np.random.RandomState(seed)
    s, d = rng.randint(0, n, size=pairs), rng.randint(0, n, size=pairs)
    if hub:
        s, d = np.concatenate([s, np.arange(n)]), np.concatenate([d, np.zeros(n, dtype=np.int64)])
    s, d = np.concatenate([s, d, np.arange(n)]), np.concatenate([d, s, np.arange(n)])
    key = np.unique(d.astype(np.int64) * n + s)
    d, s = key // n, key % n
    return np.cumsum(np.bincount(d, minlength=n)).astype(np.uint64), s.astype(np.uint32)


def directed_multigraph(n=250, e=1800, seed=3):
    """Directed, with duplicate edges, a heavy row and a self loop on every node."""
    rng = np.random.RandomState(seed)
    dst = rng.randint(0, n, size=e)
    src = (rng.zipf(1.6, size=e) - 1) % n
    src[1::4], dst[1::4] = src[0::4][:src[1::4].shape[0]], dst[0::4][:dst[1::4].shape[0]]
    dst[:120] = 9
    dst, src = np.concatenate([dst, np.arange(n)]), np.concatenate([src, np.arange(n)])
    order = np.argsort(dst, kind="stable")
    return np.cumsum(np.bincount(dst[order], minlength=n)).astype(np.uint64), src[order].astype(np.uint32)


GRAPHS = {}


def graph(kind):
    if kind not in GRAPHS:
        GRAPHS[kind] = {"sym": lambda: symmetric(300, 1200, 1), "hub": lambda: symmetric(2300, 3000, 2, hub=True),
                        "directed": directed_multigraph}[kind]()
        if kind == "hub":
            assert np.diff(np.concatenate([[0], GRAPHS[kind][0].astype(np.int64)])).max() > 2112
    return GRAPHS[kind]


# --------------------------------------------------------------------------------------------------- the runner ---
DEFAULTS = dict(fusedInto=-1, bwdFused=0, epilogue=0, bwdEpilogue=0, fwdOut=-1, bwdOut=-1, flags=0, dropOp=-1,
                dxOut=-1, dxReluOf=-1, dxNorm=0, gradOut=-1)


def fusions(infos):
    """{layer: the fields init() changed from their defaults}."""
    out = {}
    for layer, info in enumerate(infos):
        d = {k: v for k, v in info.items() if k != "kind" and v != DEFAULTS[k]}
        if d:
            out[layer] = d
    return out


def note_fusions(fz, ir):
    for layer, d in fz.items():
        kind = ir.nodes[layer]["kind"]
        if kind == "linear" and d.get("flags"):
            SEEN.add("fusion:linear_norm_sg")
        if kind == "scatter_gather" and "epilogue" in d:
            epi = d["epilogue"]
            SEEN.add("fusion:sg_norm_relu" if epi & _lib.SG_EPI_RELU else "fusion:sg_norm")
            if epi & _lib.SG_EPI_NORM_OUT:
                SEEN.add("fusion:teleport_norm_out")
        if kind == "scatter_gather" and ir.nodes[layer]["attrs"].get("dropout", 0.0) > 0 and \
                ("epilogue" in d or "bwdEpilogue" in d):
            SEEN.add("fusion:gcn_block_edge_dropout")
        if kind == "scaled_add" and d.get("fusedInto", -1) >= 0:
            SEEN.add("fusion:teleport")
            if ir.nodes[d["fusedInto"]]["attrs"].get("dropout", 0.0) > 0:
                SEEN.add("fusion:teleport_edge_dropout")
        if kind in ("batch_norm", "layer_norm") and d.get("fwdOut", -1) >= 0:
            SEEN.add("fusion:%s_relu" % kind)
        if kind == "linear" and d.get("dropOp", -1) >= 0:
            SEEN.add("fusion:dropout_linear")
        if kind in ("softmax_cross_entropy", "sigmoid_cross_entropy"):
            SEEN.add("fusion:norm_softmax")
        if kind == "linear" and d.get("dxNorm"):
            SEEN.add("fusion:norm_relu_linear" if ir.nodes[layer - 1]["kind"] == "relu" else
                     "fusion:norm_relu_dropout_linear")


def note_features(ir, dtypes, gkind):
    """What a case exercised beyond op kinds: attention dropout, edge dropout, each attention_gather mode, learned and
    constant temperatures, inputs of a gather that are one tensor, a new gather's input another op also reads (before
    or after it), the infer-mode softmax and dot forwards on the hub graph's cut rows, the sigmoid loss, bf16 tensors,
    and a norm or dropout that a later scaled_add shares its input with (the amended Q7)."""
    if any(nd["kind"] == "attention_gather" and nd["attrs"].get("dropout", 0.0) > 0 for nd in ir.nodes):
        SEEN.add("attn_dropout")
    if any(nd["kind"] == "scatter_gather" and nd["attrs"].get("dropout", 0.0) > 0 for nd in ir.nodes):
        SEEN.add("edge_dropout")
    for nd in ir.nodes:
        if nd["kind"] != "attention_gather":
            continue
        a, ins = nd["attrs"], nd["ins"]
        SEEN.add("mode:" + a["mode"])
        if a["mode"] == "softmax":
            SEEN.add("temperature:learned" if a["learn"] else "temperature:constant")
        if a["mode"] in ("softmax", "dot") and gkind == "hub":
            SEEN.add("cut_rows_infer:" + a["mode"])
        if a["mode"] == "dynamic" and ins[0] == ins[1]:
            SEEN.add("alias:xl_is_xr")
        if a["mode"] == "dot" and len(set(ins)) < 3:
            SEEN.add("alias:" + {(True, True): "q_is_k_is_v", (True, False): "q_is_k", (False, True): "k_is_v",
                                 (False, False): "q_is_v"}[(ins[0] == ins[1], ins[1] == ins[2])])
        if a["mode"] != "gat":
            for r in ir.nodes:
                if r is not nd and set(r["ins"]) & set(ins):
                    SEEN.add("gather_input_also_read_" + ("before" if r["layer"] < nd["layer"] else "after"))
    if ir.loss_node()["kind"] == "sigmoid_cross_entropy":
        SEEN.add("loss:sigmoid")
    if ir.bf16:
        SEEN.add("bf16:features")
    if any(d == "bfloat16" and t not in ir.bf16 for t, d in dtypes.items()):
        SEEN.add("bf16:aggregation")
    for nd in ir.nodes:
        if nd["kind"] in ("indegree_norm", "dropout") and any(
                r["kind"] == "scaled_add" and r["layer"] > nd["layer"] and nd["ins"][0] in r["ins"] for r in ir.nodes):
            SEEN.add("scaled_add_shared_reader")


def note_widths(ir):
    for nd in ir.nodes:
        k = nd["kind"]
        SEEN.add("op:" + k)
        if k == "linear":
            i, o = ir.width[nd["ins"][0]], nd["attrs"]["out_dim"]
            SEEN.add("op:linear_relu" if nd["attrs"]["activation"] == RELU else "op:linear_none")
            if i % 4:
                SEEN.add("width:linear_in_not_float4")
            if o > 128:
                SEEN.add("width:linear_out_over_128")
        w = ir.width.get(nd["ins"][0], 0)
        if k.startswith("scatter_gather") or k == "attention_gather":
            if w % 4 and w <= 16:
                SEEN.add("width:sg_H_not_float4")
            if 65 <= w <= 128:
                SEEN.add("width:sg_65_128")
            if 129 <= w <= 256:
                SEEN.add("width:sg_129_256")
        if k == "softmax_cross_entropy":
            SEEN.add("width:softmax_C_%d" % w)


def family(name, got, want, rtol, atol_scale):
    """rel_close, keeping the worst |error| / bound of each output family.  A dW row that vanishes identically (the
    destination-score rows of an attention score Linear when every edge's LeakyReLU is on one side: the softmax does
    not change when a row's scores shift together) holds only fp32 rounding of terms that cancel; such a row, below
    1e-12 of the matrix's largest entry in fp64, is held to 1e-4 of that entry instead."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, name
    scale = np.abs(want).max() if want.size else 0.0
    bound = rtol * np.abs(want) + atol_scale * scale + 1e-30
    if want.ndim == 2 and want.size:
        zero_rows = np.abs(want).max(axis=1) <= 1e-12 * scale
        bound[zero_rows] = 1e-4 * scale + 1e-30
    r = float((np.abs(got - want) / bound).max()) if want.size else 0.0
    WORST[name] = max(WORST.get(name, 0.0), r)
    return r


def run(build, gkind, fuse, steps=3, feats_seed=5):
    """Build with `build(ir)` (it makes the graph and the loss, returns its handles), train `steps` Adam steps and
    run one infer forward.  Per step: weights before it, logits, dW, edge gradients, weights after it, the relu masks,
    max / min choices and bf16 values; then the running statistics, the infer logits (with their masks, choices and
    bf16 values), the infer metrics and the fusion report."""
    row_end, col = graph(gkind)
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    ir = Recorder(m)
    h = build(ir)
    ir.adam(0.01, 0.05)
    ir.init()
    loss = ir.loss_node()
    logits_t, label_t, mask_t = loss["ins"]
    rng = np.random.RandomState(feats_seed)
    feats = {t: rng.uniform(-1, 1, size=(n, ir.width[t])).astype(np.float32) for t in ir.leaves if t != label_t}
    for t, a in feats.items():
        m.set_tensor(t, a)
    if loss["kind"] == "sigmoid_cross_entropy":
        _, labels, mask = datasets.multilabel_node_data(n, 1, ir.width[logits_t], seed=feats_seed)
        labels, mask = labels.numpy(), mask.numpy()
        m.set_multilabels(label_t, labels)
    else:
        _, labels, mask = datasets.node_data(n, 1, ir.width[logits_t], seed=feats_seed)
        labels, mask = labels.numpy(), mask.numpy()
        m.set_labels(label_t, labels)
    m.set_tensor(mask_t, mask.astype(np.int32))
    ev = {}
    for e in ir.edges:
        ev[e] = np.random.RandomState(e).uniform(0.05, 0.6, size=col.shape[0]).astype(np.float32)
        m.set_tensor(e, ev[e])
    relu_of = {nd["layer"]: nd["out"] for nd in ir.nodes
               if nd["kind"] == "relu" or (nd["kind"] == "linear" and nd["attrs"]["activation"] == RELU)}
    minmax = {nd["layer"]: nd["out"] for nd in ir.nodes if nd["kind"] in ("scatter_gather_max", "scatter_gather_min")}
    dtypes = {t: m.tensor_dtype(t) for t in ir.width if t < INNER}
    half = [t for t, d in dtypes.items() if d == "bfloat16" and t not in ir.bf16]

    def observe():
        return dict(logits=m.get_tensor(logits_t), relu={l: m.get_tensor(t) > 0 for l, t in relu_of.items()},
                    args={l: m.get_aggr_index(t) for l, t in minmax.items()},
                    rounded={t: m.get_tensor(t) for t in half})

    out = dict(steps=[], ir=ir, h=h, feats=feats, labels=labels, mask=mask, edges=ev, info=m.op_info(), dtypes=dtypes)
    for _ in range(steps):
        w0 = [m.get_parameter(p) for p in range(m.num_parameters())]
        m.train_mode(); m.zero_gradients(); m.forward()
        st = dict(w0=w0, **observe())
        m.backward()
        st["dw"] = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        st["de"] = {e: m.get_tensor(e, grad=True)[:, 0].copy() for e in ir.edges if ir.edge_grad[e]}
        m.update()
        st["w1"] = [m.get_parameter(p) for p in range(m.num_parameters())]
        out["steps"].append(st)
    out["run_stats"] = {nd["out"]: m.batch_norm_stats(nd["out"]) for nd in ir.nodes if nd["kind"] == "batch_norm"}
    m.infer_mode(); m.forward()
    out["infer"] = observe()
    out["metrics"] = m.metrics()
    host.close()
    return out


def check_case(build, gkind="sym", expect=None):
    """Both schedules against the witness and each other; `expect(h)`: the fused schedule's fusion report.  Returns
    the fused schedule's run."""
    fused, unfused = run(build, gkind, True), run(build, gkind, False)
    ir = fused["ir"]
    row_end, col = graph(gkind)
    n = row_end.shape[0]
    fz = fusions(fused["info"])
    assert fusions(unfused["info"]) == {}, "the unfused schedule fused something"
    if expect is not None:
        assert fz == expect(fused["h"]), fz
    note_fusions(fz, ir)
    note_widths(ir)
    note_features(ir, fused["dtypes"], gkind)
    bn_momentum = {nd["out"]: nd["attrs"]["momentum"] for nd in ir.nodes if nd["kind"] == "batch_norm"}
    # a learned temperature's and a GATv2 a's gradient sum over every edge and column, sums that cancel: the bars of
    # test_softmax_aggr_gpu.py and test_gatv2_gpu.py, as families of their own
    sums = {nd["attrs"]["param"]: "dt" if nd["attrs"]["mode"] == "softmax" else "da" for nd in ir.nodes
            if nd["kind"] == "attention_gather" and nd["attrs"].get("param") is not None}
    for r in (fused, unfused):
        name = "fused" if r is fused else "unfused"
        rec = {t: (np.zeros(ir.width[t]), np.ones(ir.width[t])) for t in bn_momentum}
        for step, st in enumerate(r["steps"]):
            what = "%s step %d" % (name, step)
            wit = witness(ir, (row_end, col), r["feats"], r["labels"], r["mask"], st["w0"], r["edges"], step=step + 1,
                          relu_masks=st["relu"], aggr_args=st["args"], rounded=st["rounded"])
            assert family("logits", st["logits"], wit["logits"], 1e-4, 1e-5) <= 1, what + " logits vs fp64"
            for p, (a, b) in enumerate(zip(st["dw"], wit["dW"])):
                fam = sums.get(p, "dW")
                bar = (1e-3, 1e-4) if p in sums else (2e-4, 2e-5)
                assert family(fam, a, b, *bar) <= 1, what + " %s[%d] vs fp64" % (fam, p)
            for e, g in st["de"].items():
                assert family("edge gradient", g, wit["edge_grad"][e], 2e-4, 2e-5) <= 1, what + " edge gradient"
            for t, (mean, var) in wit["stats"].items():
                mo, (rm, rv) = bn_momentum[t], rec[t]
                rec[t] = ((1 - mo) * rm + mo * mean, (1 - mo) * rv + mo * var * n / (n - 1))
        for t, (rm, rv) in rec.items():
            assert family("running stats", r["run_stats"][t][0], rm, 2e-4, 2e-5) <= 1, name + " running mean"
            assert family("running stats", r["run_stats"][t][1], rv, 2e-4, 2e-5) <= 1, name + " running var"
        inf = r["infer"]
        wit = witness(ir, (row_end, col), r["feats"], r["labels"], r["mask"], r["steps"][-1]["w1"], r["edges"],
                      relu_masks=inf["relu"], aggr_args=inf["args"], rounded=inf["rounded"], training=False,
                      run_stats=r["run_stats"])
        assert family("infer logits", inf["logits"], wit["logits"], 1e-4, 1e-5) <= 1, name + " infer logits vs fp64"
    same = lambda a, b: np.array_equal(np.asarray(a).view(np.int32), np.asarray(b).view(np.int32))
    if fused["dtypes"] == unfused["dtypes"]:
        for step, (a, b) in enumerate(zip(fused["steps"], unfused["steps"])):
            assert same(a["logits"], b["logits"]), "step %d: logits differ between the schedules" % step
            for p in range(len(a["dw"])):
                assert same(a["dw"][p], b["dw"][p]), "step %d: dW[%d] differs between the schedules" % (step, p)
                assert same(a["w1"][p], b["w1"][p]), "step %d: W[%d] differs between the schedules" % (step, p)
            for e in a["de"]:
                assert same(a["de"][e], b["de"][e]), "step %d: edge gradient differs" % step
        for t in fused["run_stats"]:
            for a, b in zip(fused["run_stats"][t], unfused["run_stats"][t]):
                assert same(a, b), "running statistics differ between the schedules"
        assert same(fused["infer"]["logits"], unfused["infer"]["logits"]), "infer logits differ between the schedules"
        fm, um = dict(fused["metrics"]), dict(unfused["metrics"])
        fm.pop("trainLoss"), um.pop("trainLoss")
        assert fm == um, (fm, um)
    else:
        assert ir.bf16_aggregation, "the schedules store different tensors in bf16 without set_bf16_aggregation"
    fm = fused["metrics"]
    mask = fused["mask"]
    assert (fm["trainAll"], fm["valAll"], fm["testAll"]) == tuple(int((mask == k).sum()) for k in (0, 1, 2)), fm
    return fused


def loss(ir, t, sigmoid=False):
    f = ir.sigmoid_cross_entropy if sigmoid else ir.softmax_cross_entropy
    f(t, ir.create_node_tensor(ir.width[t]), ir.create_node_tensor(1, is_int=True))


# ------------------------------------------------------------------------------------------ (a) hand-listed cases ---
def lin_norm_sg(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); n = ir.indegree_norm(t); s = ir.scatter_gather(n)
    loss(ir, s)
    return dict(t=t, n=n, s=s)


def sg_norm(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); s = ir.scatter_gather(t); n = ir.indegree_norm(s)
    loss(ir, n)
    return dict(t=t, s=s, n=n)


def sg_norm_relu(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); s = ir.scatter_gather(t); n = ir.indegree_norm(s); r = ir.relu(n)
    loss(ir, r)
    return dict(s=s, n=n, r=r)


def dropout_linear(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); d = ir.dropout(t, 0.5, seed=3); y = ir.linear(d, 5)
    loss(ir, y)
    return dict(t=t, d=d)


def norm_softmax(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 5); n = ir.indegree_norm(t)
    loss(ir, n)
    return dict(t=t, n=n)


def norm_relu_linear(ir, drop=False):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); s = ir.scatter_gather(t); n = ir.indegree_norm(s); r = ir.relu(n)
    d = ir.dropout(r, 0.5, seed=1) if drop else r
    y = ir.linear(d, 5)
    loss(ir, y)
    return dict(s=s, n=n, r=r)


def expect_fused_chain(h, sg_layer, relu=True):
    """sg -> norm [-> relu] as the downstream SG fusion leaves it (the layers follow the SG)."""
    e = {sg_layer: dict(epilogue=_lib.SG_EPI_NORM | (_lib.SG_EPI_RELU if relu else 0), fwdOut=h["r"] if relu
                        else h["n"]), sg_layer + 1: dict(fusedInto=sg_layer)}
    if relu:
        e[sg_layer + 2] = dict(fusedInto=sg_layer)
    return e


def batch_norm_relu(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); b = ir.batch_norm(t); r = ir.relu(b)
    loss(ir, ir.linear(r, 5))
    return dict(b=b, r=r)


def teleport(ir, norm_out=False, t0="before", second=False, sa_twice=False, drop=0.0):
    """linear -> norm -> sg -> norm -> scaled_add(., t0, 0.9, 0.1) [-> norm] -> linear: t0 a Linear made before the
    scatter_gather (or after it); second: the norm output is the scaled_add's second input; sa_twice: a relu also
    reads the scaled_add's output; drop: the sum's edge dropout rate."""
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16)
    u = ir.linear(x, 16) if t0 == "before" else None
    n1 = ir.indegree_norm(t); s = ir.scatter_gather(n1, dropout=drop, seed=2); n2 = ir.indegree_norm(s)
    if u is None:
        u = ir.linear(x, 16)
    y = ir.scaled_add(u, n2, 0.9, 0.1) if second else ir.scaled_add(n2, u, 0.9, 0.1)
    r = ir.relu(y) if sa_twice else None                # before the norm, which must be y's last reader
    z = ir.indegree_norm(y) if norm_out else y
    out = ir.linear(z, 5)
    if sa_twice:
        out = ir.add(out, ir.linear(r, 5))
    loss(ir, out)
    return dict(t=t, n1=n1, n2=n2, y=y, z=z)


def expect_teleport(h, fused=True, norm_out=False, sg=3):
    """the GCN block's two fusions on the layers teleport() makes, the teleport on top when `fused`"""
    e = {0: dict(flags=_lib.LINEAR_NORM_EPILOGUE, fwdOut=h["n1"]), sg - 1: dict(fusedInto=0),
         sg: dict(bwdEpilogue=_lib.SG_EPI_NORM, bwdOut=h["t"], epilogue=_lib.SG_EPI_NORM, fwdOut=h["n2"]),
         sg + 1: dict(fusedInto=sg)}
    if fused:
        e[sg]["fwdOut"] = h["y"]
        e[sg + 2] = dict(fusedInto=sg)
    if norm_out:
        e[sg]["epilogue"] |= _lib.SG_EPI_NORM_OUT
        e[sg]["fwdOut"] = h["z"]
        e[sg + 3] = dict(fusedInto=sg)
    return e


def layer_norm_relu(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); b = ir.layer_norm(t); r = ir.relu(b)
    loss(ir, ir.linear(r, 5))
    return dict(b=b, r=r)


def gcn_block_edge_dropout(ir):
    """linear -> norm -> sg(dropout) -> norm -> relu -> linear: every GCN-block fusion around a dropped sum"""
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); n1 = ir.indegree_norm(t); s = ir.scatter_gather(n1, dropout=0.5, seed=3)
    n2 = ir.indegree_norm(s); r = ir.relu(n2)
    loss(ir, ir.linear(r, 5))
    return dict(t=t, n1=n1, s=s, r=r)


HAND = {
    "batch_norm_relu": (batch_norm_relu, lambda h: {1: dict(fwdOut=h["r"]), 2: dict(fusedInto=1)}),
    "layer_norm_relu": (layer_norm_relu, lambda h: {1: dict(fwdOut=h["r"]), 2: dict(fusedInto=1)}),
    # the dropped sum's forward takes the norm (and relu) epilogue, its backward the norm epilogue into d(linear out)
    "gcn_block_edge_dropout": (gcn_block_edge_dropout, lambda h: {
        0: dict(flags=_lib.LINEAR_NORM_EPILOGUE, fwdOut=h["n1"]), 1: dict(fusedInto=0),
        2: dict(bwdEpilogue=_lib.SG_EPI_NORM, bwdOut=h["t"], epilogue=_lib.SG_EPI_NORM | _lib.SG_EPI_RELU,
                fwdOut=h["r"]),
        3: dict(fusedInto=2, bwdFused=1), 4: dict(fusedInto=2), 5: dict(dxReluOf=h["r"], dxNorm=1, dxOut=h["s"])}),
    "teleport_edge_dropout": (lambda ir: teleport(ir, drop=0.5), expect_teleport),
    "teleport_norm_out_edge_dropout": (lambda ir: teleport(ir, norm_out=True, drop=0.1),
                                       lambda h: expect_teleport(h, norm_out=True)),
    "teleport": (teleport, expect_teleport),
    "teleport_norm_out": (lambda ir: teleport(ir, norm_out=True), lambda h: expect_teleport(h, norm_out=True)),
    # each fusion alone, in its minimal pattern
    "lin_norm_sg": (lin_norm_sg, lambda h: {0: dict(flags=_lib.LINEAR_NORM_EPILOGUE, fwdOut=h["n"]), 1: dict(fusedInto=0),
                                            2: dict(bwdEpilogue=_lib.SG_EPI_NORM, bwdOut=h["t"])}),
    # the norm feeds the loss: the softmax takes its backward too
    "sg_norm": (sg_norm, lambda h: {1: dict(epilogue=_lib.SG_EPI_NORM, fwdOut=h["n"]), 2: dict(fusedInto=1, bwdFused=1),
                                    3: dict(gradOut=h["s"])}),
    "sg_norm_relu": (sg_norm_relu, lambda h: expect_fused_chain(h, 1)),
    "dropout_linear": (dropout_linear, lambda h: {1: dict(fusedInto=2), 2: dict(dropOp=1)}),
    "norm_softmax": (norm_softmax, lambda h: {1: dict(bwdFused=1), 2: dict(gradOut=h["t"])}),
    "norm_relu_linear": (norm_relu_linear, lambda h: {**expect_fused_chain(h, 1),
                                                      2: dict(fusedInto=1, bwdFused=1),
                                                      4: dict(dxReluOf=h["r"], dxNorm=1, dxOut=h["s"])}),
    "norm_relu_dropout_linear": (lambda ir: norm_relu_linear(ir, drop=True),
                                 lambda h: {**expect_fused_chain(h, 1), 2: dict(fusedInto=1, bwdFused=1),
                                            4: dict(fusedInto=5),
                                            5: dict(dropOp=4, dxReluOf=h["r"], dxNorm=1, dxOut=h["s"])}),
}


def near(name):
    SEEN.add("near:" + name)


def nm_linear_out_twice(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); r = ir.relu(t); n = ir.indegree_norm(t); s = ir.scatter_gather(n)
    loss(ir, ir.linear(ir.add(s, r), 5))


def nm_norm1_out_twice(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); n = ir.indegree_norm(t); r = ir.relu(n); s = ir.scatter_gather(n)
    loss(ir, ir.linear(ir.add(s, r), 5))


def nm_sg_out_twice(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); s = ir.scatter_gather(t); r = ir.relu(s); n = ir.indegree_norm(s)
    loss(ir, ir.linear(ir.add(n, r), 5))


def nm_norm2_out_twice(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); s = ir.scatter_gather(t); n = ir.indegree_norm(s); g = ir.sigmoid(n); r = ir.relu(n)
    loss(ir, ir.linear(ir.add(r, g), 5))
    return dict(n=n)


def nm_relu_out_twice(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); s = ir.scatter_gather(t); n = ir.indegree_norm(s); r = ir.relu(n)
    loss(ir, ir.add(ir.linear(r, 5), ir.linear(r, 5)))
    return dict(n=n, r=r)


def nm_linear_relu(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16, RELU); n = ir.indegree_norm(t); s = ir.scatter_gather(n)
    loss(ir, ir.linear(s, 5))


def nm_aggr(aggr):
    def build(ir):
        x = ir.create_node_tensor(12)
        t = ir.linear(x, 16); n = ir.indegree_norm(t)
        s = ir.scatter_gather(n, weights=ir.create_edge_tensor()) if aggr == "weighted" else ir.scatter_gather(n, aggr)
        n2 = ir.indegree_norm(s); r = ir.relu(n2)
        loss(ir, ir.linear(r, 5))
    return build


def nm_sigmoid(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); s = ir.scatter_gather(t); n = ir.indegree_norm(s); g = ir.sigmoid(n)
    loss(ir, ir.linear(g, 5))
    return dict(n=n)


def nm_dropout_twice(ir):
    x = ir.create_node_tensor(12)
    d = ir.dropout(x, 0.5, seed=2)
    loss(ir, ir.add(ir.linear(d, 5), ir.linear(d, 5)))


def nm_dropout_non_linear(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); d = ir.dropout(t, 0.5, seed=2); r = ir.relu(d)
    loss(ir, ir.linear(r, 5))


def nm_norm_softmax_no_grad(ir):
    x = ir.create_node_tensor(5)
    ir.linear(x, 4)                          # a dead parameter; the norm must be x's last consumer
    loss(ir, ir.indegree_norm(x))


def nm_norm_in_linear_feeds_softmax(ir):
    """model.cc's guard against a norm fused into a Linear feeding the softmax: the upstream fusion needs the norm's
    output read once (by the SG), the softmax fusion needs it read once (by the softmax), so the two never meet.
    With both readers the upstream fusion is refused; the SG comes after the loss so that it is the norm output's
    last consumer, and its output is dead."""
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 5); n = ir.indegree_norm(t)
    loss(ir, n)
    ir.scatter_gather(n)


def nm_competing_norm(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); n1 = ir.indegree_norm(t); s1 = ir.scatter_gather(n1); n2 = ir.indegree_norm(s1)
    s2 = ir.scatter_gather(n2)
    loss(ir, ir.linear(s2, 5))
    return dict(t=t, n1=n1, n2=n2)


def nm_bn(readers, norm="batch_norm"):
    def build(ir):
        x = ir.create_node_tensor(12)
        b = getattr(ir, norm)(ir.linear(x, 16))
        outs = [getattr(ir, k)(b) for k in readers]
        loss(ir, ir.linear(outs[0] if len(outs) == 1 else ir.add(*outs), 5))
    return build


def nm_dropped_sum_bf16(ir):
    """set_bf16_aggregation: a Linear read by a plain sum alone goes bf16; one read by a dropped sum alone stays fp32
    (edge dropout has no bf16 form)"""
    ir.set_bf16_aggregation(True)
    x = ir.create_node_tensor(12)
    a = ir.linear(x, 16); b = ir.linear(x, 16)
    s = ir.add(ir.scatter_gather(a, dropout=0.5, seed=1), ir.scatter_gather(b))
    loss(ir, ir.linear(s, 5))
    return dict(fp32=a, bf16=b)


def nm_teleport_bf16(ir):
    """set_bf16_aggregation stores the fused linear -> norm output the sum scatter_gather reads in bf16: no teleport
    kernel reads it, so the hop stays unfused"""
    ir.set_bf16_aggregation(True)
    return teleport(ir)


def nm_dropout_shared_linear(ir):
    """y = linear(dropout(h)); scaled_add(y, h): the dropout adds to what the scaled_add wrote, so it must not be
    fused into the Linear, whose dX epilogue overwrites"""
    x = ir.create_node_tensor(12)
    h = ir.linear(x, 16)
    y = ir.linear(ir.dropout(h, 0.5, seed=1), 16)
    loss(ir, ir.linear(ir.scaled_add(y, h, 0.9, 0.1), 5))


def nm_norm_shared_loss(ir):
    """norm(h) feeds the loss and a scaled_add made after the loss reads h: the norm's backward adds to what the
    scaled_add wrote, so the loss must not take it over"""
    x = ir.create_node_tensor(12)
    h = ir.linear(x, 5); u = ir.linear(x, 5)
    loss(ir, ir.indegree_norm(h))
    ir.scaled_add(h, u, 1.0, 1.0)


NEAR = {
    "bn_out_read_twice": (nm_bn(("relu", "sigmoid")), lambda h: {}),
    "bn_then_elu": (nm_bn(("elu",)), lambda h: {}),
    "bn_then_sigmoid": (nm_bn(("sigmoid",)), lambda h: {}),
    "layer_norm_out_read_twice": (nm_bn(("relu", "sigmoid"), norm="layer_norm"), lambda h: {}),
    "dropped_sum_input_stays_fp32": (nm_dropped_sum_bf16, lambda h: {}),
    "teleport_sg_input_bf16": (nm_teleport_bf16, lambda h: expect_teleport(h, fused=False)),
    "teleport_t0_after_sg": (lambda ir: teleport(ir, t0="after"), lambda h: expect_teleport(h, fused=False, sg=2)),
    "teleport_norm_second_input": (lambda ir: teleport(ir, second=True), lambda h: expect_teleport(h, fused=False)),
    "scaled_add_out_read_twice": (lambda ir: teleport(ir, norm_out=True, sa_twice=True),
                                  lambda h: expect_teleport(h)),
    "dropout_shared_with_scaled_add_into_linear": (nm_dropout_shared_linear, lambda h: {}),
    "norm_shared_with_scaled_add_into_loss": (nm_norm_shared_loss, lambda h: {}),
    "linear_out_read_twice": (nm_linear_out_twice, lambda h: {}),
    "norm1_out_read_twice": (nm_norm1_out_twice, lambda h: {}),
    "sg_out_read_twice": (nm_sg_out_twice, lambda h: {}),
    "norm2_out_read_twice": (nm_norm2_out_twice, lambda h: {1: dict(epilogue=_lib.SG_EPI_NORM, fwdOut=h["n"]),
                                                            2: dict(fusedInto=1)}),
    "relu_out_read_twice": (nm_relu_out_twice, lambda h: expect_fused_chain(h, 1)),
    "linear_relu_upstream": (nm_linear_relu, lambda h: {}),
    "max_instead_of_sum": (nm_aggr(_lib.AGGR_MAX), lambda h: {}),
    "min_instead_of_sum": (nm_aggr(_lib.AGGR_MIN), lambda h: {}),
    "weighted_instead_of_sum": (nm_aggr("weighted"), lambda h: {}),
    "sigmoid_instead_of_relu": (nm_sigmoid, lambda h: {1: dict(epilogue=_lib.SG_EPI_NORM, fwdOut=h["n"]),
                                                       2: dict(fusedInto=1)}),
    "dropout_read_twice": (nm_dropout_twice, lambda h: {}),
    "dropout_feeds_non_linear": (nm_dropout_non_linear, lambda h: {}),
    "norm_softmax_input_needs_no_grad": (nm_norm_softmax_no_grad, lambda h: {}),
    "norm_in_linear_feeds_softmax": (nm_norm_in_linear_feeds_softmax, lambda h: {}),
    # lin -> n1 -> sg1 -> n2 -> sg2: n2 goes to sg1's epilogue, so sg2 cannot take it for its upstream fusion
    "competing_norm": (nm_competing_norm, lambda h: {0: dict(flags=_lib.LINEAR_NORM_EPILOGUE, fwdOut=h["n1"]),
                                                     1: dict(fusedInto=0),
                                                     2: dict(bwdEpilogue=_lib.SG_EPI_NORM, bwdOut=h["t"],
                                                             epilogue=_lib.SG_EPI_NORM, fwdOut=h["n2"]),
                                                     3: dict(fusedInto=2)}),
}


def add_t_t(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 5)
    loss(ir, ir.add(t, t))


def attention_t_t(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 2)
    loss(ir, ir.linear(ir.attention_gather(t, t, heads=1), 5))


def three_readers(order):
    def build(ir):
        x = ir.create_node_tensor(12)
        t = ir.linear(x, 16)
        make = {"relu": lambda: ir.relu(t), "sigmoid": lambda: ir.sigmoid(t), "linear": lambda: ir.linear(t, 16)}
        outs = [make[k]() for k in order]
        loss(ir, ir.linear(ir.add(ir.add(outs[0], outs[1]), outs[2]), 5))
    return build


def linear_relu_sigmoid(ir):
    x = ir.create_node_tensor(12)
    loss(ir, ir.linear(ir.sigmoid(ir.linear(x, 16, RELU)), 5, RELU))


def sgc(ir):
    x = ir.create_node_tensor(12)
    s = ir.scatter_gather(x); n = ir.indegree_norm(s)
    loss(ir, ir.linear(n, 5))
    return dict(n=n)


def shared_edges(grad):
    def build(ir):
        x = ir.create_node_tensor(12)
        e = ir.create_edge_tensor()
        a = ir.scatter_gather(ir.linear(x, 16), weights=e)
        b = ir.scatter_gather(ir.relu(a), weights=e)
        loss(ir, ir.linear(b, 5))
        ir.set_edge_grad(e, grad)
    return build


def dead_branch(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16)
    y = ir.linear(t, 5)
    ir.relu(ir.linear(t, 8))          # created after y: its backward runs first and writes t's gradient
    loss(ir, y)


def scores_and_gather_t(ir):
    x = ir.create_node_tensor(12)
    wh = ir.linear(x, 16)
    loss(ir, ir.linear(ir.attention_gather(wh, ir.attention_scores(wh, heads=4), heads=4, dropout=0.6, seed=1), 5))


def scaled_add_t_relu_t(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16)
    loss(ir, ir.linear(ir.scaled_add(t, ir.relu(t), 0.9, 0.1), 5))


def elu_and_bn_t(ir):
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16)
    loss(ir, ir.linear(ir.add(ir.elu(t), ir.batch_norm(t)), 5))


def gather(kind, ir, t, u=None, v=None):
    """one of the new gathers over (t, u, v) (the ones its mode reads)"""
    if kind == "dynamic":
        return ir.dynamic_attention_gather(t, u, heads=4)
    if kind == "softmax":
        return ir.softmax_gather(t, 3.0, learn_temperature=False)
    return ir.dot_attention_gather(t, u, v, heads=2)


def aliased(kind, names):
    """the gather's inputs drawn from three Linears by name: "ttt" is q = k = v = t"""
    def build(ir):
        x = ir.create_node_tensor(12)
        lin = {c: ir.linear(x, 16) for c in sorted(set(names))}
        loss(ir, ir.linear(gather(kind, ir, *(lin[c] for c in names)), 5))
    return build


def gather_input_also_read(kind, before):
    """a relu reads the gather's first input t, created before or after the gather: its backward writes t's gradient
    first or last"""
    def build(ir):
        x = ir.create_node_tensor(12)
        t, u, v = ir.linear(x, 16), ir.linear(x, 16), ir.linear(x, 16)
        r = ir.relu(t) if before else None
        g = gather(kind, ir, t, u, v)
        if r is None:
            r = ir.relu(t)
        loss(ir, ir.linear(ir.add(g, r), 5))
    return build


def over_leaves(kind):
    """the gather reads leaves only: the dynamic one's a and the learned temperature still give its output a gradient;
    the dot one has none, its backward runs nothing"""
    def build(ir):
        x, y, z = (ir.create_node_tensor(16) for _ in range(3))
        g = ir.softmax_gather(x, 1.0, learn_temperature=True) if kind == "softmax" else gather(kind, ir, x, y, z)
        loss(ir, ir.linear(g, 5))
    return build


SHARED = {
    "dynamic_xl_is_xr": (aliased("dynamic", "tt"), lambda h: {}),
    "dot_q_is_k_is_v": (aliased("dot", "ttt"), lambda h: {}),
    "dot_q_is_k": (aliased("dot", "ttu"), lambda h: {}),
    "dot_k_is_v": (aliased("dot", "tuu"), lambda h: {}),
    "softmax_learned_over_a_leaf": (over_leaves("softmax"), lambda h: {}),
    "dynamic_over_leaves": (over_leaves("dynamic"), lambda h: {}),
    "dot_over_leaves": (over_leaves("dot"), lambda h: {}),
    "attention_scores_and_gather_t": (scores_and_gather_t, lambda h: {}),
    "scaled_add_t_relu_t": (scaled_add_t_relu_t, lambda h: {}),
    "elu_and_batch_norm_t": (elu_and_bn_t, lambda h: {}),
    "add_t_t": (add_t_t, lambda h: {}),
    "attention_t_t_H2": (attention_t_t, lambda h: {}),
    "linear_relu_and_sigmoid": (linear_relu_sigmoid, lambda h: {}),
    "sgc_raw_features": (sgc, lambda h: {0: dict(epilogue=_lib.SG_EPI_NORM, fwdOut=h["n"]), 1: dict(fusedInto=0)}),
    "shared_edges_grad_on": (shared_edges(True), lambda h: {}),
    "shared_edges_grad_off": (shared_edges(False), lambda h: {}),
    "dead_branch": (dead_branch, lambda h: {}),
}
for _o in itertools.permutations(("relu", "sigmoid", "linear")):
    SHARED["three_readers_" + "_".join(_o)] = (three_readers(_o), lambda h: {})
for _k in ("dynamic", "softmax", "dot"):
    for _b in (True, False):
        SHARED["%s_input_also_read_%s" % (_k, "before" if _b else "after")] = (gather_input_also_read(_k, _b),
                                                                              lambda h: {})


def exact_gcn(ir):
    ir.set_exact_backward(True)
    x = ir.create_node_tensor(12)
    t = ir.linear(ir.dropout(x, 0.5), 16); s = ir.scatter_gather(ir.indegree_norm(t)); r = ir.relu(ir.indegree_norm(s))
    t2 = ir.linear(ir.dropout(r, 0.5), 5)
    loss(ir, ir.indegree_norm(ir.scatter_gather(ir.indegree_norm(t2))))


def exact_pool(aggr):
    def build(ir):
        ir.set_exact_backward(True)
        x = ir.create_node_tensor(12)
        p = ir.relu(ir.linear(x, 16))
        loss(ir, ir.add(ir.linear(ir.scatter_gather(p, aggr), 5), ir.linear(x, 5)))
    return build


def exact_attention_weighted(ir):
    ir.set_exact_backward(True)
    x = ir.create_node_tensor(12)
    e = ir.create_edge_tensor()
    wh = ir.linear(x, 16)
    a = ir.relu(ir.attention_gather(wh, ir.linear(wh, 8), heads=4))
    b = ir.scatter_gather(ir.scatter_gather(a, _lib.AGGR_AVG), weights=e)
    ir.set_edge_grad(e, True)
    loss(ir, ir.linear(b, 5))


def exact_gather(kind):
    def build(ir):
        ir.set_exact_backward(True)
        x = ir.create_node_tensor(12)
        t, u, v = ir.linear(x, 16), ir.linear(x, 16), ir.linear(x, 16)
        g = ir.softmax_gather(ir.relu(t), 1.0, learn_temperature=True) if kind == "softmax" else \
            gather(kind, ir, t, u, v)
        loss(ir, ir.linear(ir.relu(g), 5))
    return build


def exact_edge_dropout(ir):
    """two GCN layers on dropped sums: the backward's keep bits are the transposed plan's"""
    ir.set_exact_backward(True)
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16); s = ir.scatter_gather(ir.indegree_norm(t), dropout=0.5, seed=1)
    r = ir.relu(ir.indegree_norm(s))
    t2 = ir.linear(r, 5)
    loss(ir, ir.indegree_norm(ir.scatter_gather(ir.indegree_norm(t2), dropout=0.1, seed=1)))


EXACT = {"gcn_dropout": exact_gcn, "pool_max": exact_pool(_lib.AGGR_MAX), "pool_min": exact_pool(_lib.AGGR_MIN),
         "attention_avg_weighted": exact_attention_weighted, "dynamic": exact_gather("dynamic"),
         "softmax_learned": exact_gather("softmax"), "dot": exact_gather("dot"), "edge_dropout": exact_edge_dropout}


def cut_rows(kind):
    """a softmax or dot gather on the hub graph: the infer forward keeps no stats, and each cut row's raw (m, s) go
    through the plan's shared workspace"""
    def build(ir):
        x = ir.create_node_tensor(12)
        t, u, v = ir.linear(x, 16), ir.linear(x, 16), ir.linear(x, 16)
        g = ir.softmax_gather(t, 1.0, learn_temperature=True) if kind == "softmax" else \
            ir.dot_attention_gather(t, u, v, heads=4)
        loss(ir, ir.linear(g, 5))
    return build


CUT = {"softmax": cut_rows("softmax"), "dot": cut_rows("dot")}


@pytest.mark.parametrize("name", list(HAND))
def test_each_fusion_alone(name):
    build, expect = HAND[name]
    check_case(build, expect=expect)


@pytest.mark.parametrize("name", list(NEAR))
def test_fusion_near_miss(name):
    build, expect = NEAR[name]
    r = check_case(build, expect=expect)
    if name == "dropped_sum_input_stays_fp32":
        assert (r["dtypes"][r["h"]["fp32"]], r["dtypes"][r["h"]["bf16"]]) == ("float32", "bfloat16"), r["dtypes"]
    near(name)


@pytest.mark.parametrize("name", list(SHARED))
def test_shared_and_aliased(name):
    build, expect = SHARED[name]
    check_case(build, expect=expect)
    SEEN.add("shared:" + name)


@pytest.mark.parametrize("name", list(EXACT))
def test_exact_mode_on_a_directed_multigraph(name):
    check_case(EXACT[name], gkind="directed")
    SEEN.add("exact:" + name)


@pytest.mark.parametrize("name", list(CUT))
def test_softmax_and_dot_on_cut_rows(name):
    check_case(CUT[name], gkind="hub")


# ------------------------------------------------------------------------------------------ (b) random graphs ---
SMALL, RING_U, RING_T = (3, 5, 7, 12, 16), (72, 100, 128), (132, 160, 256)
CLASSES = (5, 32, 33, 64, 65, 128, 129)


SEEDS = 64
COEFFS = ((1.0, 1.0), (0.9, 0.1), (1.5, -0.5), (0.0, 1.0))
TEMPERATURES = (0.0, 1.0, -0.5, 3.0)
EDGE_DROPOUT = (0.1, 0.5)


def random_graph(seed):
    """A seeded DAG over every op, obeying the rules in the module docstring.  Tensors a ScatterGather, a norm or a
    dropout (whose input needs a gradient) have read are closed: nothing reads them again, except the scaled_add a
    "shared" step makes.  Every tensor nothing reads at the end goes through a Linear into one sum that feeds the
    loss, except, now and then, a dead one."""
    exact = seed % 6 == 5
    gkind = "directed" if exact else ("hub" if seed % 8 == 3 else "sym")
    half_x, half_aggr, sigmoid = seed % 5 == 2, seed % 7 == 4, seed % 3 == 1

    def build(ir):                       # called once per schedule: the same graph each time
        rng = np.random.RandomState(seed)
        if exact:
            ir.set_exact_backward(True)
        if half_aggr:
            ir.set_bf16_aggregation(True)
        open_, grad, closed = [], {}, set()
        edges = []

        def take(t, closes):
            open_.remove(t) if closes and t in open_ else None
            if closes:
                closed.add(t)

        def new(t, g):
            open_.append(t)
            grad[t] = g
            return t

        def partner(t):
            """an open fp32 tensor of t's width other than t, or None"""
            same = [u for u in open_ if ir.width[u] == ir.width[t] and u != t and u not in ir.bf16]
            return same[rng.randint(len(same))] if same else None

        def coeffs():
            return COEFFS[rng.randint(len(COEFFS))]

        def drop_rate():
            return EDGE_DROPOUT[rng.randint(len(EDGE_DROPOUT))]

        x = ir.create_node_tensor(int(rng.choice((7, 12, 16, 33))), dtype="bfloat16" if half_x else "float32")
        new(x, False)
        for _ in range(rng.randint(3, 10)):
            t = open_[rng.randint(len(open_))]
            w = ir.width[t]
            k = rng.choice(["linear", "linear", "norm", "sg", "sg_mm", "sg_w", "attn", "relu", "sigmoid", "add",
                            "dropout", "batch_norm", "elu", "scaled_add", "shared", "teleport", "dynamic", "softmax",
                            "dot", "layer_norm"])
            if t in ir.bf16 and k not in ("linear", "dropout"):
                k = "linear"
            if k == "linear":
                pick = rng.randint(4)
                o = int(rng.choice(SMALL + (136, 7) if pick == 0 else RING_U if pick == 1 else RING_T if pick == 2
                                   else SMALL))
                new(ir.linear(t, o, RELU if rng.rand() < 0.3 else NONE), True)
            elif k == "norm":
                take(t, True)
                new(ir.indegree_norm(t), grad[t])
            elif k == "sg":
                take(t, True)
                pick = rng.rand()
                if pick < 0.25:
                    new(ir.scatter_gather(t, _lib.AGGR_AVG), grad[t])
                elif pick < 0.5:
                    new(ir.scatter_gather(t, dropout=drop_rate(), seed=int(rng.randint(4))), grad[t])
                else:
                    new(ir.scatter_gather(t), grad[t])
            elif k == "sg_mm":
                take(t, True)
                new(ir.scatter_gather(t, _lib.AGGR_MAX if rng.rand() < 0.5 else _lib.AGGR_MIN), grad[t])
            elif k == "sg_w":
                if not edges or rng.rand() < 0.3:
                    edges.append(ir.create_edge_tensor())
                e = edges[rng.randint(len(edges))]
                new(ir.scatter_gather(t, weights=e), True)     # WeightedScatterGather adds where it must: no closing
            elif k == "attn":
                heads = int(rng.choice([h for h in (1, 2, 4, 8) if h == 1 or (w % h == 0 and w // h >= 4 and
                                                                               (w // h) & (w // h - 1) == 0)]))
                if w > 512:
                    continue
                sc = ir.attention_scores(t, heads) if rng.rand() < 0.5 else ir.linear(t, 2 * heads)
                rate = 0.6 if rng.rand() < 0.4 else 0.0
                new(ir.attention_gather(t, sc, heads=heads, dropout=rate, seed=int(rng.randint(4))), True)
            elif k in ("dynamic", "dot"):
                heads = [h for h in range(1, 9) if w % h == 0]
                if w > 256:
                    continue
                heads = heads[rng.randint(len(heads))]
                ins = [t] + [t if u is None or rng.rand() < 0.3 else u for u in
                             (partner(t) for _ in range(1 if k == "dynamic" else 2))]
                if k == "dot" and rng.rand() < 0.5:
                    ins = [ins[j] for j in rng.permutation(3)]
                if k == "dynamic":
                    new(ir.dynamic_attention_gather(*ins, heads=heads), True)
                else:
                    new(ir.dot_attention_gather(*ins, heads=heads), any(grad[u] for u in ins))
            elif k == "softmax":
                learn = rng.rand() < 0.5
                new(ir.softmax_gather(t, TEMPERATURES[rng.randint(len(TEMPERATURES))], learn), grad[t] or learn)
            elif k == "layer_norm":
                b = ir.layer_norm(t)
                new(ir.relu(b) if rng.rand() < 0.4 else b, True)   # read by a relu alone: the norm-relu fusion
            elif k in ("relu", "sigmoid", "elu"):
                new(getattr(ir, k)(t), grad[t])
            elif k == "batch_norm":
                b = ir.batch_norm(t)
                if rng.rand() < 0.4:
                    new(ir.relu(b), True)                     # read by a relu alone: the BN-relu fusion
                else:
                    new(b, True)
            elif k == "add":
                same = [u for u in open_ if ir.width[u] == w and u not in ir.bf16]
                u = same[rng.randint(len(same))]
                new(ir.add(t, u), grad[t] or grad[u])
            elif k == "scaled_add":
                u = partner(t)
                if u is None:
                    continue
                a, b = (t, u) if rng.rand() < 0.5 else (u, t)
                new(ir.scaled_add(a, b, *coeffs()), grad[t] or grad[u])
            elif k == "shared":
                # a norm or dropout and a scaled_add reading t, in either creation order; t is then closed
                u = partner(t)
                if u is None:
                    continue
                norm = rng.rand() < 0.5
                rate = float(rng.choice([0.0, 0.5]))
                first = rng.rand() < 0.5
                if first:
                    sa = ir.scaled_add(t, u, *coeffs())
                r = ir.indegree_norm(t) if norm else ir.dropout(t, rate, seed=int(rng.randint(4)))
                if not first:
                    sa = ir.scaled_add(t, u, *coeffs())
                take(t, True)
                new(r, grad[t])
                new(sa, grad[t] or grad[u])
            elif k == "dropout":
                take(t, grad[t])
                new(ir.dropout(t, float(rng.choice([0.0, 0.5])), seed=int(rng.randint(4))), grad[t])
            else:
                # the teleport hop: t0 a leaf, an earlier tensor (t itself: APPNP's shape), or one made after the SG
                take(t, True)
                n1 = ir.indegree_norm(t)
                s = ir.scatter_gather(n1, dropout=drop_rate() if rng.rand() < 0.3 else 0.0, seed=int(rng.randint(4)))
                n2 = ir.indegree_norm(s)
                where = rng.randint(3)
                if where == 1:
                    t0, g0 = t, grad[t]
                elif where == 2 and open_:
                    t0, g0 = new(ir.linear(open_[rng.randint(len(open_))], w), True), True
                else:
                    t0, g0 = ir.create_node_tensor(w), False
                y = ir.scaled_add(n2, t0, *coeffs())
                new(ir.indegree_norm(y) if rng.rand() < 0.5 else y, grad[t] or g0)
        C = int(rng.choice(CLASSES))
        sinks = [t for t in open_ if t != x or len(open_) == 1]
        if len(sinks) > 1 and rng.rand() < 0.25:
            sinks = sinks[1:]                                     # the first one stays dead
        z = None
        for t in sinks:
            y = ir.linear(t, C)
            z = y if z is None else ir.add(z, y)
        if rng.rand() < 0.3:
            z = ir.indegree_norm(z)
        loss(ir, z, sigmoid=sigmoid)
        for e in edges:
            ir.set_edge_grad(e, bool(rng.rand() < 0.7))
    return build, gkind


@pytest.mark.parametrize("seed", range(SEEDS))
def test_random_graph(seed):
    build, gkind = random_graph(seed)
    check_case(build, gkind=gkind)
    SEEN.add("random")
    if gkind == "hub":
        SEEN.add("graph:hub")


# ----------------------------------------------------------------------------------------------- (e) refusals ---
def rf_sg(leaf):
    def build(ir):
        x = ir.create_node_tensor(12)
        t = x if leaf else ir.linear(x, 16)
        s = ir.scatter_gather(t)
        loss(ir, ir.add(ir.linear(s, 5), ir.linear(t, 5)))     # t read again after the SG
    return build


def rf_norm(leaf):
    def build(ir):
        x = ir.create_node_tensor(12)
        t = x if leaf else ir.linear(x, 16)
        n = ir.indegree_norm(t)
        loss(ir, ir.add(ir.linear(n, 5), ir.linear(t, 5)))
    return build


def rf_dropout(into_linear):
    def build(ir):
        x = ir.create_node_tensor(12)
        t = ir.linear(x, 16)
        d = ir.dropout(t, 0.5)
        y = ir.linear(d, 5) if into_linear else ir.linear(ir.relu(d), 5)
        loss(ir, ir.add(y, ir.linear(t, 5)))
    return build


def rf_norm_softmax(ir):
    """The softmax takes the norm's backward (gradOut); a reader of the norm's input created after the loss."""
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 5)
    loss(ir, ir.indegree_norm(t))
    ir.relu(t)


def rf_norm_shared_with_add(ir):
    """A plain add reads the norm's input after it: only a scaled_add makes that wiring legal."""
    x = ir.create_node_tensor(12)
    t = ir.linear(x, 16)
    n = ir.indegree_norm(t)
    loss(ir, ir.linear(ir.add(n, t), 5))


REFUSE = {"norm_shared_with_add_not_last": rf_norm_shared_with_add, "sg_not_last": rf_sg(False),
          "sg_on_leaf_not_last": rf_sg(True), "norm_not_last": rf_norm(False),
          "norm_on_leaf_not_last": rf_norm(True), "dropout_not_last": rf_dropout(False),
          "dropout_into_linear_not_last": rf_dropout(True), "norm_into_softmax_not_last": rf_norm_softmax}


def refusal_prog(name, fuse):
    """Run in a subprocess: build case `name`, forward, backward."""
    row_end, col = graph("sym")
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    ir = Recorder(m)
    REFUSE[name](ir)
    ir.adam(0.01, 0.05)
    ir.init()
    n = row_end.shape[0]
    logits_t, label_t, mask_t = ir.loss_node()["ins"]
    for t in ir.leaves:
        if t != label_t:
            m.set_tensor(t, np.random.RandomState(t).uniform(-1, 1, size=(n, ir.width[t])).astype(np.float32))
    m.set_labels(label_t, np.arange(n, dtype=np.int32) % ir.width[logits_t])
    m.set_tensor(mask_t, np.zeros(n, dtype=np.int32))
    m.train_mode(); m.zero_gradients(); m.forward()
    print("forward done", flush=True)
    m.backward()
    host.synchronize()
    print("backward done", flush=True)


RUNS = {}                  # (refusal case, fuse) -> (its process, its stdout and stderr files)


def start_refusals():
    """Every refusal case in both schedules, each in its own process (the abort ends it), all started together on
    first use: each process spends most of its time starting Python, torch and the CUDA context."""
    if RUNS:
        return
    for name in REFUSE:
        for fuse in (True, False):
            prog = "\n".join(["import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)" %
                              (ROOT, os.path.join(ROOT, "tests")),
                              "from test_opgraph_gpu import refusal_prog",
                              "refusal_prog(%r, %r)" % (name, fuse)])
            out, err = tempfile.TemporaryFile("w+"), tempfile.TemporaryFile("w+")
            RUNS[(name, fuse)] = (subprocess.Popen([sys.executable, "-c", prog], stdout=out, stderr=err, text=True,
                                                   cwd=ROOT, env=dict(os.environ)), out, err)


@atexit.register
def _stop_refusals():
    for proc, _, _ in RUNS.values():
        if proc.poll() is None:
            proc.kill()
            proc.wait()


def run_refusal(name, fuse):
    start_refusals()
    proc, out, err = RUNS[(name, fuse)]
    try:
        proc.wait(timeout=300)
    except subprocess.TimeoutExpired:
        proc.kill()
        proc.wait()
    out.seek(0), err.seek(0)
    return subprocess.CompletedProcess(proc.args, proc.returncode, out.read(), err.read())


@pytest.mark.parametrize("name", list(REFUSE))
def test_q7_refusal_is_the_same_in_both_schedules(name):
    got = {}
    for fuse in (True, False):
        p = run_refusal(name, fuse)
        assert p.returncode != 0, "%s (fuse=%s) trained where Q7 refuses:\n%s" % (name, fuse, p.stdout)
        assert p.stdout.strip().splitlines()[-1:] == ["forward done"], (fuse, p.stdout, p.stderr[-2000:])
        lines = p.stderr.strip().splitlines()
        assert len(lines) >= 3 and lines[-3].startswith("assertion failed: resetInputGrads[0]"), p.stderr[-2000:]
        got[fuse] = lines[-3:-1]
    assert got[True] == got[False], got
    SEEN.add("refusal:" + name)


# ------------------------------------------------------------------------------------------------ (f) coverage ---
def test_opgraph_covered():
    """Every op kind, fusion, near-miss and width class was reached (run the whole file: this test comes last)."""
    want = {"op:" + k for k in _lib.HOST_OPS} | {"op:linear_relu", "op:linear_none", "op:layer_norm"}
    want |= {"fusion:" + f for f in ("linear_norm_sg", "sg_norm", "sg_norm_relu", "dropout_linear", "norm_softmax",
                                     "norm_relu_linear", "norm_relu_dropout_linear", "batch_norm_relu", "teleport",
                                     "teleport_norm_out", "layer_norm_relu", "gcn_block_edge_dropout",
                                     "teleport_edge_dropout")}
    want |= {"attn_dropout", "edge_dropout", "loss:sigmoid", "bf16:features", "bf16:aggregation",
             "scaled_add_shared_reader"}
    want |= {"mode:" + m for m in ("gat", "dynamic", "softmax", "dot")}
    want |= {"temperature:learned", "temperature:constant", "cut_rows_infer:softmax", "cut_rows_infer:dot"}
    want |= {"alias:" + a for a in ("xl_is_xr", "q_is_k_is_v", "q_is_k", "k_is_v")}
    want |= {"gather_input_also_read_before", "gather_input_also_read_after"}
    want |= {"near:" + n for n in NEAR} | {"shared:" + s for s in SHARED} | {"exact:" + e for e in EXACT}
    want |= {"refusal:" + r for r in REFUSE} | {"random", "graph:hub"}
    want |= {"width:" + w for w in ("linear_in_not_float4", "linear_out_over_128", "sg_H_not_float4", "sg_65_128",
                                    "sg_129_256")}
    want |= {"width:softmax_C_%d" % c for c in CLASSES}
    missing = sorted(want - SEEN)
    assert not missing, missing
    print("\nworst |error| / bound: %s; %.0f s" % (", ".join("%s %.3f" % kv for kv in sorted(WORST.items())),
                                                  time.time() - T0))
