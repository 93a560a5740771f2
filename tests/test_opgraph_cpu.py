"""The fp64 op-graph interpreter (tests/opgraph.py) pinned against every hand witness of the composed models, and
against the fp32 oracle's GCN with dropout.  The IR comes from the model builders of roc_b200.model run on a
Recorder with no product behind it, so it also pins the recorder's layer numbering (the dropout keys)."""
import numpy as np
import pytest
import torch

import appnp_witness
import attn_dropout_oracle as ado
import edge_dropout_witness
import gatv2_witness
import layernorm_witness
import softmax_aggr_witness
import transformer_witness
from conftest import rel_close
from oracle import oracle
from opgraph import Recorder, witness
from roc_b200 import _lib, datasets
from roc_b200.model import (build_appnp, build_deepergcn, build_gat, build_gatv2, build_gcn, build_gcn_weighted,
                            build_gcnii, build_graph_transformer, build_sage_mean, build_sage_pool)
from test_attn_dropout_cpu import _sym_graph
from test_attn_dropout_gpu import witness as attn_dropout_witness
from test_batchnorm_cpu import BUILDERS as BN_BUILDERS
from test_batchnorm_gpu import _bce_train_loss, bn_witness
from test_gat_heads_gpu import witness as gat_heads_witness
from witness import torch_witness
from witness_exact import gcn_sage_witness
from witness_gat import gat_witness
from witness_pool import sage_pool_witness
from witness_weighted import gcn_weighted_witness


def case(layers, n=120, pairs=400, seed=2, directed=False):
    re_t, col_t = datasets.uniform_graph(n, pairs, seed=seed, directed=directed)
    feats, labels, mask = datasets.node_data(n, layers[0], layers[-1], seed=seed)
    return (re_t.numpy().astype(np.uint64), col_t.numpy().astype(np.uint32), feats.numpy(), labels.numpy(),
            mask.numpy())


def glorot(ir, seed=4):
    rng = np.random.RandomState(seed)
    ws = []
    for nd in ir.nodes:
        if nd["kind"] == "linear":
            i, o = ir.width[nd["ins"][0]], nd["attrs"]["out_dim"]
            s = np.sqrt(6.0 / (i + o))
            ws.append(rng.uniform(-s, s, size=(o, i)).astype(np.float32))
    return ws


def close12(a, b, what):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, what
    assert np.abs(a - b).max() <= 1e-12 * max(np.abs(b).max(), 1e-300), what


def check(ir, got, want_logits, want_dw, what):
    close12(got["logits"], want_logits, what + " logits")
    assert len(got["dW"]) == len(want_dw) == ir.params
    for p, (a, b) in enumerate(zip(got["dW"], want_dw)):
        close12(a, b, what + " dW[%d]" % p)


@pytest.mark.parametrize("layers", [(10, 16, 5), (10, 16, 12, 5)], ids=["2layer", "3layer_residual"])
def test_gcn_matches_the_witnesses(layers):
    row_end, col, feats, labels, mask = case(layers)
    ir = Recorder()
    h = build_gcn(ir, list(layers), 0.0)
    ws = glorot(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    check(ir, got, *torch_witness("gcn", row_end, col, feats, labels, mask, layers, ws), what="torch_witness")
    check(ir, got, *gcn_sage_witness("gcn", row_end, col, feats, labels, mask, layers, ws), what="gcn_sage_witness")
    assert h["logits"] == ir.loss_node()["ins"][0]


@pytest.mark.parametrize("layers", [(10, 16, 5), (10, 16, 12, 5)])
def test_sage_mean_matches_the_witnesses(layers):
    row_end, col, feats, labels, mask = case(layers)
    ir = Recorder()
    build_sage_mean(ir, list(layers), 0.0)
    ws = glorot(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    check(ir, got, *torch_witness("sage", row_end, col, feats, labels, mask, layers, ws), what="torch_witness")
    check(ir, got, *gcn_sage_witness("sage_mean", row_end, col, feats, labels, mask, layers, ws),
          what="gcn_sage_witness")


def test_gcn_on_a_directed_multigraph_matches_the_witness():
    """Duplicate edges count twice in the aggregation and in the in-degree."""
    layers = (10, 16, 5)
    row_end, col, feats, labels, mask = case(layers, directed=True)
    col = col.copy()
    col[1::5] = col[0::5][:col[1::5].shape[0]]                 # duplicates (within a row or not: both are edges)
    ir = Recorder()
    build_gcn(ir, list(layers), 0.0, exact_backward=True)
    assert ir.exact
    ws = glorot(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    check(ir, got, *gcn_sage_witness("gcn", row_end, col, feats, labels, mask, layers, ws), what="gcn_sage_witness")


@pytest.mark.parametrize("aggr", [_lib.AGGR_MAX, _lib.AGGR_MIN], ids=["max", "min"])
def test_sage_pool_matches_the_witness(aggr):
    layers = (10, 16, 12, 5)
    row_end, col, feats, labels, mask = case(layers)
    ir = Recorder()
    build_sage_pool(ir, list(layers), 0.0, aggr=aggr)
    ws = glorot(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    wl, wdw, chosen, _ = sage_pool_witness(row_end, col, feats, labels, mask, layers, ws, aggr == _lib.AGGR_MAX)
    check(ir, got, wl, wdw, what="sage_pool_witness")
    # the product's choice is taken where it differs only at a tie; a choice away from a tie is refused
    pools = [n["layer"] for n in ir.nodes if n["kind"].startswith("scatter_gather_m")]
    again = witness(ir, (row_end, col), feats, labels, mask, ws, aggr_args=dict(zip(pools, chosen)))
    check(ir, again, wl, wdw, what="sage_pool_witness, given its own choice")
    bad = chosen[0].copy()
    bad[3, 0] = col[int(row_end[2])] if bad[3, 0] != col[int(row_end[2])] else col[int(row_end[2]) + 1]
    with pytest.raises(AssertionError, match="away from a tie"):
        witness(ir, (row_end, col), feats, labels, mask, ws, aggr_args={pools[0]: bad})


@pytest.mark.parametrize("heads", [1, 4])
def test_gat_matches_the_witness(heads):
    layers = (10, 16, 5)
    row_end, col, feats, labels, mask = case(layers)
    ir = Recorder()
    build_gat(ir, list(layers), 0.0, heads=heads)
    ws = glorot(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    # the interpreter takes the product's fp32 slope
    check(ir, got, *gat_witness(row_end, col, feats, labels, mask, layers, ws, [heads], slope=float(np.float32(0.2))),
          what="gat_witness")


def test_weighted_gcn_matches_the_witness():
    layers = (10, 16, 12, 5)
    row_end, col, feats, labels, mask = case(layers, directed=True)
    w = datasets.gcn_edge_weights(row_end, col, np.random.RandomState(1).uniform(0.2, 3.0, size=col.shape[0]))
    ir = Recorder()
    h = build_gcn_weighted(ir, list(layers), 0.0, w, edge_grad=True)
    assert ir.edge_grad == {h["edges"]: True}
    ws = glorot(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws, edge_values={h["edges"]: w})
    wl, wdw, wde = gcn_weighted_witness(row_end, col, feats, labels, mask, layers, ws, w)
    check(ir, got, wl, wdw, what="gcn_weighted_witness")
    close12(got["edge_grad"][h["edges"]], wde, "edge gradient")


def test_relu_mask_is_taken_only_at_a_tie():
    layers = (10, 16, 5)
    row_end, col, feats, labels, mask = case(layers)
    ir = Recorder()
    build_gcn(ir, list(layers), 0.0)
    ws = glorot(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    (layer, pre), = got["pre"].items()
    assert ir.nodes[layer]["kind"] == "relu"
    again = witness(ir, (row_end, col), feats, labels, mask, ws, relu_masks={layer: pre > 0})
    check(ir, again, got["logits"], got["dW"], what="given its own mask")
    flipped = pre > 0
    k = np.unravel_index(np.abs(pre).argmax(), pre.shape)
    flipped[k] = not flipped[k]
    with pytest.raises(AssertionError, match="away from zero"):
        witness(ir, (row_end, col), feats, labels, mask, ws, relu_masks={layer: flipped})


@pytest.mark.parametrize("layers", [(10, 16, 5), (10, 16, 12, 5)], ids=["2layer", "3layer_residual"])
def test_gcn_with_dropout_matches_the_oracle(layers):
    """Dropout 0.5 over three steps: the keep masks (key (seed << 32) | layer index, the step counter from 1) and the
    fp32 scale are the oracle's; logits and dW agree to the fp32 parity bar."""
    row_end, col, feats, labels, mask = case(layers)
    ir = Recorder()
    build_gcn(ir, list(layers), 0.5)
    assert [n["attrs"]["key"] for n in ir.nodes if n["kind"] == "dropout"] == \
        [oracle.GcnOracle(row_end, col, layers, glorot(ir))._dropout_op_index(i) for i in range(1, len(layers))]
    ws = glorot(ir)
    o = oracle.GcnOracle(row_end, col, layers, ws, dropout=0.5)
    for step in range(1, 4):
        w0 = [w.copy() for w in o.W]
        o.forward(feats, train=True)
        o.backward(datasets.onehot(labels, layers[-1]), mask)
        got = witness(ir, (row_end, col), feats, labels, mask, w0, step=step)
        rel_close(got["logits"], o.logits, what="step %d logits" % step)
        for p, (a, b) in enumerate(zip(got["dW"], o.dW)):
            rel_close(a, b, rtol=2e-4, atol_scale=2e-5, what="step %d dW[%d]" % (step, p))
        o.update()
    # a different step draws a different mask
    a = witness(ir, (row_end, col), feats, labels, mask, ws, step=1)["logits"]
    b = witness(ir, (row_end, col), feats, labels, mask, ws, step=2)["logits"]
    assert np.abs(a - b).max() > 1e-3


# --------------------------------------------- the ops added since: each feature's own reference, on its builders ---
def draw(ir, seed=4):
    """A value for every parameter, in the shapes get_parameter gives them: a Linear's W (out, in), an
    attention_scores' A (2 * heads, F), a dynamic gather's a (F, heads), a learned temperature (1, 1), a batch_norm's
    or layer_norm's gamma and beta (1, H) (gamma near 1)."""
    rng = np.random.RandomState(seed)
    ws = [None] * ir.params
    for nd in ir.nodes:
        a = nd["attrs"]
        if nd["kind"] == "linear":
            i, o = ir.width[nd["ins"][0]], a["out_dim"]
            s = np.sqrt(6.0 / (i + o))
            ws[a["param"]] = rng.uniform(-s, s, size=(o, i))
        elif nd["kind"] == "attention_scores":
            hd = a["heads"]
            ws[a["param"]] = rng.uniform(-0.5, 0.5, size=(2 * hd, ir.width[nd["ins"][0]] // hd))
        elif nd["kind"] == "attention_gather" and a["mode"] == "dynamic":
            hd = a["heads"]
            ws[a["param"]] = rng.uniform(-0.5, 0.5, size=(ir.width[nd["ins"][0]] // hd, hd))
        elif nd["kind"] == "attention_gather" and a["mode"] == "softmax" and a["learn"]:
            ws[a["param"]] = rng.uniform(0.5, 2.0, size=(1, 1))
        elif nd["kind"] in ("batch_norm", "layer_norm"):
            h = ir.width[nd["out"]]
            ws[a["gamma"]] = rng.uniform(0.5, 1.5, size=(1, h))
            ws[a["beta"]] = rng.uniform(-0.3, 0.3, size=(1, h))
    return [w.astype(np.float32) for w in ws]


def bn_case(name, loss="softmax", features="float32"):
    """A builder of test_batchnorm_cpu.BUILDERS with norm="batch" on a recorder, and inputs for it (12 classes)."""
    n = 120
    re_t, col_t = datasets.uniform_graph(n, 400, seed=2)
    row_end, col = re_t.numpy().astype(np.uint64), col_t.numpy().astype(np.uint32)
    data = datasets.multilabel_node_data if loss == "sigmoid" else datasets.node_data
    feats, labels, mask = (t.numpy() for t in data(n, 24, 12, seed=2))
    w = np.random.RandomState(1).uniform(0.05, 0.6, size=col.shape[0]).astype(np.float32)
    ir = Recorder()
    kw = dict(edge_weights=w) if name == "gcn_weighted" else {}
    h = BN_BUILDERS[name](ir, norm="batch", loss=loss, features=features, **kw)
    return ir, h, (row_end, col), feats, labels, mask, {e: w for e in ir.edges}


@pytest.mark.parametrize("name", ["gcn", "gcn4", "sage_mean", "sage_pool", "gat", "gcn_weighted"])
def test_batch_norm_matches_bn_witness(name):
    """Train (batch statistics, dropout at step 2) and infer (running statistics, dropout a copy)."""
    ir, h, graph, feats, labels, mask, ev = bn_case(name)
    ws = draw(ir)
    got = witness(ir, graph, feats, labels, mask, ws, edge_values=ev, step=2)
    want = bn_witness(ir, graph, feats, labels, mask, ws, None, edge_values=ev, step=2)
    check(ir, got, want["logits"], want["dW"], what="bn_witness")
    assert sorted(got["stats"]) == sorted(h["bns"]) == sorted(want["stats"])
    for t, (mean, var) in want["stats"].items():
        close12(got["stats"][t][0], mean.numpy(), "batch mean")
        close12(got["stats"][t][1], var.numpy(), "batch var")
    rng = np.random.RandomState(3)
    run = {t: (rng.uniform(-1, 1, ir.width[t]), rng.uniform(0.5, 2, ir.width[t])) for t in h["bns"]}
    got = witness(ir, graph, feats, labels, mask, ws, edge_values=ev, training=False, run_stats=run)
    want = bn_witness(ir, graph, feats, labels, mask, ws, run, training=False, edge_values=ev)
    close12(got["logits"], want["logits"], "infer logits")
    assert not any(np.any(d) for d in got["dW"]), "infer mode differentiates nothing"


def test_sigmoid_loss_and_bf16_features_match_bn_witness():
    ir, h, graph, feats, labels, mask, ev = bn_case("gcn", loss="sigmoid", features="bfloat16")
    assert ir.loss_node()["kind"] == "sigmoid_cross_entropy" and ir.bf16 == {h["input"]}
    ws = draw(ir)
    got = witness(ir, graph, feats, labels, mask, ws, step=1)
    rounded = torch.from_numpy(feats).bfloat16().double().numpy()
    assert np.abs(rounded - feats).max() > 0                       # the rounding is visible
    want = bn_witness(ir, graph, rounded, labels, mask, ws, None, loss_fn=_bce_train_loss)
    check(ir, got, want["logits"], want["dW"], what="bn_witness, sigmoid loss")


@pytest.mark.parametrize("name", ["appnp", "gcnii"])
def test_appnp_and_gcnii_match_appnp_witness(name):
    row_end, col, feats, labels, mask = case((24, 16, 12))
    ir = Recorder()
    if name == "appnp":
        build_appnp(ir, [24, 16, 12], 0.5, K=4, alpha=0.1)
    else:
        build_gcnii(ir, [24, 16, 12], 0.5, 3, alpha=0.1, theta=0.5)
    assert any(nd["kind"] == "scaled_add" for nd in ir.nodes)
    ws = draw(ir)
    for step in (1, 3):
        got = witness(ir, (row_end, col), feats, labels, mask, ws, step=step)
        want = appnp_witness.witness(ir, (row_end, col), feats, labels, mask, ws, step=step)
        check(ir, got, want["logits"], want["dW"], what="appnp_witness step %d" % step)
    got = witness(ir, (row_end, col), feats, labels, mask, ws, training=False)
    want = appnp_witness.witness(ir, (row_end, col), feats, labels, mask, ws, training=False)
    close12(got["logits"], want["logits"], "infer logits")


@pytest.mark.parametrize("norm", [None, "batch"])
def test_paper_gat_matches_the_gat_heads_witness(norm):
    """Per-head attention_scores, ELU, dropout 0.5 (and a batch_norm before each ELU)."""
    row_end, col, feats, labels, mask = case((24, 16, 32, 12))
    ir = Recorder()
    build_gat(ir, [24, 16, 32, 12], 0.5, heads=[2, 8], scores="per_head", activation="elu", norm=norm)
    assert {"attention_scores", "elu"} <= {nd["kind"] for nd in ir.nodes}
    ws = draw(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws, step=2)
    logits, dw = gat_heads_witness(ir, (row_end, col), feats, labels, mask, ws, step=2)
    check(ir, got, logits, dw, what="test_gat_heads_gpu.witness")


def test_paper_gat_with_attention_dropout_matches_its_witness():
    row_end, col, feats, labels, mask = case((24, 16, 32, 12))
    ir = Recorder()
    build_gat(ir, [24, 16, 32, 12], 0.5, heads=[2, 8], scores="per_head", activation="elu", attn_dropout=0.6)
    ws = draw(ir)
    for step in (1, 2):
        got = witness(ir, (row_end, col), feats, labels, mask, ws, step=step)
        logits, dw = attn_dropout_witness(ir, (row_end, col), feats, labels, mask, ws, step, None)
        check(ir, got, logits, dw, what="test_attn_dropout_gpu.witness step %d" % step)
    # infer mode: no attention dropout, no dropout
    plain = Recorder()
    build_gat(plain, [24, 16, 32, 12], 0.0, heads=[2, 8], scores="per_head", activation="elu")
    a = witness(ir, (row_end, col), feats, labels, mask, ws, training=False)["logits"]
    close12(a, witness(plain, (row_end, col), feats, labels, mask, ws)["logits"], "infer = the undropped model")


@pytest.mark.parametrize("heads,f", [(1, 5), (2, 4), (8, 4)])
def test_attention_dropout_matches_attn_dropout_oracle(heads, f):
    """attention_gather(wh, sc, dropout=0.6, seed=5) read straight into the loss: its forward is
    attn_dropout_oracle.forward with the step's key (seed << 32) | layer, and the gradients its two Linears see
    are attn_dropout_oracle.backward's."""
    n, rate, step = 60, 0.6, 3
    row_end, col = _sym_graph(n, 150, heads)
    ir = Recorder()
    x0 = ir.create_node_tensor(7)
    wh, sc = ir.linear(x0, heads * f), ir.linear(x0, 2 * heads)
    out = ir.attention_gather(wh, sc, heads=heads, dropout=rate, seed=5)
    ir.softmax_cross_entropy(out, ir.create_node_tensor(heads * f), ir.create_node_tensor(1, is_int=True))
    assert ir.nodes[2]["attrs"]["key"] == (5 << 32) | 2
    rng = np.random.RandomState(heads)
    x = rng.uniform(-1, 1, size=(n, 7))
    ws = [rng.uniform(-1, 1, size=(heads * f, 7)), rng.uniform(-1, 1, size=(2 * heads, 7))]
    labels, mask = rng.randint(0, heads * f, size=n), rng.randint(0, 3, size=n)
    got = witness(ir, (row_end, col), x, labels, mask, ws, step=step)
    key = (5 << 32) | 2
    m1 = ado.multipliers(ado.edge_keep(row_end, col, rate, key, step), heads, rate)
    m2 = ado.multipliers(ado.edge_keep(row_end, col, rate, key, step, row_is_source=True), heads, rate)
    xw, s, slope = x @ ws[0].T, x @ ws[1].T, float(np.float32(0.2))
    o, stats = ado.forward(row_end, col, xw, s, heads, slope, m1)
    close12(got["logits"], o, "forward")
    p = np.exp(o - o.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    gy = np.where((mask == _lib.MASK_TRAIN)[:, None], p - np.eye(heads * f)[labels], 0.0)
    ig, sg = ado.backward(row_end, col, xw, s, o, stats, gy, heads, slope, m1, m2)
    np.testing.assert_allclose(got["dW"][0], ig.T @ x, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(got["dW"][1], sg.T @ x, rtol=1e-10, atol=1e-12)


# ------------------------- edge dropout, GATv2, softmax aggregation, layer norm, dot attention: their own witnesses ---
@pytest.mark.parametrize("share_weights", [False, True])
def test_gatv2_matches_gatv2_witness(share_weights):
    row_end, col, feats, labels, mask = case((24, 16, 12))
    ir = Recorder()
    h = build_gatv2(ir, [24, 16, 12], 0.0, heads=2, share_weights=share_weights)
    assert [n["attrs"]["mode"] for n in ir.nodes if n["kind"] == "attention_gather"] == ["dynamic", "dynamic"]
    assert all(xl == xr for xl, xr in h["attn_ins"]) == share_weights
    ws = draw(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    # the interpreter takes the product's fp32 slope; a is (F, heads) as get_parameter returns it
    logits, dw = gatv2_witness.model_witness(row_end, col, feats, labels, mask, (24, 16, 12), ws, [2],
                                             share_weights=share_weights, slope=float(np.float32(0.2)))
    check(ir, got, logits, dw, what="gatv2_witness")


@pytest.mark.parametrize("norm", ["batch", "layer_norm"])
@pytest.mark.parametrize("learn", [True, False])
def test_deepergcn_matches_its_witnesses(learn, norm):
    """softmax_aggr_witness.model_witness for batch norm, layernorm_witness.deepergcn_witness for layer norm; a
    constant temperature of -0.5 leans towards the min."""
    row_end, col, feats, labels, mask = case((24, 16, 12))
    ir = Recorder()
    temperature = 1.0 if learn else -0.5
    h = build_deepergcn(ir, [24, 16, 12], 0.0, 3, temperature=temperature, learn_temperature=learn, norm=norm)
    modes = [n["attrs"] for n in ir.nodes if n["kind"] == "attention_gather"]
    assert [a["mode"] for a in modes] == ["softmax"] * 3 and [a["param"] for a in modes] == h["temperatures"]
    ws = draw(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    if norm == "batch":
        logits, dw = softmax_aggr_witness.model_witness(row_end, col, feats, labels, mask, (24, 16, 12), ws, 3,
                                                        learn_temperature=learn, temperature=temperature)
    else:
        logits, dw = layernorm_witness.deepergcn_witness(row_end, col, feats, labels, mask, (24, 16, 12), ws, 3,
                                                         learn_temperature=learn, temperature=temperature)
    check(ir, got, logits, dw, what="deepergcn witness")


@pytest.mark.parametrize("root_weight", [True, False])
def test_graph_transformer_matches_transformer_witness(root_weight):
    row_end, col, feats, labels, mask = case((24, 16, 12))
    ir = Recorder()
    build_graph_transformer(ir, [24, 16, 12], 0.0, heads=2, root_weight=root_weight, norm="layer_norm")
    ws = draw(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    logits, dw = transformer_witness.model_witness(row_end, col, feats, labels, mask, (24, 16, 12), ws, [2],
                                                   root_weight=root_weight, norm="layer_norm")
    check(ir, got, logits, dw, what="transformer_witness")


def test_dot_attention_default_scale_comes_from_the_widths():
    """No product behind the recorder: the default scale is fp32(1 / sqrt(F)) from the recorder's own widths."""
    ir = Recorder()
    q = ir.create_node_tensor(24)
    ir.dot_attention_gather(q, q, q, heads=8)
    ir.dot_attention_gather(q, q, q, heads=2, scale=0.3)
    assert [n["attrs"]["scale"] for n in ir.nodes] == [transformer_witness.dot_scale(3), float(np.float32(0.3))]


@pytest.mark.parametrize("name", ["gcn", "gcn_residual", "appnp"])
def test_edge_dropout_matches_edge_dropout_witness(name):
    """Three steps of keep masks: the keys (seed << 32) | layer and the step counter pin the recorder's layer
    numbering; infer mode drops nothing."""
    layers = (24, 16, 16, 12) if name == "gcn_residual" else (24, 16, 12)
    row_end, col, feats, labels, mask = case(layers)
    ir = Recorder()
    if name == "appnp":
        build_appnp(ir, list(layers), 0.0, K=3, edge_dropout=0.5)
    else:
        build_gcn(ir, list(layers), 0.0, edge_dropout=0.5)
    sgs = [n for n in ir.nodes if n["kind"] == "scatter_gather"]
    assert sgs and all(n["attrs"]["key"] == n["layer"] and n["attrs"]["dropout"] == 0.5 for n in sgs)
    ws = draw(ir)
    for step in (1, 2, 3):
        got = witness(ir, (row_end, col), feats, labels, mask, ws, step=step)
        want = edge_dropout_witness.witness(ir, (row_end, col), feats, labels, mask, ws, step=step)
        check(ir, got, want["logits"], want["dW"], what="edge_dropout_witness step %d" % step)
    got = witness(ir, (row_end, col), feats, labels, mask, ws, training=False)
    want = edge_dropout_witness.witness(ir, (row_end, col), feats, labels, mask, ws, training=False)
    close12(got["logits"], want["logits"], "infer logits")
    a = witness(ir, (row_end, col), feats, labels, mask, ws, step=1)["logits"]
    assert np.abs(a - got["logits"]).max() > 1e-3, "edge dropout changed nothing"


LN_BUILDERS = {"gcn4": lambda ir: build_gcn(ir, [24, 16, 16, 12], 0.0, norm="layer_norm"),
               "sage_mean": lambda ir: build_sage_mean(ir, [24, 16, 16, 12], 0.0, norm="layer_norm"),
               "gat": lambda ir: build_gat(ir, [24, 16, 12], 0.0, heads=2, norm="layer_norm")}


@pytest.mark.parametrize("name", list(LN_BUILDERS))
def test_layer_norm_matches_layernorm_witness(name):
    row_end, col, feats, labels, mask = case((24, 16, 12))
    ir = Recorder()
    h = LN_BUILDERS[name](ir)
    assert h["bns"] and [n["out"] for n in ir.nodes if n["kind"] == "layer_norm"] == h["bns"]
    ws = draw(ir)
    got = witness(ir, (row_end, col), feats, labels, mask, ws)
    want = layernorm_witness.graph_witness(ir, (row_end, col), feats, labels, mask, ws)
    check(ir, got, want["logits"], want["dW"], what="layernorm_witness")
    assert not got["stats"], "a layer norm keeps no batch statistics"
