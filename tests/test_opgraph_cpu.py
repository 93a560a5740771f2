"""The fp64 op-graph interpreter (tests/opgraph.py) pinned against every hand witness of the composed models, and
against the fp32 oracle's GCN with dropout.  The IR comes from the model builders of roc_b200.model run on a
Recorder with no product behind it, so it also pins the recorder's layer numbering (the dropout keys)."""
import numpy as np
import pytest

from conftest import rel_close
from oracle import oracle
from opgraph import Recorder, witness
from roc_b200 import _lib, datasets
from roc_b200.model import build_gat, build_gcn, build_gcn_weighted, build_sage_mean, build_sage_pool
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
