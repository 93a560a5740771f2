"""tests/scale_witness.py pinned on the CPU: the models bench.py benchmarks (configs 1-5, recorded by bench.build_model
on a Recorder with no product behind it) at their real layer widths on small graphs of each config's kind, against
opgraph.witness to 1e-12 with dropout 0.5 at steps 1 and 2, with every aggregation and dropout mask cut into several
chunks; the aggregation's backward against autograd of the dense A on a directed graph; the loss metrics against the
fp32 oracle on rows with exact ties; and the refusal of every other op."""
import numpy as np
import pytest
import torch

from bench_inputs import bench_module
from oracle import oracle
from opgraph import Recorder, witness
from roc_b200 import datasets
from roc_b200.model import build_gat, build_gcn_weighted, build_sage_pool
from scale_witness import Aggregate, SUPPORTED, metrics, scale_witness

B = bench_module()


def small_graph(cfg):
    """a graph of config cfg's kind with 120-400 vertices"""
    g = B.CONFIGS[cfg]["graph"]
    if g == "uniform":
        re_t, col_t = datasets.uniform_graph(150, 700, seed=3)
    elif g == "rmat":
        re_t, col_t = datasets.rmat_graph(8, 1500, seed=3)
    elif g == "products":
        re_t, col_t = datasets.powerlaw_graph(400, 3000, alpha=1.6, seed=3)
    else:                                             # Reddit-shaped: dense rows
        re_t, col_t = datasets.powerlaw_graph(200, 9000, alpha=1.3, seed=3)
    return re_t.numpy().astype(np.uint64), col_t.numpy().astype(np.uint32)


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


@pytest.mark.parametrize("cfg", sorted(B.CONFIGS))
def test_bench_models_record_only_supported_ops(cfg):
    """bench.build_model's IR at the config's real widths: every op is one the witness covers, and the Linear widths
    are the config's."""
    ir = Recorder(None)
    h = B.build_model(ir, cfg)
    assert {n["kind"] for n in ir.nodes} <= set(SUPPORTED)
    assert h["logits"] == ir.loss_node()["ins"][0]
    layers = B.CONFIGS[cfg]["layers"]
    outs = [n["attrs"]["out_dim"] for n in ir.nodes if n["kind"] == "linear"]
    per = 1 if len(outs) == len(layers) - 1 else 2       # GraphSAGE-mean and the residual GCN: two Linears a layer
    assert outs == [d for d in layers[1:] for _ in range(per)]


@pytest.mark.parametrize("cfg", sorted(B.CONFIGS))
def test_matches_opgraph_witness_with_dropout(cfg):
    """Each bench model at its real widths on a small graph of its kind, dropout 0.5 (bench.DROPOUT), steps 1 and 2:
    logits, every dW and the ReLU pre-activations to 1e-12.  Chunks of 97 edges and 23 rows put every aggregation
    and every mask in several chunks; the graphs' sizes are not multiples of them, so the last chunks are partial."""
    assert B.DROPOUT == 0.5
    row_end, col = small_graph(cfg)
    n = row_end.shape[0]
    assert 120 <= n <= 400
    layers = B.CONFIGS[cfg]["layers"]
    ir = Recorder(None)
    B.build_model(ir, cfg)
    feats, labels, mask = datasets.node_data(n, layers[0], layers[-1], seed=cfg)
    feats, labels, mask = feats.numpy(), labels.numpy(), mask.numpy()
    ws = glorot(ir, seed=cfg)
    for step in (1, 2):
        want = witness(ir, (row_end, col), feats, labels, mask, ws, step=step)
        got = scale_witness(ir, (row_end, col), feats, labels, mask, ws, step=step, edge_chunk=97, mask_rows=23)
        close12(got["logits"], want["logits"], "cfg %d step %d logits" % (cfg, step))
        assert len(got["dW"]) == len(want["dW"]) == ir.params
        for p, (a, b) in enumerate(zip(got["dW"], want["dW"])):
            close12(a, b, "cfg %d step %d dW[%d]" % (cfg, step, p))
        assert sorted(got["pre"]) == sorted(want["pre"]) and got["pre"]
        for layer in want["pre"]:
            close12(got["pre"][layer], want["pre"][layer], "cfg %d step %d pre[%d]" % (cfg, step, layer))
        aggs = [c for c in got["chunks"] if c[0] == "aggregate"]
        masks = [c for c in got["chunks"] if c[0] == "dropout mask"]
        assert len(aggs) == 2 * sum(n["kind"] == "scatter_gather" for n in ir.nodes)     # forward and backward
        assert len(masks) == sum(n["kind"] == "dropout" for n in ir.nodes)
        assert all(c[1] >= 3 for c in aggs + masks), got["chunks"]
        assert all(0 < c[2] < c[3] for c in aggs + masks), got["chunks"]                   # partial last chunks
    # the same model with its mask taken from the previous step differs: the step reaches every mask
    other = scale_witness(ir, (row_end, col), feats, labels, mask, ws, step=1, edge_chunk=97, mask_rows=23)
    assert np.abs(other["logits"] - got["logits"]).max() > 1e-3


def test_chunk_size_does_not_matter_and_one_chunk_is_exact():
    """One chunk holding every edge and row, and chunks that divide the sizes exactly, give the same result."""
    row_end, col = small_graph(5)
    n, e = row_end.shape[0], col.shape[0]
    layers = B.CONFIGS[5]["layers"]
    ir = Recorder(None)
    B.build_model(ir, 5)
    feats, labels, mask = (t.numpy() for t in datasets.node_data(n, layers[0], layers[-1], seed=1))
    ws = glorot(ir)
    whole = scale_witness(ir, (row_end, col), feats, labels, mask, ws, step=1, edge_chunk=e, mask_rows=n)
    assert all(c[1] == 1 for c in whole["chunks"])
    d_e = next(d for d in range(7, e) if e % d == 0)
    d_n = next(d for d in range(7, n) if n % d == 0)
    even = scale_witness(ir, (row_end, col), feats, labels, mask, ws, step=1, edge_chunk=d_e, mask_rows=d_n)
    assert all(c[2] == c[3] for c in even["chunks"])
    close12(even["logits"], whole["logits"], "logits")
    for a, b in zip(even["dW"], whole["dW"]):
        close12(a, b, "dW")


def test_dw_bound_and_dy_leave_the_result_unchanged():
    """The dW error bound and the kept dL/dY come from hooks that change nothing.  dY^T X rebuilds dW[0] from the
    kept dY and the dropped features; the bound has dW's shape, holds an fp32 GEMM of the same operands, and is not
    loose: it is under 1e-3 of max|dW|."""
    row_end, col = small_graph(2)
    n = row_end.shape[0]
    layers = B.CONFIGS[2]["layers"]
    ir = Recorder(None)
    B.build_model(ir, 2)
    feats, labels, mask = (t.numpy() for t in datasets.node_data(n, layers[0], layers[-1], seed=1))
    ws = glorot(ir)
    plain = scale_witness(ir, (row_end, col), feats, labels, mask, ws, step=1)
    got = scale_witness(ir, (row_end, col), feats, labels, mask, ws, step=1, dw_split={0: 64, 1: 32}, keep_dy=(0,))
    close12(got["logits"], plain["logits"], "logits")
    for a, b in zip(got["dW"], plain["dW"]):
        close12(a, b, "dW")
    assert sorted(got["dW_bound"]) == [0, 1] and sorted(got["dy"]) == [0]
    drop = next(nd for nd in ir.nodes if nd["kind"] == "dropout")["attrs"]
    keep = oracle.dropout_mask(0, n, layers[0], drop["rate"], drop["key"], 1).astype(np.float64)
    x = feats.astype(np.float64) * keep * 2.0
    close12(got["dy"][0].T @ x, plain["dW"][0], "dY^T X")
    for p in (0, 1):
        bnd, dw = got["dW_bound"][p], plain["dW"][p]
        assert bnd.shape == dw.shape and (bnd > 0).all()
        assert bnd.max() <= 1e-3 * np.abs(dw).max()
    dw32 = got["dy"][0].astype(np.float32).T @ x.astype(np.float32)
    assert (np.abs(dw32 - plain["dW"][0]) <= got["dW_bound"][0]).all()


def test_aggregation_backward_is_the_transpose_on_a_directed_graph():
    """On a directed graph (A != A^T) the aggregation's gradient equals autograd through the dense A @ x (tests/
    witness.py's construction), and differs from A @ g: a backward that assumed symmetry would fail here."""
    re_t, col_t = datasets.uniform_graph(90, 400, seed=5, directed=True)
    row_end, col = re_t.numpy().astype(np.int64), col_t.numpy().astype(np.int64)
    n = row_end.shape[0]
    deg = np.diff(np.concatenate([[0], row_end]))
    dst = np.repeat(np.arange(n), deg)
    a = torch.zeros((n, n), dtype=torch.float64)
    a[torch.from_numpy(dst), torch.from_numpy(col)] = 1.0
    assert not torch.equal(a, a.T)
    rng = np.random.RandomState(6)
    x0 = torch.from_numpy(rng.randn(n, 12))
    g = torch.from_numpy(rng.randn(n, 12))
    x = x0.clone().requires_grad_(True)
    y = Aggregate.apply(x, torch.from_numpy(dst), torch.from_numpy(col), 17, [])
    y.backward(g)
    xd = x0.clone().requires_grad_(True)
    yd = a @ xd
    yd.backward(g)
    close12(y.detach(), yd.detach(), "forward")
    close12(x.grad, xd.grad, "backward")
    assert (x.grad - a @ g).abs().max() > 1e-3


def test_metrics_match_the_oracle_with_exact_ties():
    """trainLoss (the sum of 1 - P[true], not the cross-entropy), the three row counts and the three correct-counts
    against oracle.softmax_xent_bwd, on rows whose largest logits tie exactly: the first maximum is the prediction."""
    rng = np.random.RandomState(7)
    n, c = 600, 7
    logits = (rng.randn(n, c) * 2).astype(np.float32)
    labels = rng.randint(0, c, size=n).astype(np.int32)
    mask = rng.randint(0, 3, size=n).astype(np.int32)
    tie = np.arange(0, n, 3)
    j = rng.randint(0, c - 1, size=tie.shape[0])
    logits[tie, j + 1] = logits[tie, j] = logits[tie].max(axis=1) + 1.0        # two equal maxima, at j and j + 1
    labels[tie[::2]] = j[::2]                       # the first maximum is the true class: a hit
    labels[tie[1::2]] = j[1::2] + 1                 # the second one is: a miss
    _, want = oracle.softmax_xent_bwd(logits, datasets.onehot(labels, c), mask)
    got = metrics(torch.from_numpy(logits.astype(np.float64)), torch.from_numpy(labels), torch.from_numpy(mask))
    for k in ("trainAll", "valAll", "testAll", "trainCorrect", "valCorrect", "testCorrect"):
        assert got[k] == want[k], (k, got[k], want[k])
    assert abs(got["trainLoss"] - want["trainLoss"]) <= 1e-5 * abs(want["trainLoss"])
    assert got["near_ties"]["trainCorrect"] == int((mask[tie] == 0).sum())
    # not the cross-entropy
    p = torch.softmax(torch.from_numpy(logits.astype(np.float64)), 1).numpy()
    xent = -np.log(p[np.arange(n), labels])[mask == 0].sum()
    assert abs(got["trainLoss"] - xent) > 1.0


@pytest.mark.parametrize("builder", ["sage_pool", "gat", "gcn_weighted"])
def test_other_ops_are_refused_by_name(builder):
    ir = Recorder(None)
    if builder == "sage_pool":
        build_sage_pool(ir, [8, 8, 3], 0.5)
        op = "scatter_gather_max"
    elif builder == "gat":
        build_gat(ir, [8, 8, 3], 0.5)
        op = "attention_gather"
    else:
        build_gcn_weighted(ir, [8, 8, 3], 0.5, np.ones(10, dtype=np.float32))
        op = "scatter_gather_weighted"
    row_end = np.arange(1, 11, dtype=np.uint64)
    col = np.arange(10, dtype=np.uint32)
    feats, labels, mask = np.zeros((10, 8), np.float32), np.zeros(10, np.int32), np.zeros(10, np.int32)
    with pytest.raises(ValueError, match="op %s is not supported" % op):
        scale_witness(ir, (row_end, col), feats, labels, mask, glorot(ir))
