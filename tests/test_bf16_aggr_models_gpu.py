"""GPU suite: bf16 aggregation inputs (aggregation="bfloat16") on the models whose aggregations are max / min,
edge-weighted or attention: GraphSAGE-pool with max and with min, GAT with one head and with 8 heads then 1, the
weighted GCN with its edge gradient, and the pool and GAT models with the exact backward on a directed multigraph.

* tensor_dtype marks exactly the tensors the rule of Model.set_bf16_aggregation derives from the recorded op graph
  (one per layer here: the pool's relu output, GAT's wh, the weighted GCN's Linear output); every other tensor stays
  fp32.
* Each bf16 tensor holds f32_to_bf16 of its producer's fp32 result on the model's own input rows, and the first
  aggregation's outputs are the fp32 kernel's on the widened bits, bit for bit.  For GAT, the score Linear's dW is
  linear_dw_bf16 on the stored bits and its dY.
* One training step at dropout 0.5 against an fp64 torch autograd interpreter of the recorded graph (witness below,
  on opgraph's op helpers), taking the product's bf16 values (each a correct rounding of the fp64 one) with
  straight-through gradients, and the product's relu masks and max / min choices where fp32 and fp64 tie: logits,
  every dW, the edge gradient, and every weight after Adam, at the bounds of the op-graph tests.
* With the mode off, a model that calls set_bf16_aggregation(False) is byte-identical to one that never calls it."""
import math

import numpy as np
import pytest
import torch

from opgraph import INNER, Recorder, _extreme_sources, _relu_with_mask
from oracle import oracle
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_gat, build_gcn_weighted, build_sage_pool
from witness_gat import attend, edge_lists, train_loss

pytestmark = pytest.mark.gpu
DEV = "cuda"
LR, WD = 0.01, 0.05
NONE, RELU = _lib.AC_MODE_NONE, _lib.AC_MODE_RELU
AGGREGATING = ("scatter_gather_max", "scatter_gather_min", "scatter_gather_weighted", "attention_gather")


def symmetric(n, pairs, seed):
    """Symmetric, deduplicated, a self loop on every node, sources strictly increasing per row."""
    rng = np.random.RandomState(seed)
    s, d = rng.randint(0, n, size=pairs), rng.randint(0, n, size=pairs)
    s, d = np.concatenate([s, d, np.arange(n)]), np.concatenate([d, s, np.arange(n)])
    key = np.unique(d.astype(np.int64) * n + s)
    d, s = key // n, key % n
    return np.cumsum(np.bincount(d, minlength=n)).astype(np.uint64), s.astype(np.uint32)


def directed(n, e, seed):
    """Directed, with duplicate edges, a heavy row and a self loop on every node."""
    rng = np.random.RandomState(seed)
    dst, src = rng.randint(0, n, size=e), (rng.zipf(1.6, size=e) - 1) % n
    src[1::4], dst[1::4] = src[0::4][:src[1::4].shape[0]], dst[0::4][:dst[1::4].shape[0]]
    dst[:150] = 9
    dst, src = np.concatenate([dst, np.arange(n)]), np.concatenate([src, np.arange(n)])
    order = np.argsort(dst, kind="stable")
    return np.cumsum(np.bincount(dst[order], minlength=n)).astype(np.uint64), src[order].astype(np.uint32)


GRAPHS = {"sym": symmetric(700, 3500, 4), "directed": directed(500, 3000, 6)}
EDGE_W = {k: np.random.RandomState(7).uniform(0.05, 0.6, size=g[1].shape[0]).astype(np.float32)
          for k, g in GRAPHS.items()}
CASES = {   # name: (graph, builder(model, dropout, aggregation))
    "pool_max": ("sym", lambda m, d, a: build_sage_pool(m, [24, 16, 7], d, aggr=_lib.AGGR_MAX, aggregation=a)),
    "pool_min": ("sym", lambda m, d, a: build_sage_pool(m, [24, 16, 7], d, aggr=_lib.AGGR_MIN, aggregation=a)),
    "gat_1head": ("sym", lambda m, d, a: build_gat(m, [24, 16, 7], d, heads=1, aggregation=a)),
    "gat_8_1heads": ("sym", lambda m, d, a: build_gat(m, [24, 64, 16, 7], d, heads=(8, 1), aggregation=a)),
    "gcn_weighted": ("sym", lambda m, d, a: build_gcn_weighted(m, [24, 16, 7], d, EDGE_W["sym"], edge_grad=True,
                                                              aggregation=a)),
    "pool_max_exact": ("directed", lambda m, d, a: build_sage_pool(m, [24, 16, 7], d, aggr=_lib.AGGR_MAX,
                                                                   exact_backward=True, aggregation=a)),
    "gat_exact": ("directed", lambda m, d, a: build_gat(m, [24, 32, 7], d, heads=(4,), exact_backward=True,
                                                        aggregation=a)),
}


def model(name, dropout, aggregation, off_call=False, weights=None):
    gkind, build = CASES[name]
    row_end, col = GRAPHS[gkind]
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    if off_call:
        m.set_bf16_aggregation(False)
    ir = Recorder(m)
    h = build(ir, dropout, aggregation)
    if weights is not None:
        for p, w in enumerate(weights):
            m.set_parameter(p, w)
    feats, labels, mask = (t.numpy() for t in datasets.node_data(n, 24, 7, seed=2))
    m.set_tensor(h["input"], feats)
    m.set_labels(h["label"], labels)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    return host, m, ir, h, dict(feats=feats, labels=labels, mask=mask, graph=(row_end, col), gkind=gkind)


def expected_bf16(ir):
    """From the recorded graph (no sum aggregation in these models, so only the rule for the other kinds): each output
    of a Linear(NONE) or a relu that some max / min, weighted or attention aggregation reads as its input 0 and that
    nothing else reads but those and Linears (a Linear reading it directly has no fused dropout)."""
    out = {}
    for nd in ir.nodes:
        if not (nd["kind"] == "relu" or (nd["kind"] == "linear" and nd["attrs"]["activation"] == NONE)):
            continue
        t = nd["out"]
        rd = [(r, j) for r in ir.nodes for j, x in enumerate(r["ins"]) if x == t]
        agg = [r for r, j in rd if j == 0 and r["kind"] in AGGREGATING]
        if agg and all((j == 0 and r["kind"] in AGGREGATING + ("linear",)) for r, j in rd):
            out[t] = (nd, agg[0], [r for r, j in rd if r["kind"] == "linear"])
    return out


def dev_rows(a):
    return K.padded(a.shape[0], a.shape[1], fill=torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV))


def bits_dev(bits):
    x = K.bf16_padded(bits.shape[0], bits.shape[1])
    x.copy_(torch.from_numpy(bits.view(np.int16)).to(DEV).view(torch.bfloat16))
    return x


def bf16_bits(y):
    return K.f32_to_bf16(y).view(torch.int16).cpu().numpy().view(np.uint16)


def source(m, ir, t):
    """the fp32 rows a node reads as input t (a rate-0 dropout is a copy)"""
    byid = {nd["out"]: nd for nd in ir.nodes}
    if t in byid and byid[t]["kind"] == "dropout":
        t = byid[t]["ins"][0]
    return m.get_tensor(t)


@pytest.mark.parametrize("name", list(CASES))
def test_bf16_tensors_and_first_aggregation(name):
    host, m, ir, h, d = model(name, 0.0, "bfloat16")
    want = expected_bf16(ir)
    assert len(want) == sum(1 for nd in ir.nodes if nd["kind"] in AGGREGATING)          # one per layer
    for t in (t for t in ir.width if t < INNER):
        assert m.tensor_dtype(t) == ("bfloat16" if t in want else ("int32" if t == h["mask"] else "float32")), t
    m.train_mode(); m.zero_gradients(); m.forward()
    row_end, col = d["graph"]
    n = row_end.shape[0]
    d_re = torch.from_numpy(row_end.astype(np.int64)).to(DEV)
    d_col = torch.from_numpy(col.astype(np.int32)).to(DEV)
    plan = K.SgPlan(0, n - 1, 0, d_re, d_col)
    first = min(want, key=lambda t: want[t][0]["layer"])
    for t, (prod, agg, _) in want.items():
        bits = m.get_tensor(t, raw=True)
        x = dev_rows(source(m, ir, prod["ins"][0]))
        if prod["kind"] == "linear":
            w = torch.from_numpy(m.get_parameter(prod["attrs"]["param"])).to(DEV).contiguous()
            y = K.linear_fwd(x, w)
        else:
            y = K.activation_fwd(x, RELU)
        assert np.array_equal(bits, bf16_bits(y)), "%s: tensor %d is not f32_to_bf16 of its producer's result" % (
            name, t)
        if t != first:
            continue
        xw = K.bf16_to_f32(bits_dev(bits))
        got = m.get_tensor(agg["out"])
        if agg["kind"] == "attention_gather":
            ref, _ = plan.attn_forward(xw, dev_rows(m.get_tensor(agg["ins"][1])), agg["attrs"]["heads"],
                                       agg["attrs"]["slope"])
        elif agg["kind"] == "scatter_gather_weighted":
            ref = plan.weighted_forward(xw, torch.from_numpy(EDGE_W[d["gkind"]]).to(DEV))
        else:
            ref, arg = plan.minmax_forward(xw, agg["attrs"]["aggr"])
            assert np.array_equal(m.get_aggr_index(agg["out"]), arg.cpu().numpy().view(np.uint32)), name + " arg"
        assert np.array_equal(got.view(np.int32), ref.cpu().numpy().view(np.int32)), name + ": first aggregation"
    if name.startswith("gat"):
        # the score Linear reads wh in bf16: its dW is linear_dw_bf16 on the stored bits and its dY
        m.backward()
        for t, (_, _, lins) in want.items():
            for lin in lins:
                dy = dev_rows(m.get_tensor(lin["out"], grad=True))
                p = lin["attrs"]["param"]
                dw = torch.zeros(m.get_parameter(p).shape, device=DEV)
                K.linear_dw_bf16(bits_dev(m.get_tensor(t, raw=True)), dy, dw)
                assert np.array_equal(m.get_parameter(p, "grad").view(np.int32), dw.cpu().numpy().view(np.int32)), \
                    "%s: score Linear dW[%d]" % (name, p)
    plan.close()
    host.close()


def witness(ir, graph, feats, labels, mask, weights, edge_values, relu_masks, aggr_args, rounded, step=1):
    """The recorded graph in torch fp64 with autograd for one training step, with opgraph.witness's op semantics for
    the ops these models use.  relu_masks / aggr_args: {layer: the product's relu output > 0 / get_aggr_index}, taken
    where fp32 and fp64 tie.  rounded: {tensor id: the product's values of a tensor it stores in bf16}; the forward
    takes them (each checked to be a correct rounding of the fp64 value) and passes the gradient straight through.
    Returns (logits, [dW], {edge tensor: dL/dw})."""
    row_end, col = graph
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(True) for w in weights]
    ew = {e: torch.from_numpy(np.asarray(v, dtype=np.float64)).requires_grad_(True) for e, v in edge_values.items()}
    val = {ir.leaves[0]: torch.from_numpy(np.asarray(feats, dtype=np.float64))}
    for nd in ir.nodes:
        k, a, ins, what = nd["kind"], nd["attrs"], nd["ins"], "layer %d (%s)" % (nd["layer"], nd["kind"])
        x = val.get(ins[0])
        if k == "linear":
            y = x @ ws[a["param"]].T
            if a["activation"] == RELU:
                y = _relu_with_mask(y, relu_masks.get(nd["layer"]), what)
        elif k in ("scatter_gather_max", "scatter_gather_min"):
            s = _extreme_sources(row_end, col, x.detach().numpy(), k.endswith("max"), aggr_args.get(nd["layer"]), what)
            y = x.gather(0, torch.from_numpy(s))
        elif k == "scatter_gather_weighted":
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, ew[a["edges"]][:, None] * x[src])
        elif k == "attention_gather":
            y = attend(x, val[ins[1]], dst, src, n, a["heads"], a["slope"])
        elif k == "relu":
            y = _relu_with_mask(x, relu_masks.get(nd["layer"]), what)
        elif k == "add":
            y = x + val[ins[1]]
        elif k == "dropout":
            keep = oracle.dropout_mask(0, n, x.shape[1], a["rate"], a["key"], step)
            scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(a["rate"])))
            y = x * torch.from_numpy(keep.astype(np.float64) * scale)
        elif k == "softmax_cross_entropy":
            loss, logits = train_loss(x, np.asarray(labels), np.asarray(mask)), x
            continue
        else:
            raise AssertionError("op not in these models: " + k)
        if nd["out"] in rounded:
            r, p = torch.from_numpy(np.asarray(rounded[nd["out"]], dtype=np.float64)), y.detach()
            assert ((r - p).abs() <= 2.0 ** -8 * 1.001 * p.abs() + 1e-5 * p.abs().max()).all(), \
                "%s: the product's bf16 value is not a rounding of the fp64 one" % what
            y = y + (r - p)
        val[nd["out"]] = y
    loss.backward()
    return (logits.detach().numpy(), [w.grad.numpy() if w.grad is not None else np.zeros(w.shape) for w in ws],
            {e: t.grad.numpy() if t.grad is not None else np.zeros(t.shape) for e, t in ew.items()})


def close(got, want, rtol, atol_scale, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = np.abs(want).max() if want.size else 0.0
    bound = rtol * np.abs(want) + atol_scale * scale + 1e-30
    if want.ndim == 2 and want.size:      # a dW row that vanishes in fp64 holds only rounding of cancelling terms
        bound[np.abs(want).max(axis=1) <= 1e-12 * scale] = 1e-4 * scale + 1e-30
    r = float((np.abs(got - want) / bound).max()) if want.size else 0.0
    assert r <= 1, "%s: %.2f of the bound" % (what, r)


def adam_w(w, g, t=1):
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
    alpha_t = float(np.float32(LR * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)))
    wd, eps = float(np.float32(WD)), float(np.float32(1e-8))
    w, g = np.asarray(w, np.float64), np.asarray(g, np.float64)
    gt = g + wd * w
    mm, v = (1 - b1) * gt, (1 - b2) * gt * gt
    return w - alpha_t * mm / (np.sqrt(v) + eps)


@pytest.mark.parametrize("name", list(CASES))
def test_bf16_training_step_vs_fp64(name):
    host, m, ir, h, d = model(name, 0.5, "bfloat16")
    want = expected_bf16(ir)
    w0 = [m.get_parameter(p) for p in range(m.num_parameters())]
    m.train_mode(); m.zero_gradients(); m.forward()
    logits = m.get_tensor(h["logits"])
    rounded = {t: m.get_tensor(t) for t in want}
    relu = {nd["layer"]: m.get_tensor(nd["out"]) > 0 for nd in ir.nodes if nd["kind"] == "relu"}
    args = {nd["layer"]: m.get_aggr_index(nd["out"]) for nd in ir.nodes
            if nd["kind"] in ("scatter_gather_max", "scatter_gather_min")}
    m.backward()
    dw = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
    de = {e: m.get_tensor(e, grad=True)[:, 0].copy() for e in ir.edges if ir.edge_grad[e]}
    m.update()
    w1 = [m.get_parameter(p) for p in range(m.num_parameters())]
    host.close()
    wl, wdw, wde = witness(ir, d["graph"], d["feats"], d["labels"], d["mask"], w0,
                           {e: EDGE_W[d["gkind"]] for e in ir.edges}, relu, args, rounded)
    close(logits, wl, 1e-4, 1e-5, name + " logits")
    for p in range(len(w0)):
        close(dw[p], wdw[p], 2e-4, 2e-5, "%s dW[%d]" % (name, p))
        close(w1[p], adam_w(w0[p], dw[p]), 1e-6, 1e-7, "%s W[%d] after Adam" % (name, p))
    for e, g in de.items():
        close(g, wde[e], 2e-4, 2e-5, name + " edge gradient")
    assert de or not name.startswith("gcn_weighted")


@pytest.mark.parametrize("name", list(CASES))
def test_mode_off_is_unchanged(name):
    runs = []
    for off_call in (False, True):
        host, m, ir, h, _ = model(name, 0.5, "float32", off_call=off_call)
        assert all(m.tensor_dtype(t) != "bfloat16" for t in ir.width if t < INNER)
        m.train_mode(); m.zero_gradients(); m.forward()
        lg = m.get_tensor(h["logits"])
        m.backward()
        dw = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        de = [m.get_tensor(e, grad=True) for e in ir.edges if ir.edge_grad[e]]
        m.update()
        runs.append((lg, dw + de, [m.get_parameter(p) for p in range(m.num_parameters())]))
        host.close()
    (a, da, wa), (b, db, wb) = runs
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    for x, y in zip(da + wa, db + wb):
        assert np.array_equal(x.view(np.int32), y.view(np.int32))
