"""GPU suite: models with bf16 aggregation inputs (Model.set_bf16_aggregation, aggregation="bfloat16" on build_gcn and
build_sage_mean): a 2-layer GCN, a 4-layer GCN with its residual branch and a 2-layer GraphSAGE-mean.

* tensor_dtype marks exactly the tensors a Linear without activation writes (its output, or the indegree_norm fused
  into it) that one sum scatter_gather alone reads, as the recorded op graph says; every other tensor stays fp32.
* Each bf16 tensor holds f32_to_bf16 of what the Linear computes in fp32 from the model's own input rows (the first
  one also of the same tensor in an fp32 twin model), and the first aggregation's output is the fp32 ScatterGather
  run on the widened bits, bit for bit.
* One training step at dropout 0.5 against an fp64 torch witness of the recorded graph that rounds those tensors to
  bf16 in the forward pass (taking the product's rounding, which must be a correct rounding of the fp64 value) and
  passes gradients straight through: logits, every dW, and every weight after Adam, within the bounds the op-graph
  witness uses.
* With the mode off, a model that calls set_bf16_aggregation(False) is byte-identical to one that never calls it."""
import math

import numpy as np
import pytest
import torch

from opgraph import INNER, Recorder
from oracle import oracle
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_gcn, build_sage_mean
from witness_gat import edge_lists, train_loss

pytestmark = pytest.mark.gpu
DEV = "cuda"
N, PAIRS = 900, 5000
LR, WD = 0.01, 0.05
BUILDERS = {
    "gcn2": lambda m, d, a: build_gcn(m, [40, 24, 7], d, aggregation=a),
    "gcn4_residual": lambda m, d, a: build_gcn(m, [40, 24, 16, 12, 7], d, aggregation=a),
    "sage_mean": lambda m, d, a: build_sage_mean(m, [40, 24, 7], d, aggregation=a),
}
ROW_END, COL = (t.numpy() for t in datasets.uniform_graph(N, PAIRS, seed=3))
ROW_END, COL = ROW_END.astype(np.uint64), COL.astype(np.uint32)
FEATS, LABELS, MASK = (t.numpy() for t in datasets.node_data(N, 40, 7, seed=2))


def model(name, dropout, aggregation, off_call=False, weights=None):
    host = Host(0, 0, 1)
    host.graph_from_arrays(ROW_END, COL)
    m = Model(host, seed=1)
    if off_call:
        m.set_bf16_aggregation(False)
    ir = Recorder(m)
    h = BUILDERS[name](ir, dropout, aggregation)
    if weights is not None:
        for p, w in enumerate(weights):
            m.set_parameter(p, w)
    m.set_tensor(h["input"], FEATS)
    m.set_labels(h["label"], LABELS)
    m.set_tensor(h["mask"], MASK.astype(np.int32))
    return host, m, ir, h


def expected_bf16(ir):
    """From the recorded graph: each Linear(NONE)'s output, or its fused norm's, that one sum scatter_gather reads."""
    readers = {}
    for nd in ir.nodes:
        for t in nd["ins"]:
            readers.setdefault(t, []).append(nd)
    out = {}
    for nd in ir.nodes:
        if nd["kind"] != "linear" or nd["attrs"]["activation"] != _lib.AC_MODE_NONE:
            continue
        t, rd = nd["out"], readers.get(nd["out"], [])
        if len(rd) == 1 and rd[0]["kind"] == "indegree_norm":        # the fused linear -> indegree_norm
            t, rd, norm = rd[0]["out"], readers.get(rd[0]["out"], []), True
        else:
            norm = False
        if len(rd) == 1 and rd[0]["kind"] == "scatter_gather" and rd[0]["attrs"]["aggr"] == _lib.AGGR_SUM:
            out[t] = (nd, norm, rd[0])
    return out


def dev_rows(a):
    return K.padded(a.shape[0], a.shape[1], fill=torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV))


def bits_dev(bits):
    h = bits.shape[1]
    x = K.bf16_padded(bits.shape[0], h)
    x.copy_(torch.from_numpy(bits.view(np.int16)).to(DEV).view(torch.bfloat16))
    return x


@pytest.mark.parametrize("name", list(BUILDERS))
def test_bf16_tensors_and_first_aggregation(name):
    host, m, ir, h = model(name, 0.0, "bfloat16")
    want = expected_bf16(ir)
    assert len(want) == sum(1 for nd in ir.nodes if nd["kind"] == "scatter_gather")   # one per layer here
    ids = {t for t in ir.width if t < INNER}
    for t in ids:
        assert m.tensor_dtype(t) == ("bfloat16" if t in want else ("int32" if t == h["mask"] else "float32")), t
    m.train_mode(); m.zero_gradients(); m.forward()
    d_re = torch.from_numpy(ROW_END.astype(np.int64)).to(DEV)
    d_col = torch.from_numpy(COL.astype(np.int32)).to(DEV)
    byid = {nd["out"]: nd for nd in ir.nodes}
    first = min(want, key=lambda t: want[t][0]["layer"])
    for t, (lin, norm, sg) in want.items():
        bits = m.get_tensor(t, raw=True)
        assert np.array_equal(m.get_tensor(t), K.bf16_to_f32(bits_dev(bits)).cpu().numpy())   # widened exactly
        x = lin["ins"][0]
        if x in byid and byid[x]["kind"] == "dropout":        # rate 0: the dropout is a copy
            x = byid[x]["ins"][0]
        w = torch.from_numpy(m.get_parameter(lin["attrs"]["param"])).to(DEV).contiguous()
        y = K.linear_fwd(dev_rows(m.get_tensor(x)), w, norm_row_end=d_re if norm else None)
        r = K.f32_to_bf16(y).view(torch.int16).cpu().numpy().view(np.uint16)
        assert np.array_equal(bits, r), "%s: tensor %d is not f32_to_bf16 of its Linear's fp32 result" % (name, t)
        if t == first:
            info = m.op_info()[sg["layer"]]
            out = info["fwdOut"] if info["fwdOut"] >= 0 else sg["out"]
            plan = K.SgPlan(0, N - 1, 0, d_re, d_col)
            ref = plan.forward(K.bf16_to_f32(bits_dev(bits)), epilogue=info["epilogue"]).cpu().numpy()
            got = m.get_tensor(out)
            assert np.array_equal(got.view(np.int32), ref.view(np.int32)), "%s: first aggregation" % name
            plan.close()
    w0 = [m.get_parameter(p) for p in range(m.num_parameters())]
    host.close()
    # the first bf16 tensor against an fp32 twin with the same weights and inputs
    host, m2, _, _ = model(name, 0.0, "float32", weights=w0)
    m2.train_mode(); m2.zero_gradients(); m2.forward()
    twin = K.f32_to_bf16(dev_rows(m2.get_tensor(first))).view(torch.int16).cpu().numpy().view(np.uint16)
    host.close()
    host, m, _, _ = model(name, 0.0, "bfloat16", weights=w0)
    m.train_mode(); m.zero_gradients(); m.forward()
    assert np.array_equal(m.get_tensor(first, raw=True), twin), "%s: the fp32 twin rounds differently" % name
    host.close()


def witness(ir, w0, bf16_vals, relu_masks, step=1):
    """fp64 forward + autograd of the recorded graph; the bf16 tensors take the product's rounding (checked to be a
    correct rounding of the fp64 value), with a straight-through gradient."""
    n = ROW_END.shape[0]
    dst, src = edge_lists(ROW_END, COL)
    deg = np.diff(np.concatenate([[0], ROW_END.astype(np.int64)]))
    dinv = torch.from_numpy(1.0 / np.sqrt(deg.astype(np.float64))).unsqueeze(1)
    ws = [torch.from_numpy(w.astype(np.float64)).requires_grad_(True) for w in w0]
    val = {ir.leaves[0]: torch.from_numpy(FEATS.astype(np.float64))}
    for nd in ir.nodes:
        k, a = nd["kind"], nd["attrs"]
        x = val.get(nd["ins"][0])
        if k == "linear":
            y = x @ ws[a["param"]].T
        elif k == "indegree_norm":
            y = x * dinv
        elif k == "scatter_gather":
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, x[src])
        elif k == "relu":
            pm = torch.from_numpy(relu_masks[nd["out"]])
            p = x.detach()
            off = (p > 0) != pm
            assert not off.any() or p[off].abs().max() <= 1e-4 * p.abs().max(), "relu masks differ away from zero"
            y = torch.where(pm, x, 0.0)
        elif k == "add":
            y = x + val[nd["ins"][1]]
        elif k == "dropout":
            keep = oracle.dropout_mask(0, n, x.shape[1], a["rate"], a["key"], step)
            y = x * torch.from_numpy(keep.astype(np.float64) * float(np.float32(1) / (np.float32(1) - np.float32(a["rate"]))))
        elif k == "softmax_cross_entropy":
            loss, logits = train_loss(x, LABELS, MASK), x
            continue
        else:
            raise AssertionError(k)
        if nd["out"] in bf16_vals:
            r = torch.from_numpy(bf16_vals[nd["out"]].astype(np.float64))
            p = y.detach()
            assert ((r - p).abs() <= 2.0 ** -8 * 1.001 * p.abs() + 1e-5 * p.abs().max()).all(), \
                "tensor %d: the product's bf16 value is not a rounding of the fp64 one" % nd["out"]
            y = y + (r - p)
        val[nd["out"]] = y
    loss.backward()
    return logits.detach().numpy(), [w.grad.numpy() for w in ws]


def close(got, want, rtol, atol_scale, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    bound = rtol * np.abs(want) + atol_scale * np.abs(want).max() + 1e-30
    r = float((np.abs(got - want) / bound).max())
    assert r <= 1, "%s: %.2f of the bound" % (what, r)


def adam_w(w, g, t=1):
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
    alpha_t = float(np.float32(LR * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)))
    wd, eps = float(np.float32(WD)), float(np.float32(1e-8))
    w, g = np.asarray(w, np.float64), np.asarray(g, np.float64)
    gt = g + wd * w
    m, v = (1 - b1) * gt, (1 - b2) * gt * gt
    return w - alpha_t * m / (np.sqrt(v) + eps)


@pytest.mark.parametrize("name", list(BUILDERS))
def test_bf16_training_step_vs_fp64(name):
    host, m, ir, h = model(name, 0.5, "bfloat16")
    want = expected_bf16(ir)
    w0 = [m.get_parameter(p) for p in range(m.num_parameters())]
    m.train_mode(); m.zero_gradients(); m.forward()
    logits = m.get_tensor(h["logits"])
    vals = {t: m.get_tensor(t) for t in want}
    relu = {nd["out"]: m.get_tensor(nd["out"]) > 0 for nd in ir.nodes if nd["kind"] == "relu"}
    m.backward()
    dw = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
    m.update()
    w1 = [m.get_parameter(p) for p in range(m.num_parameters())]
    host.close()
    wl, wdw = witness(ir, w0, vals, relu)
    close(logits, wl, 1e-4, 1e-5, name + " logits")
    for p in range(len(w0)):
        close(dw[p], wdw[p], 2e-4, 2e-5, "%s dW[%d]" % (name, p))
        close(w1[p], adam_w(w0[p], dw[p]), 1e-6, 1e-7, "%s W[%d] after Adam" % (name, p))


@pytest.mark.parametrize("name", list(BUILDERS))
def test_mode_off_is_unchanged(name):
    runs = []
    for off_call in (False, True):
        host, m, ir, h = model(name, 0.5, "float32", off_call=off_call)
        assert all(m.tensor_dtype(t) != "bfloat16" for t in ir.width if t < INNER)
        m.train_mode(); m.zero_gradients(); m.forward()
        lg = m.get_tensor(h["logits"])
        m.backward()
        dw = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
        runs.append((lg, dw, [m.get_parameter(p) for p in range(m.num_parameters())]))
        host.close()
    (a, da, wa), (b, db, wb) = runs
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    for x, y in zip(da + wa, db + wb):
        assert np.array_equal(x.view(np.int32), y.view(np.int32))
