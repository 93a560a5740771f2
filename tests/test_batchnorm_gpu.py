"""Batch normalisation on the GPU: roc_batchnorm_fwd / roc_batchnorm_bwd against the fp64 reference of
tests/test_batchnorm_cpu.py over rows x widths with NaN padding, relu, inference and accumulation, byte-identical on
repeat; then the five builders with norm="batch" over three Adam steps against an fp64 autograd interpreter of the
recorded op graph, fused and unfused, with the running statistics, inference, the other model options and the
refusals."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import oracle
from opgraph import Recorder, _extreme_sources, _relu_with_mask
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model
from test_batchnorm_cpu import BUILDERS, bn_backward, bn_forward
from witness_gat import attend, edge_lists, train_loss

pytestmark = pytest.mark.gpu
U = 2.0 ** -24          # fp32 unit roundoff
K_Y = 3                 # |y - y64| <= K_Y U (|x a| + |b|): a, b rounded to fp32, one fma
K_DX = 4                # |dx - dx64| <= K_DX U (|A g| + |B x| + |C|): A, B, C rounded to fp32, two fmas
K_RED = 4               # |dgamma - ref| <= K_RED U sum |g xhat|, |dbeta - ref| <= K_RED U sum |g|: fp64 sums, one rounding


# ------------------------------------------------------------------------------------------------- the kernel ---
def _inputs(rows, h, seed):
    """x and g in NaN-padded [rows][round_up4(h)] buffers.  Column c % 4: 0 plain normal, 1 mean 1e4 std 1,
    2 constant (var 0), 3 normal with a third of the values +-0; column 0 also holds +-0 when h < 4."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((rows, h), generator=gen, device="cuda")
    col = torch.arange(h, device="cuda") % 4
    x = torch.where(col == 1, x + 1e4, x)
    x = torch.where(col == 2, torch.full_like(x, 3.25), x)
    zeros = (torch.rand((rows, h), generator=gen, device="cuda") < 0.33) & ((col == 3) | (h < 4))
    x = torch.where(zeros, torch.where(torch.rand((rows, h), generator=gen, device="cuda") < 0.5, 0.0, -0.0), x)
    g = torch.randn((rows, h), generator=gen, device="cuda")
    gamma = torch.rand(h, generator=gen, device="cuda") + 0.5
    beta = torch.randn(h, generator=gen, device="cuda")
    rm = torch.randn(h, generator=gen, device="cuda")
    rv = torch.rand(h, generator=gen, device="cuda") + 0.5
    return _nan_padded(x), _nan_padded(g), gamma, beta, rm, rv


def _nan_padded(v):
    rows, h = v.shape
    buf = torch.full((rows, (h + 3) // 4 * 4), float("nan"), device=v.device)
    buf[:, :h] = v
    return buf[:, :h]


def _bits(t):
    """every element of t's storage window, padding included, as int32 bits"""
    rows, h = t.shape
    return torch.as_strided(t, (rows, t.stride(0)), (t.stride(0), 1)).contiguous().view(torch.int32)


def _pad_untouched(t):
    rows, h = t.shape
    full = torch.as_strided(t, (rows, t.stride(0)), (t.stride(0), 1))
    return bool(torch.isnan(full[:, h:]).all()) if full.shape[1] > h else True


def _ratio(got, want, bound):
    return float(((got.double() - want).abs() / (bound + 1e-300)).max())


def _check_case(rows, h, seed):
    what = "rows=%d H=%d" % (rows, h)
    x, g, gamma, beta, rm0, rv0 = _inputs(rows, h, seed)
    x64 = x.double()
    ref = bn_forward(x, gamma, beta, rm0, rv0, training=True)
    for relu in (False, True):
        rm, rv = rm0.clone(), rv0.clone()
        y, st = K.batchnorm_fwd(x, gamma, beta, rm, rv, relu=relu, out=_nan_padded(torch.zeros_like(x)))
        assert _pad_untouched(y), what
        bound = K_Y * U * ((x64 * ref["a"]).abs() + ref["b"].abs())
        want = torch.relu(ref["y"]) if relu else ref["y"]
        assert _ratio(y, want, bound) <= 1.0, (what, relu)
        assert bool((st.mean - ref["mean"]).abs().le(1e-12 * (1 + ref["mean"].abs())).all()), what
        assert _ratio(rm, ref["run_mean"], 2 * U * ref["run_mean"].abs() + 1e-30) <= 1.0, what
        assert _ratio(rv, ref["run_var"], 2 * U * ref["run_var"].abs() + 1e-30) <= 1.0, what
        # repeat: the same bits everywhere
        rm2, rv2 = rm0.clone(), rv0.clone()
        y2, st2 = K.batchnorm_fwd(x, gamma, beta, rm2, rv2, relu=relu, out=_nan_padded(torch.zeros_like(x)))
        assert torch.equal(_bits(y), _bits(y2)) and torch.equal(rm.view(torch.int32), rm2.view(torch.int32)), what
        assert torch.equal(rv.view(torch.int32), rv2.view(torch.int32)), what
        assert torch.equal(st.a.view(torch.int32), st2.a.view(torch.int32)), what
        assert torch.equal(st.b.view(torch.int32), st2.b.view(torch.int32)), what
        # backward: the mask is the forward's own test, fma(x, a, b) > 0 on the saved fp32 a, b
        gm = g.double()
        if relu:
            gm = torch.where(x64 * st.a.double() + st.b.double() > 0, gm, 0.0)
        bwd = bn_backward(x, gm, gamma, ref["mean"], ref["var"])
        dbound = K_DX * U * (bwd["Ag"].abs() + bwd["Bx"].abs() + bwd["C"].abs())
        for acc in (False, True):
            base = torch.randn_like(x) if acc else torch.zeros_like(x)
            dx = _nan_padded(base.clone())
            dx, dgam, dbet = K.batchnorm_bwd(x, g, gamma, st, relu=relu, dx=dx, accumulate=acc)
            assert _pad_untouched(dx), what
            want = bwd["dx"] + (base.double() if acc else 0)
            bnd = dbound + (2 * U * (base.double().abs() + bwd["dx"].abs()) if acc else 0)
            assert _ratio(dx, want, bnd) <= 1.0, (what, relu, acc)
            assert _ratio(dgam, bwd["dgamma"], K_RED * U * bwd["gxhat"].abs().sum(0)) <= 1.0, (what, relu)
            assert _ratio(dbet, bwd["dbeta"], K_RED * U * gm.abs().sum(0)) <= 1.0, (what, relu)
            dx2, dgam2, dbet2 = K.batchnorm_bwd(x, g, gamma, st2, relu=relu, dx=_nan_padded(base.clone()),
                                                accumulate=acc)
            assert torch.equal(_bits(dx), _bits(dx2)), what
            assert torch.equal(dgam.view(torch.int32), dgam2.view(torch.int32)), what
            assert torch.equal(dbet.view(torch.int32), dbet2.view(torch.int32)), what
        _, dg3, db3 = K.batchnorm_bwd(x, g, gamma, st, relu=relu, need_dx=False)
        assert torch.equal(dg3.view(torch.int32), dgam.view(torch.int32)), what
        assert torch.equal(db3.view(torch.int32), dbet.view(torch.int32)), what
    # inference: the running statistics' affine map, nothing updated
    eref = bn_forward(x, gamma, beta, rm0, rv0, training=False)
    for relu in (False, True):
        rm, rv = rm0.clone(), rv0.clone()
        y, st = K.batchnorm_fwd(x, gamma, beta, rm, rv, training=False, relu=relu, out=_nan_padded(torch.zeros_like(x)))
        bound = K_Y * U * ((x64 * eref["a"]).abs() + eref["b"].abs())
        assert _ratio(y, torch.relu(eref["y"]) if relu else eref["y"], bound) <= 1.0, (what, "infer", relu)
        assert torch.equal(rm, rm0) and torch.equal(rv, rv0) and _pad_untouched(y), what
        assert not st.a.any() and not st.mean.any(), what


@pytest.mark.parametrize("h", [1, 3, 4, 41, 64, 128, 256])
@pytest.mark.parametrize("rows", [2, 3, 1000, 65537])
def test_kernel_matches_fp64(rows, h):
    _check_case(rows, h, seed=rows * 7 + h)


def test_kernel_at_production_rows():
    _check_case(4194304, 64, seed=11)


def test_kernel_refuses_bad_arguments():
    rows, h = 8, 6
    x = K.padded(rows, h)
    gamma, beta = torch.ones(h, device="cuda"), torch.zeros(h, device="cuda")
    rm, rv = torch.zeros(h, device="cuda"), torch.ones(h, device="cuda")
    st = K.BatchNormState(rows, h)
    p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    ok = dict(rows=rows, x=x, ldX=8, y=K.padded(rows, h), ldY=8, eps=1e-5, mom=0.1, rm=rm, rv=rv, train=1,
              ws=st.ws_bytes)

    def fwd(**kw):
        a = dict(ok, **kw)
        rc = _lib.lib.roc_batchnorm_fwd(a["rows"], h, p(a["x"]), a["ldX"], p(gamma), p(beta), a["eps"], a["mom"],
                                        p(a["rm"]), p(a["rv"]), a["train"], 0, p(a["y"]), a["ldY"], p(st.a), p(st.b),
                                        p(st.mean), p(st.invstd), p(st.ws), a["ws"], None)
        torch.cuda.synchronize()
        return rc

    assert fwd() == _lib.ROC_OK
    assert fwd(rm=None, rv=None) == _lib.ROC_OK          # training without running statistics
    for bad in (dict(rows=1), dict(rows=-1), dict(ldX=6), dict(ldX=5), dict(ldY=10), dict(x=None), dict(y=None),
                dict(eps=-1.0), dict(mom=1.5), dict(rm=None), dict(train=0, rm=None, rv=None), dict(ws=st.ws_bytes - 1)):
        assert fwd(**bad) == _lib.ROC_ERR_INVALID, bad
    assert fwd(train=0, rows=1) == _lib.ROC_OK           # inference takes any row count


# ------------------------------------------------------------------------------------------------- the models ---
def bn_witness(ir, graph, feats, labels, mask, weights, run_stats, training=True, edge_values=None, step=1,
               relu_masks=None, aggr_args=None, loss_fn=train_loss):
    """The recorded graph in torch fp64 with autograd for one step (opgraph.witness's semantics, plus batch_norm):
    training uses the batch statistics and the dropout masks of `step`; training=False is the infer-mode model
    (dropout a copy, batch_norm on run_stats {bn output: (mean, var)}).  Returns logits, dW and, per batch_norm
    output, its batch (mean, var)."""
    row_end, col = np.asarray(graph[0]), np.asarray(graph[1])
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dinv = torch.from_numpy(1.0 / np.sqrt(deg.astype(np.float64))).unsqueeze(1)
    relu_masks, aggr_args = relu_masks or {}, aggr_args or {}
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(True) for w in weights]
    ew = {e: torch.from_numpy(np.asarray(v, dtype=np.float64)) for e, v in (edge_values or {}).items()}
    val = {ir.leaves[0]: torch.from_numpy(np.asarray(feats, dtype=np.float64))}
    stats, loss = {}, None
    for node in ir.nodes:
        k, a, ins, what = node["kind"], node["attrs"], node["ins"], "layer %d (%s)" % (node["layer"], node["kind"])
        x = val.get(ins[0])
        if k == "linear":
            y = x @ ws[a["param"]].T
            if a["activation"] == _lib.AC_MODE_RELU:
                y = _relu_with_mask(y, relu_masks.get(node["layer"]), what)
        elif k == "batch_norm":
            gam, bet = ws[a["gamma"]][0], ws[a["beta"]][0]
            if training:
                mean = x.detach().mean(0)
                stats[node["out"]] = (mean, ((x.detach() - mean) ** 2).mean(0))
                y = torch.nn.functional.batch_norm(x, None, None, gam, bet, training=True, eps=a["eps"])
            else:
                rm, rv = (torch.from_numpy(np.asarray(s, dtype=np.float64)) for s in run_stats[node["out"]])
                y = torch.nn.functional.batch_norm(x, rm, rv, gam, bet, training=False, eps=a["eps"])
        elif k == "indegree_norm":
            y = x * dinv
        elif k == "scatter_gather":
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, x[src])
        elif k in ("scatter_gather_max", "scatter_gather_min"):
            s = _extreme_sources(row_end, col, x.detach().numpy(), k.endswith("max"), aggr_args.get(node["layer"]),
                                 what)
            y = x.gather(0, torch.from_numpy(s))
        elif k == "scatter_gather_weighted":
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, ew[a["edges"]][:, None] * x[src])
        elif k == "attention_gather":
            y = attend(x, val[ins[1]], dst, src, n, a["heads"], a["slope"])
        elif k == "relu":
            y = _relu_with_mask(x, relu_masks.get(node["layer"]), what)
        elif k == "add":
            y = x + val[ins[1]]
        elif k == "dropout":
            if a["rate"] > 0 and training:
                keep = oracle.dropout_mask(0, n, x.shape[1], a["rate"], a["key"], step)
                scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(a["rate"])))
                y = x * torch.from_numpy(keep.astype(np.float64) * scale)
            else:
                y = x
        elif k in ("softmax_cross_entropy", "sigmoid_cross_entropy"):
            logits = x
            if training:
                loss = loss_fn(x, np.asarray(labels), np.asarray(mask))
            continue
        else:
            raise AssertionError("unknown op " + k)
        val[node["out"]] = y
    if loss is not None:
        loss.backward()
    return dict(logits=logits.detach().numpy(), stats=stats,
                dW=[w.grad.numpy() if w.grad is not None else np.zeros(w.shape) for w in ws])


def _bce_train_loss(x, labels, mask):
    train = torch.from_numpy(np.asarray(mask) == _lib.MASK_TRAIN)
    y = torch.from_numpy(np.asarray(labels, dtype=np.float64))
    return torch.nn.functional.binary_cross_entropy_with_logits(x[train], y[train], reduction="sum")


def sym_graph():
    re_, col = datasets.rmat_graph(9, 2500, seed=3)
    return re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


def directed_graph():
    re_, col = datasets.rmat_graph(9, 2500, seed=4, directed=True)
    return re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


def train(name, graph, fuse, steps=3, norm="batch", loss="softmax", **kw):
    row_end, col = graph
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    ir = Recorder(m)
    ir.edge_w = np.random.RandomState(2).uniform(0.05, 0.6, size=col.shape[0]).astype(np.float32)
    if name == "gcn_weighted":
        kw = dict(kw, edge_weights=ir.edge_w)
    h = BUILDERS[name](ir, norm=norm, loss=loss, **kw)
    if loss == "sigmoid":
        feats, labels, mask = (t.numpy() for t in datasets.multilabel_node_data(n, 24, 12, seed=5))
        m.set_multilabels(h["label"], labels)
    else:
        feats, labels, mask = (t.numpy() for t in datasets.node_data(n, 24, 12, seed=5))
        m.set_labels(h["label"], labels)
    m.set_tensor(h["input"], feats)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    relu_of = {nd["layer"]: nd["out"] for nd in ir.nodes if nd["kind"] == "relu"}
    minmax = {nd["layer"]: nd["out"] for nd in ir.nodes if nd["kind"] in ("scatter_gather_max", "scatter_gather_min")}
    out = dict(ir=ir, h=h, feats=feats, labels=labels, mask=mask, info=m.op_info(), steps=[], graph=graph, loss=loss)
    for _ in range(steps):
        st = dict(w0=[m.get_parameter(p) for p in range(m.num_parameters())])
        m.train_mode(); m.zero_gradients(); m.forward()
        st["logits"] = m.get_tensor(h["logits"])
        st["relu"] = {l: m.get_tensor(t) > 0 for l, t in relu_of.items()}
        st["args"] = {l: m.get_aggr_index(t) for l, t in minmax.items()}
        m.backward()
        st["dw"] = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
        st["w1"] = [m.get_parameter(p) for p in range(m.num_parameters())]
        out["steps"].append(st)
    out["run_stats"] = {t: m.batch_norm_stats(t) for t in h["bns"]}
    out["w_final"] = [m.get_parameter(p) for p in range(m.num_parameters())]
    m.infer_mode(); m.forward()
    out["infer_logits"] = m.get_tensor(h["logits"])
    out["dtypes"] = {t: m.tensor_dtype(t) for t in ir.width}
    host.close()
    return out


def close(name, got, want, rtol=2e-4, atol_scale=2e-5):
    """test_opgraph_gpu.py's bar"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    bound = rtol * np.abs(want) + atol_scale * np.abs(want).max() + 1e-30
    r = float((np.abs(got - want) / bound).max())
    assert r <= 1.0, (name, r)


def check_witness(run, feats=None):
    """each step's logits and gradients against the fp64 interpreter; the running statistics against the recurrence
    over the interpreter's batch statistics; the infer-mode logits against the eval-mode model"""
    ir = run["ir"]
    edges = {e: ir.edge_w for e in ir.edges}
    feats = run["feats"] if feats is None else feats
    loss_fn = _bce_train_loss if run["loss"] == "sigmoid" else train_loss
    n = feats.shape[0]
    rec = {t: (np.zeros(ir.width[t]), np.ones(ir.width[t])) for t in run["h"]["bns"]}
    for k, st in enumerate(run["steps"]):
        wt = bn_witness(ir, run["graph"], feats, run["labels"], run["mask"], st["w0"], None, edge_values=edges,
                        step=k + 1, relu_masks=st["relu"], aggr_args=st["args"], loss_fn=loss_fn)
        close("step %d logits" % k, st["logits"], wt["logits"])
        for p, (a, b) in enumerate(zip(st["dw"], wt["dW"])):
            close("step %d dW%d" % (k, p), a, b)
        for t, (mean, var) in wt["stats"].items():
            rm, rv = rec[t]
            rec[t] = (0.9 * rm + 0.1 * mean.numpy(), 0.9 * rv + 0.1 * var.numpy() * n / (n - 1))
    for t, (rm, rv) in rec.items():
        close("running mean", run["run_stats"][t][0], rm)
        close("running var", run["run_stats"][t][1], rv)
    ev = bn_witness(ir, run["graph"], feats, run["labels"], run["mask"], run["w_final"], run["run_stats"],
                    training=False, edge_values=edges)
    close("infer logits", run["infer_logits"], ev["logits"])


def check_identical(a, b):
    for sa, sb in zip(a["steps"], b["steps"]):
        assert np.array_equal(sa["logits"].view(np.int32), sb["logits"].view(np.int32))
        for k in ("dw", "w1"):
            for x, y in zip(sa[k], sb[k]):
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), k
    for t in a["run_stats"]:
        for x, y in zip(a["run_stats"][t], b["run_stats"][t]):
            assert np.array_equal(x.view(np.int32), y.view(np.int32))
    assert np.array_equal(a["infer_logits"].view(np.int32), b["infer_logits"].view(np.int32))


def check_fusion(fused, unfused):
    """each relu after a batch_norm is fused into it (op_info), and left apart by set_fusion(false)"""
    ir = fused["ir"]
    for nd in ir.nodes:
        if nd["kind"] != "batch_norm":
            continue
        relu = next(r for r in ir.nodes if r["ins"] == [nd["out"]])
        assert fused["info"][relu["layer"]]["fusedInto"] == nd["layer"]
        assert fused["info"][nd["layer"]]["fwdOut"] == relu["out"]
        assert unfused["info"][relu["layer"]]["fusedInto"] == -1 and unfused["info"][nd["layer"]]["fwdOut"] == -1


@pytest.mark.parametrize("name", list(BUILDERS))
def test_builder_with_batch_norm_matches_the_witness(name):
    g = sym_graph()
    fused, unfused = train(name, g, True), train(name, g, False)
    check_witness(fused)
    check_identical(fused, unfused)
    check_fusion(fused, unfused)
    assert [i["kind"] for i in fused["info"]] == [nd["kind"] for nd in fused["ir"].nodes]
    # BN draws no random numbers: the Linears start where they start without it
    plain = train(name, g, True, steps=1, norm=None)
    lin = [nd["attrs"]["param"] for nd in fused["ir"].nodes if nd["kind"] == "linear"]
    assert len(lin) == len(plain["steps"][0]["w0"])
    for p, q in zip(lin, range(len(lin))):
        assert np.array_equal(fused["steps"][0]["w0"][p], plain["steps"][0]["w0"][q])
    for nd in fused["ir"].nodes:
        if nd["kind"] == "batch_norm":     # gamma 1 and beta 0 at the start, shape (1, H)
            w = fused["steps"][0]["w0"]
            assert np.all(w[nd["attrs"]["gamma"]] == 1) and np.all(w[nd["attrs"]["beta"]] == 0)
            assert w[nd["attrs"]["gamma"]].shape == (1, fused["ir"].width[nd["out"]])


def test_batch_norm_with_exact_backward_on_a_directed_graph():
    g = directed_graph()
    fused, unfused = train("gcn4", g, True, exact_backward=True), train("gcn4", g, False, exact_backward=True)
    check_witness(fused)
    check_identical(fused, unfused)


def test_batch_norm_with_bf16_features():
    run = train("sage_mean", sym_graph(), True, features="bfloat16")
    assert run["dtypes"][run["h"]["input"]] == "bfloat16"
    check_witness(run, feats=torch.from_numpy(run["feats"]).bfloat16().float().numpy())


def test_batch_norm_with_sigmoid_loss():
    check_witness(train("gcn", sym_graph(), True, loss="sigmoid"))


@pytest.mark.parametrize("name", ["gcn", "sage_pool", "gat", "gcn_weighted"])
def test_batch_norm_with_bf16_aggregation(name):
    """The aggregation inputs are rounded, so no fp32 witness applies: the BN tensors and the relus fused into them
    stay fp32, some tensor is bf16, fused equals unfused, and the run repeats bit for bit."""
    a = train(name, sym_graph(), True, aggregation="bfloat16")
    b = train(name, sym_graph(), True, aggregation="bfloat16")
    assert "bfloat16" in a["dtypes"].values()
    for nd in a["ir"].nodes:
        if nd["kind"] == "batch_norm":
            relu = next(r for r in a["ir"].nodes if r["ins"] == [nd["out"]])
            assert a["dtypes"][nd["ins"][0]] == a["dtypes"][nd["out"]] == a["dtypes"][relu["out"]] == "float32"
    for st in a["steps"]:
        assert all(np.isfinite(d).all() for d in st["dw"])
    check_identical(a, b)


def test_bf16_aggregation_never_picks_a_batch_norm_tensor():
    """A relu fused into a BN is not a bf16 candidate even when a max aggregation reads it (its unfused twin is); a
    Linear(NONE) output that a BN also reads is disqualified (without the BN reader it is bf16)."""
    row_end, col = sym_graph()

    def build(fuse, bn_reads_lin):
        host = Host(0, 0, 1)
        host.graph_from_arrays(row_end, col)
        m = Model(host, seed=1)
        m.set_fusion(fuse)
        x = m.create_node_tensor(8)
        lab = m.create_node_tensor(4)
        mk = m.create_node_tensor(1, is_int=True)
        lin = m.linear(x, 8)
        r = m.relu(m.batch_norm(m.linear(x, 8)))
        t = m.add(m.scatter_gather(r, _lib.AGGR_MAX), m.scatter_gather(lin, _lib.AGGR_MAX))
        if bn_reads_lin:
            t = m.add(t, m.batch_norm(lin))
        m.softmax_cross_entropy(m.linear(t, 4), lab, mk)
        m.adam()
        m.set_bf16_aggregation(True)
        m.init()
        d = (m.tensor_dtype(r), m.tensor_dtype(lin))
        host.close()
        return d

    assert build(True, False) == ("float32", "bfloat16")
    assert build(False, False) == ("bfloat16", "bfloat16")
    assert build(True, True) == ("float32", "float32")


def test_batch_norm_stats_round_trip():
    row_end, col = sym_graph()
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    (t,) = BUILDERS["gcn"](m, norm="batch")["bns"]
    mean0, var0 = m.batch_norm_stats(t)
    m.set_batch_norm_stats(t, np.arange(16, dtype=np.float32), np.full(16, 2.5, dtype=np.float32))
    mean1, var1 = m.batch_norm_stats(t)
    host.close()
    assert np.all(mean0 == 0) and np.all(var0 == 1)
    assert np.array_equal(mean1, np.arange(16)) and np.all(var1 == 2.5)


REFUSALS = {
    "bf16_leaf": ("x = m.create_node_tensor(8, dtype='bfloat16'); y = m.create_node_tensor(4);"
                  " mk = m.create_node_tensor(1, True); m.softmax_cross_entropy(m.linear(m.batch_norm(x), 4), y, mk);"
                  " m.adam(); m.init()", 100, "batch_norm cannot read a bf16 tensor"),
    "one_row": ("x = m.create_node_tensor(8); y = m.create_node_tensor(4); mk = m.create_node_tensor(1, True);"
                " m.softmax_cross_entropy(m.linear(m.batch_norm(x), 4), y, mk); m.adam(); m.init()", 1,
                "batch_norm: the partition has fewer than 2 rows"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_refusals(name):
    body, n, message = REFUSALS[name]
    prog = "\n".join([
        "import numpy as np",
        "from roc_b200.model import Host, Model",
        "host = Host(0, 0, 1)",
        "host.graph_from_arrays(np.arange(1, %d, dtype=np.uint64), np.arange(%d, dtype=np.uint32))" % (n + 1, n),
        "m = Model(host, seed=1)",
        body,
        "host.synchronize()",
        "print('NO REFUSAL')",
    ])
    p = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ))
    assert p.returncode != 0, p.stdout + p.stderr
    assert message in p.stderr, p.stderr[-2000:]
    assert "NO REFUSAL" not in p.stdout
