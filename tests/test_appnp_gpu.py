"""APPNP (K = 10) and GCNII (depth 8) on the GPU: three Adam steps against the torch fp64 autograd interpreter of
appnp_witness.py at test_batchnorm_gpu.py's bars, fused and unfused (set_fusion(False)) byte-identical, the teleport
fused into every hop (op_info), and composition with the exact backward on a directed multigraph, bf16 features and
the sigmoid loss.  bf16 aggregation picks no tensor in either model."""
import numpy as np
import pytest

from appnp_witness import bce_train_loss, witness
from opgraph import Recorder
from roc_b200 import _lib, bf16, datasets
from roc_b200.model import Host, Model, build_appnp, build_gcnii
from test_batchnorm_gpu import close, directed_graph, sym_graph
from witness_gat import train_loss

pytestmark = pytest.mark.gpu
NORM, NORM_OUT = _lib.SG_EPI_NORM, _lib.SG_EPI_NORM_OUT
BUILDERS = {
    "appnp": lambda m, **kw: build_appnp(m, [24, 16, 12], 0.5, K=10, alpha=0.1, **kw),
    "gcnii": lambda m, **kw: build_gcnii(m, [24, 16, 12], 0.5, 8, alpha=0.1, theta=0.5, **kw),
}


def gcn_residual(m, loss="softmax"):
    """A GCN layer with an initial residual, z = scaled_add(norm(SG(norm(linear(x0)))), x0): with bf16 aggregation the
    fused linear -> norm output the scatter_gather reads is stored in bf16."""
    x = m.create_node_tensor(24)
    label, mask = m.create_node_tensor(12), m.create_node_tensor(1, is_int=True)
    x0 = m.relu(m.linear(x, 16, _lib.AC_MODE_NONE))
    t = m.indegree_norm(m.scatter_gather(m.indegree_norm(m.linear(x0, 16, _lib.AC_MODE_NONE))))
    z = m.scaled_add(t, x0, 0.875, 0.125)
    logits = m.linear(z, 12, _lib.AC_MODE_NONE)
    m.softmax_cross_entropy(logits, label, mask)
    m.adam(0.01, 0.05)
    m.init()
    return {"input": x, "label": label, "mask": mask, "logits": logits}


MODELS = dict(BUILDERS, gcn_residual=gcn_residual)


def train(name, graph, fuse, steps=3, loss="softmax", bf16_aggregation=False, **kw):
    row_end, col = graph
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    if bf16_aggregation:
        m.set_bf16_aggregation(True)
    ir = Recorder(m)
    h = MODELS[name](ir, loss=loss, **kw)
    if loss == "sigmoid":
        feats, labels, mask = (t.numpy() for t in datasets.multilabel_node_data(n, 24, 12, seed=5))
        m.set_multilabels(h["label"], labels)
    else:
        feats, labels, mask = (t.numpy() for t in datasets.node_data(n, 24, 12, seed=5))
        m.set_labels(h["label"], labels)
    m.set_tensor(h["input"], feats)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    relu_of = {nd["layer"]: nd["out"] for nd in ir.nodes if nd["kind"] == "relu"}
    out = dict(ir=ir, h=h, feats=feats, labels=labels, mask=mask, info=m.op_info(), steps=[], graph=graph, loss=loss,
               dtypes={t: m.tensor_dtype(t) for t in ir.width})
    for _ in range(steps):
        st = dict(w0=[m.get_parameter(p) for p in range(m.num_parameters())])
        m.train_mode(); m.zero_gradients(); m.forward()
        st["logits"] = m.get_tensor(h["logits"])
        st["relu"] = {l: m.get_tensor(t) > 0 for l, t in relu_of.items()}
        m.backward()
        st["dw"] = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
        st["w1"] = [m.get_parameter(p) for p in range(m.num_parameters())]
        out["steps"].append(st)
    host.close()
    return out


def check_witness(run, feats=None):
    feats = run["feats"] if feats is None else feats
    loss_fn = bce_train_loss if run["loss"] == "sigmoid" else train_loss
    for k, st in enumerate(run["steps"]):
        wt = witness(run["ir"], run["graph"], feats, run["labels"], run["mask"], st["w0"], step=k + 1,
                     relu_masks=st["relu"], loss_fn=loss_fn)
        close("step %d logits" % k, st["logits"], wt["logits"])
        for p, (a, b) in enumerate(zip(st["dw"], wt["dW"])):
            close("step %d dW%d" % (k, p), a, b)


def check_identical(a, b):
    for sa, sb in zip(a["steps"], b["steps"]):
        assert np.array_equal(sa["logits"].view(np.int32), sb["logits"].view(np.int32))
        for k in ("dw", "w1"):
            for x, y in zip(sa[k], sb[k]):
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), k


def check_fusion(name, fused, unfused):
    """every hop's scaled_add is fused into its scatter_gather; APPNP's next hop's first norm too, all but the last"""
    ir, info = fused["ir"], fused["info"]
    sgs = [nd for nd in ir.nodes if nd["kind"] == "scatter_gather"]
    for i, sg in enumerate(sgs):
        n2 = next(nd for nd in ir.nodes if nd["ins"] == [sg["out"]])
        sa = next(nd for nd in ir.nodes if nd["kind"] == "scaled_add" and nd["ins"][0] == n2["out"])
        assert info[n2["layer"]]["fusedInto"] == sg["layer"] and info[sa["layer"]]["fusedInto"] == sg["layer"]
        nxt = [nd for nd in ir.nodes if nd["ins"] == [sa["out"]] and nd["kind"] == "indegree_norm"]
        if name == "appnp" and i != len(sgs) - 1:
            assert info[sg["layer"]]["epilogue"] == NORM | NORM_OUT, i
            assert info[sg["layer"]]["fwdOut"] == nxt[0]["out"]
            assert info[nxt[0]["layer"]]["fusedInto"] == sg["layer"]
        else:
            assert info[sg["layer"]]["epilogue"] == NORM, i
            assert info[sg["layer"]]["fwdOut"] == sa["out"]
        assert unfused["info"][sg["layer"]]["epilogue"] == 0 and unfused["info"][sa["layer"]]["fusedInto"] == -1
    assert len(sgs) == (10 if name == "appnp" else 8)
    assert [i["kind"] for i in info] == [nd["kind"] for nd in ir.nodes]


@pytest.mark.parametrize("name", list(BUILDERS))
def test_model_matches_the_witness(name):
    g = sym_graph()
    fused, unfused = train(name, g, True), train(name, g, False)
    check_witness(fused)
    check_identical(fused, unfused)
    check_fusion(name, fused, unfused)


@pytest.mark.parametrize("name", list(BUILDERS))
def test_model_with_exact_backward_on_a_directed_multigraph(name):
    re_, col = directed_graph()
    # a duplicate of every 7th edge, kept in its row
    deg = np.diff(np.concatenate([[0], re_.astype(np.int64)]))
    rows = np.split(col, np.cumsum(deg)[:-1])
    rows = [np.concatenate([r, r[::7]]) for r in rows]
    g = (np.cumsum([len(r) for r in rows]).astype(np.uint64), np.concatenate(rows).astype(np.uint32))
    fused, unfused = train(name, g, True, exact_backward=True), train(name, g, False, exact_backward=True)
    check_witness(fused)
    check_identical(fused, unfused)


@pytest.mark.parametrize("name", list(BUILDERS))
def test_model_with_bf16_features(name):
    g = sym_graph()
    fused, unfused = train(name, g, True, features="bfloat16"), train(name, g, False, features="bfloat16")
    assert fused["dtypes"][fused["h"]["input"]] == "bfloat16"
    check_witness(fused, bf16.round_f32(fused["feats"]))
    check_identical(fused, unfused)


@pytest.mark.parametrize("name", list(BUILDERS))
def test_model_with_sigmoid_loss(name):
    g = sym_graph()
    fused, unfused = train(name, g, True, loss="sigmoid"), train(name, g, False, loss="sigmoid")
    check_witness(fused)
    check_identical(fused, unfused)


@pytest.mark.parametrize("name", list(BUILDERS))
def test_bf16_aggregation_picks_no_tensor(name):
    g = sym_graph()
    run = train(name, g, True, steps=1, bf16_aggregation=True)
    assert "bfloat16" not in run["dtypes"].values(), run["dtypes"]
    check_fusion(name, run, train(name, g, False, steps=1))
    plain = train(name, g, True, steps=1)
    check_identical(run, plain)


def test_teleport_left_unfused_where_bf16_aggregation_reads_the_sum():
    """bf16 aggregation stores the scatter_gather's input in bf16, for which there is no teleport: the scaled_add stays
    apart, the model trains, and it computes the unfused model's values to bf16 rounding.  Without bf16 aggregation the
    same layer is fused and matches the fp64 witness."""
    g = sym_graph()
    run = train("gcn_residual", g, True, bf16_aggregation=True)
    ir, info = run["ir"], run["info"]
    sg = next(nd for nd in ir.nodes if nd["kind"] == "scatter_gather")
    sa = next(nd for nd in ir.nodes if nd["kind"] == "scaled_add")
    assert run["dtypes"][sg["ins"][0]] == "bfloat16"
    assert info[sa["layer"]]["fusedInto"] == -1 and info[sg["layer"]]["epilogue"] == NORM
    plain = train("gcn_residual", g, False, steps=1, bf16_aggregation=True)
    assert "bfloat16" not in plain["dtypes"].values()
    close("bf16 logits", run["steps"][0]["logits"], plain["steps"][0]["logits"], rtol=2e-2, atol_scale=1e-2)
    for st in run["steps"]:
        assert all(np.isfinite(w).all() for w in st["w1"])
    fused = train("gcn_residual", g, True)
    assert fused["info"][sa["layer"]]["fusedInto"] == sg["layer"]
    assert fused["info"][sg["layer"]]["epilogue"] == NORM and fused["info"][sg["layer"]]["fwdOut"] == sa["out"]
    check_witness(fused)
    check_identical(fused, train("gcn_residual", g, False))
