"""The graph transformer's dot-product attention on the GPU.

Kernels: roc_sg_attn_dot_forward_planned, roc_sg_attn_dot_backward_planned and roc_sg_attn_dot_backward_exact against
the fp64 autograd witness of tests/transformer_witness.py, over GATv2's SHAPES matrix (H in {1, ..., 256} with every
head count of {1, 2, 3, 4, 6, 8} that divides H, so that F divides 32, straddles float4 groups, or spans several
warps' columns, and J = 1..8), on a symmetric graph with heavy rows cut across chunks and a hub over 32 chunks (the
same-CSR backward is exact there), and on a directed multigraph for the exact backward; plus the whole graphs of
tests/sg_matrix.py with restated launch lists.  Rows live in NaN-padded buffers.  Also q is k is v, the packed
[q | k | v] buffer, logits up to |s| = 1e3, the inference forward, repeat calls and three SM budgets byte-identical,
and the refusals.

Models: build_graph_transformer over three Adam steps against the witness (each step from the product's weights), at
1 head and 8 heads of 8, root_weight both ways, exact_backward on a directed graph, activation="elu", loss="sigmoid"
and norm; infer mode, fusion off against fusion on, and set_bf16_aggregation.

Bounds: each output against fp64 with |got - want| <= 2e-4 |want| + 2e-5 max|want| (GATv2's)."""
import numpy as np
import pytest
import torch

import sg_matrix as sgm

from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_graph_transformer
from test_gatv2_gpu import SHAPES, bce_loss, close, directed_model_graph, graph, nan_rows, sym_model_graph
from transformer_witness import dot_scale, kernel_witness, model_witness
from witness_gat import train_loss

pytestmark = pytest.mark.gpu


def inputs(n, h, seed, amp=1.0):
    rng = np.random.RandomState(seed)
    return tuple((amp * rng.standard_normal((n, h))).astype(np.float32) for _ in range(4))   # q, k, v, gy


def run(g, q, k, v, gy, heads, exact=False, share=None, packed=False, scale=None):
    """the forward and a backward on the GPU -> numpy dict.  share: None, "qkv" (one tensor) or "kv"; packed: q, k and v
    as column blocks of one [q | k | v] buffer"""
    h = q.shape[1]
    scale = dot_scale(h // heads) if scale is None else scale
    if packed:
        buf = nan_rows(np.concatenate([q, k, v], axis=1))
        q_, k_, v_ = buf[:, :h], buf[:, h:2 * h], buf[:, 2 * h:]
    else:
        q_ = nan_rows(q)
        k_ = q_ if share == "qkv" else nan_rows(k)
        v_ = q_ if share == "qkv" else k_ if share == "kv" else nan_rows(v)
    out, stats = g["plan"].attn_dot_forward(q_, k_, v_, heads, scale)
    gy_ = nan_rows(gy)
    if exact:
        dq, dk, dv = g["tr"].attn_dot_backward(g["plan"], q_, k_, v_, out, stats, gy_, heads, scale)
    else:
        dq, dk, dv = g["plan"].attn_dot_backward(q_, k_, v_, out, stats, gy_, heads, scale)
    torch.cuda.synchronize()
    return dict(out=out.cpu().numpy(), stats=stats.cpu().numpy(), dq=dq.cpu().numpy(), dk=dk.cpu().numpy(),
                dv=dv.cpu().numpy())


def check(got, want, heads, what, share=None):
    close(what + " out", got["out"], want["out"])
    close(what + " m", got["stats"][:, :heads], want["m"])
    close(what + " 1/Z", got["stats"][:, heads:2 * heads], want["iz"])
    if share == "qkv":
        close(what + " dqkv", got["dq"] + got["dk"] + got["dv"], want["dq"])
    elif share == "kv":
        close(what + " dq", got["dq"], want["dq"])
        close(what + " dkv", got["dk"] + got["dv"], want["dk"])
    else:
        for n in ("dq", "dk", "dv"):
            close(what + " " + n, got[n], want[n])


def witness(g, q, k, v, gy, heads, share=None, scale=None):
    h = q.shape[1]
    scale = dot_scale(h // heads) if scale is None else scale
    kk = q if share == "qkv" else k
    vv = q if share == "qkv" else kk if share == "kv" else v
    return kernel_witness(g["row_end"], g["col"], q, kk, vv, gy, heads, scale)


@pytest.mark.parametrize("h,heads", SHAPES)
def test_kernels_against_fp64_on_a_symmetric_graph(h, heads):
    g = graph("sym")
    q, k, v, gy = inputs(g["n"], h, seed=h * 10 + heads)
    check(run(g, q, k, v, gy, heads), witness(g, q, k, v, gy, heads), heads, "H=%d heads=%d" % (h, heads))
    assert g["plan"].info()["heavy_rows"] > 0


@pytest.mark.parametrize("h,heads", [(1, 1), (12, 3), (24, 8), (64, 1), (64, 8), (129, 3), (256, 4)])
def test_exact_backward_on_a_directed_multigraph(h, heads):
    g = graph("directed")
    q, k, v, gy = inputs(g["n"], h, seed=h + heads)
    check(run(g, q, k, v, gy, heads, exact=True), witness(g, q, k, v, gy, heads), heads,
          "exact H=%d heads=%d" % (h, heads))


@pytest.mark.parametrize("h,heads", [(8, 4), (64, 1), (65, 5), (256, 8)])
@pytest.mark.parametrize("share", ["qkv", "kv"])
def test_shared_inputs(h, heads, share):
    for name, exact in (("sym", False), ("directed", True)):
        g = graph(name)
        q, k, v, gy = inputs(g["n"], h, seed=3)
        check(run(g, q, k, v, gy, heads, exact=exact, share=share), witness(g, q, k, v, gy, heads, share=share),
              heads, "%s %s" % (name, share), share=share)


@pytest.mark.parametrize("h,heads", [(3, 3), (41, 1), (64, 8), (128, 1)])
def test_packed_qkv_buffer(h, heads):
    """q, k and v as column blocks of one [q | k | v] buffer (ld 3H, padded), the same bits as three buffers"""
    for name, exact in (("sym", False), ("directed", True)):
        g = graph(name)
        q, k, v, gy = inputs(g["n"], h, seed=5)
        got = run(g, q, k, v, gy, heads, exact=exact, packed=True)
        check(got, witness(g, q, k, v, gy, heads), heads, "packed " + name)
        sep = run(g, q, k, v, gy, heads, exact=exact)
        assert all(np.array_equal(got[n].view(np.int32), sep[n].view(np.int32)) for n in got), name


@pytest.mark.parametrize("h,heads", [(8, 1), (64, 8), (200, 8)])
def test_large_logits(h, heads):
    """|s| up to about 1e3: every exponent is of a difference, so nothing overflows.  q and k hold small integers and
    the scale is 4, so every s is exact in fp32 and the logits of a row differ by 4 or more, or not at all: the
    comparison with fp64 measures the softmax alone."""
    g = graph("sym")
    _, _, v, gy = inputs(g["n"], h, seed=9)
    rng = np.random.RandomState(10)
    q, k = (rng.randint(-8, 9, (g["n"], h)).astype(np.float32) for _ in range(2))
    scale = 4.0
    want = witness(g, q, k, v, gy, heads, scale=scale)
    got = run(g, q, k, v, gy, heads, scale=scale)
    smax = np.abs(want["m"]).max()
    assert 3e2 <= smax <= 3e3, smax
    check(got, want, heads, "large logits H=%d heads=%d" % (h, heads))


def test_inference_forward_writes_no_stats():
    """stats=None: the same out as a training forward, bit for bit (cut rows keep their (m, s) in the plan's
    workspace)"""
    for name in ("sym", "directed"):
        g = graph(name)
        for h, heads in ((24, 3), (64, 1), (256, 8)):
            q, k, v, _ = inputs(g["n"], h, seed=6)
            q_, k_, v_ = nan_rows(q), nan_rows(k), nan_rows(v)
            ref, _ = g["plan"].attn_dot_forward(q_, k_, v_, heads)
            out, stats = g["plan"].attn_dot_forward(q_, k_, v_, heads, keep_stats=False)
            assert stats is None
            assert np.array_equal(out.cpu().numpy().view(np.int32), ref.cpu().numpy().view(np.int32)), (name, h)


def _bits(r):
    return {k: v.view(np.int32).copy() for k, v in r.items()}


@pytest.mark.parametrize("h,heads", [(3, 3), (64, 1), (64, 8), (129, 3), (256, 8)])
def test_repeats_and_sm_budgets_are_byte_identical(h, heads):
    for name, exact in (("sym", False), ("directed", True)):
        g = graph(name)
        q, k, v, gy = inputs(g["n"], h, seed=11)
        ref = _bits(run(g, q, k, v, gy, heads, exact=exact))
        assert all(np.array_equal(x, ref[n]) for n, x in _bits(run(g, q, k, v, gy, heads, exact=exact)).items())
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        prev = _lib.lib.roc_set_sm_reserve(0)
        try:
            for reserve in (sms - 8, sms // 2 + 1):     # 8 SMs and an odd count, beside the whole chip above
                _lib.lib.roc_set_sm_reserve(int(reserve))
                got = _bits(run(g, q, k, v, gy, heads, exact=exact))
                assert all(np.array_equal(x, ref[n]) for n, x in got.items()), (name, reserve)
        finally:
            _lib.lib.roc_set_sm_reserve(prev)


# The launch lists, restated (kind, red, vec, lanes, nch, grid), on a plan of schedule s and, for the source pass, sB
# (s itself, or the transposed plan's).  J = ceil(H / 32); (L, NCH) the sum's row shape for H scalar columns.
def dot_forward_launches(s, h):
    j = sgm.cdiv(h, 32)
    out = [("main", 80, 1, 32, j, sgm.cdiv(s.chunks, 8))]
    if s.heavy:
        out.append(("fixup", 80, 1, 32, j, sgm.cdiv(s.heavy, 8)))
    if s.big:
        out.append(("big_fixup", 80, 1, 32, j, s.big))
    return out


def dot_backward_launches(s, sb, n, h):
    j, (lanes, nch) = sgm.cdiv(h, 32), sgm.shape(h)
    out = [("record", -1, 1, 32, j, sgm.cdiv(n, 8))] if n else []
    out += [("main", 81, 1, 32, j, sgm.cdiv(s.chunks, 8))] + sgm.fixups(s, 0, 1, lanes, nch)       # dq
    out += [("main", 82, 1, 32, j, sgm.cdiv(sb.chunks, 8))] + 2 * sgm.fixups(sb, 0, 1, lanes, nch)  # dk, then dv
    return out


def launched():
    return [(l["kind"], l["red"], l["vec"], l["lanes"], l["nch"], l["grid"]) for l in K.sg_launches()]


SEEN = set()     # (red, J) of every main launch the file made


def run_matrix(g, h, heads, seed):
    """forward, same-CSR backward and exact backward of one sg_matrix graph, each launch list checked"""
    q, k, v, gy = inputs(g.n, h, seed)
    q_, k_, v_, gy_ = nan_rows(q), nan_rows(k), nan_rows(v), nan_rows(gy)

    def check_list(want, what):
        got = launched()
        assert got == want, (g.name, h, what, got, want)
        SEEN.update((l[1], l[4]) for l in got if l[0] == "main")
    out, stats = g.plan.attn_dot_forward(q_, k_, v_, heads)
    check_list(dot_forward_launches(g.sched, h), "forward")
    got = dict(out=out, stats=stats)
    got["dq"], got["dk"], got["dv"] = g.plan.attn_dot_backward(q_, k_, v_, out, stats, gy_, heads)
    check_list(dot_backward_launches(g.sched, g.sched, g.n, h), "backward")
    ex = g.tr.attn_dot_backward(g.plan, q_, k_, v_, out, stats, gy_, heads)
    check_list(dot_backward_launches(g.sched, g.sched_t, g.n, h), "exact backward")
    torch.cuda.synchronize()
    got = {n: x.cpu().numpy() for n, x in got.items()}
    got["exact"] = [x.cpu().numpy() for x in ex]
    return got, kernel_witness(g.row_end, g.col, q, k, v, gy, heads, dot_scale(h // heads))


@pytest.mark.parametrize("h,heads", [(3, 3), (64, 8), (200, 8)])
@pytest.mark.parametrize("name", ["empty", "single", "tiny", "aligned", "straddle", "carry32", "ragged", "directed",
                                  "hub", "fanout"])
def test_sg_matrix_graphs(name, h, heads):
    """The whole graphs of tests/sg_matrix.py: rows of degree 0 (no self loops), rows ending on chunk boundaries, 32
    and 33 carries, heavy and big rows, directed multigraphs.  The forward and the exact backward against the witness
    in full; the same-CSR backward's dq, which comes from the forward plan's rows and so is exact on any graph."""
    g = sgm.xgraphs()[name]
    got, want = run_matrix(g, h, heads, seed=h + heads)
    what = "%s H=%d heads=%d" % (name, h, heads)
    close(what + " out", got["out"], want["out"])
    close(what + " m", got["stats"][:, :heads], want["m"])
    close(what + " 1/Z", got["stats"][:, heads:2 * heads], want["iz"])
    deg0 = g.deg == 0
    if deg0.any():    # a row of degree 0: out 0 and stats 0 | 0, and dq 0
        assert not got["out"][deg0].any() and not got["stats"][deg0, :2 * heads].any(), what
        assert not got["dq"][deg0].any(), what
    close(what + " dq", got["dq"], want["dq"])
    dq, dk, dv = got["exact"]
    close(what + " exact dq", dq, want["dq"])
    close(what + " exact dk", dk, want["dk"])
    close(what + " exact dv", dv, want["dv"])
    no_out = np.ones(g.n, bool)
    no_out[g.col.astype(np.int64)] = False
    assert not dk[no_out].any() and not dv[no_out].any(), what     # a node with no out-edge gets no dk, dv


@pytest.mark.parametrize("h", [1, 33, 65, 97, 129, 161, 193, 225])
def test_every_instantiation(h):
    """J = 1..8: the three passes' main kernels, the forward fix-ups and the record kernel launched, with their lists,
    on the ragged graph (heavy and big rows), against the witness"""
    g = sgm.xgraphs()["ragged"]
    got, want = run_matrix(g, h, 1, seed=h)
    j = sgm.cdiv(h, 32)
    close("J=%d out" % j, got["out"], want["out"])
    close("J=%d exact dk" % j, got["exact"][1], want["dk"])
    close("J=%d exact dv" % j, got["exact"][2], want["dv"])
    assert {(r, j) for r in (80, 81, 82)} <= SEEN


def test_refusals():
    g = graph("sym")
    n = g["n"]
    x, y, z = (torch.zeros((n, 8), device="cuda") for _ in range(3))
    o = torch.zeros((n, 8), device="cuda")
    st = torch.zeros((n, 16), device="cuda")
    p = g["plan"].handle
    f = _lib.lib.roc_sg_attn_dot_forward_planned

    def fw(heads=1, H=8, scale=0.5, q=x, k=y, v=z, out=o, stats=st, ld=8, lds=16, plan=p):
        return f(plan, heads, H, scale, K._ptr(q), ld, K._ptr(k), ld, K._ptr(v), ld, K._ptr(out), ld, K._ptr(stats),
                 lds, None)
    assert fw() == 0 and fw(stats=None, lds=0) == 0 and fw(k=x, v=x) == 0
    assert fw(q=None) == _lib.ROC_ERR_INVALID and fw(v=None) == _lib.ROC_ERR_INVALID
    assert fw(out=None) == _lib.ROC_ERR_INVALID
    assert fw(heads=0) == _lib.ROC_ERR_INVALID and fw(H=0) == _lib.ROC_ERR_INVALID
    assert fw(ld=7, H=8) == _lib.ROC_ERR_INVALID and fw(lds=1) == _lib.ROC_ERR_INVALID
    for bad in (0.0, float("nan"), float("inf"), -float("inf")):
        assert fw(scale=bad) == _lib.ROC_ERR_INVALID, bad
    assert fw(out=x) == _lib.ROC_ERR_INVALID and fw(stats=o) == _lib.ROC_ERR_INVALID
    assert fw(heads=3) == _lib.ROC_ERR_UNSUPPORTED
    wide = torch.zeros((n, 260), device="cuda")
    wo = torch.zeros((n, 260), device="cuda")
    assert fw(H=257, q=wide, k=wide, v=wide, out=wo, ld=260) == _lib.ROC_ERR_UNSUPPORTED
    assert fw(heads=16, H=256, q=wide, k=wide, v=wide, out=wo, ld=260, lds=32) == _lib.ROC_ERR_UNSUPPORTED
    # a plan over a graph slice names ids outside its rows
    sl = sgm.graphs()["slice"]
    xs, os_, ss = (torch.zeros((sl.n, c), device="cuda") for c in (8, 8, 16))
    assert f(sl.plan.handle, 1, 8, 0.5, K._ptr(xs), 8, K._ptr(xs), 8, K._ptr(xs), 8, K._ptr(os_), 8, K._ptr(ss), 16,
             None) == _lib.ROC_ERR_UNSUPPORTED
    b = _lib.lib.roc_sg_attn_dot_backward_planned
    d1, d2, d3 = (torch.zeros_like(x) for _ in range(3))

    def bw(dq=d1, dk=d2, dv=d3, H=8, scale=0.5, stats=st, heads=1):
        return b(p, heads, H, scale, K._ptr(x), 8, K._ptr(y), 8, K._ptr(z), 8, K._ptr(o), 8, K._ptr(stats), 16,
                 K._ptr(o), 8, K._ptr(dq), 8, K._ptr(dk), 8, K._ptr(dv), 8, None)
    assert bw() == 0
    assert bw(dk=d1) == _lib.ROC_ERR_INVALID and bw(dv=d1) == _lib.ROC_ERR_INVALID and bw(dv=d2) == _lib.ROC_ERR_INVALID
    assert bw(dq=x) == _lib.ROC_ERR_INVALID and bw(dv=o) == _lib.ROC_ERR_INVALID
    assert bw(stats=None) == _lib.ROC_ERR_INVALID and bw(dq=None) == _lib.ROC_ERR_INVALID
    assert bw(scale=0.0) == _lib.ROC_ERR_INVALID and bw(heads=3) == _lib.ROC_ERR_UNSUPPORTED
    e = _lib.lib.roc_sg_attn_dot_backward_exact
    other = graph("directed")
    for tr, want in ((g["tr"], 0), (other["tr"], _lib.ROC_ERR_INVALID)):
        assert e(p, tr.handle, 1, 8, 0.5, K._ptr(x), 8, K._ptr(y), 8, K._ptr(z), 8, K._ptr(o), 8, K._ptr(st), 16,
                 K._ptr(o), 8, K._ptr(d1), 8, K._ptr(d2), 8, K._ptr(d3), 8, None) == want
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------- the models ---
def train(layers, heads, graph_, steps=3, loss="softmax", fuse=True, bf16_aggregation=False, **kw):
    row_end, col = graph_
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    if not fuse:
        m.set_fusion(False)
    if bf16_aggregation:
        m.set_bf16_aggregation(True)
    h = build_graph_transformer(m, layers, 0.0, heads=heads, loss=loss, **kw)
    if loss == "sigmoid":
        feats, labels, mask = (t.numpy() for t in datasets.multilabel_node_data(n, layers[0], layers[-1], seed=5))
        m.set_multilabels(h["label"], labels)
    else:
        feats, labels, mask = (t.numpy() for t in datasets.node_data(n, layers[0], layers[-1], seed=5))
        m.set_labels(h["label"], labels)
    m.set_tensor(h["input"], feats)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    out = dict(h=h, feats=feats, labels=labels, mask=mask, info=m.op_info(), steps=[], m=m, host=host,
               shapes=[m.parameter_shape(p) for p in range(m.num_parameters())])
    for _ in range(steps):
        st = dict(w0=[m.get_parameter(p) for p in range(m.num_parameters())])
        m.train_mode(); m.zero_gradients(); m.forward()
        st["logits"] = m.get_tensor(h["logits"])
        m.backward()
        st["dw"] = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
        out["steps"].append(st)
    return out


def check_model(run_, graph_, layers, heads, loss="softmax", **kw):
    row_end, col = graph_
    hs = list(heads) if isinstance(heads, list) else [heads] * (len(layers) - 2)
    for k, st in enumerate(run_["steps"]):
        logits, dw = model_witness(row_end, col, run_["feats"], run_["labels"], run_["mask"], layers, st["w0"], hs,
                                   loss_fn=bce_loss if loss == "sigmoid" else train_loss, **kw)
        close("step %d logits" % k, st["logits"], logits)
        for p, (a, b) in enumerate(zip(st["dw"], dw)):
            close("step %d dW%d" % (k, p), a, b, rtol=1e-3, atol_scale=1e-4)


@pytest.mark.parametrize("layers,heads,root_weight", [([24, 16, 12], 1, True), ([24, 64, 12], 8, True),
                                                       ([24, 64, 12], 8, False), ([24, 16, 12], 1, False)])
def test_build_graph_transformer_against_the_witness(layers, heads, root_weight):
    g = sym_model_graph()
    r = train(layers, heads, g, root_weight=root_weight)
    check_model(r, g, layers, heads, root_weight=root_weight)
    per_layer = 4 if root_weight else 3
    assert len(r["shapes"]) == per_layer * (len(layers) - 1)
    kinds = [o["kind"] for o in r["info"]]
    assert kinds.count("attention_gather") == len(layers) - 1 and "attention_scores" not in kinds
    # infer mode: the logits the witness gives from the trained weights
    m, h = r["m"], r["h"]
    m.infer_mode(); m.forward()
    logits, _ = model_witness(g[0], g[1], r["feats"], r["labels"], r["mask"], layers,
                              [m.get_parameter(p) for p in range(m.num_parameters())], [heads] * (len(layers) - 2),
                              root_weight=root_weight)
    close("infer logits", m.get_tensor(h["logits"]), logits)
    r["host"].close()


def test_exact_backward_on_a_directed_graph():
    g = directed_model_graph()
    r = train([24, 16, 12], 4, g, exact_backward=True)
    check_model(r, g, [24, 16, 12], 4)
    r["host"].close()


@pytest.mark.parametrize("norm", ["batch", "layer_norm"])
def test_elu_sigmoid_loss_and_norm(norm):
    g = sym_model_graph()
    r = train([24, 16, 12], 2, g, activation="elu", loss="sigmoid", norm=norm)
    check_model(r, g, [24, 16, 12], 2, loss="sigmoid", activation="elu", norm=norm)
    r["host"].close()


def test_fusion_off_is_bit_identical_to_fusion_on():
    g = sym_model_graph()
    a = train([24, 64, 12], 8, g, norm="batch")
    b = train([24, 64, 12], 8, g, norm="batch", fuse=False)
    for sa, sb in zip(a["steps"], b["steps"]):
        assert np.array_equal(sa["logits"].view(np.int32), sb["logits"].view(np.int32))
        assert all(np.array_equal(x.view(np.int32), y.view(np.int32)) for x, y in zip(sa["dw"], sb["dw"]))
    a["host"].close(); b["host"].close()


def test_bf16_aggregation_leaves_q_k_v_fp32():
    g = sym_model_graph()
    r = train([24, 16, 12], 2, g, bf16_aggregation=True, steps=1)
    m, h = r["m"], r["h"]
    for qkv in h["attn_ins"]:
        assert all(m.tensor_dtype(t) == "float32" for t in qkv)
    check_model(r, g, [24, 16, 12], 2)
    r["host"].close()


def test_repeat_training_is_byte_identical():
    g = sym_model_graph()
    a = train([24, 64, 12], 8, g)
    b = train([24, 64, 12], 8, g)
    for sa, sb in zip(a["steps"], b["steps"]):
        assert np.array_equal(sa["logits"].view(np.int32), sb["logits"].view(np.int32))
        assert all(np.array_equal(x.view(np.int32), y.view(np.int32)) for x, y in zip(sa["dw"], sb["dw"]))
    a["host"].close(); b["host"].close()
