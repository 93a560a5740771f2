"""GATv2's dynamic attention on the GPU.

Kernels: roc_sg_attn_v2_forward_planned, roc_sg_attn_v2_backward_planned and roc_sg_attn_v2_backward_exact against the
fp64 autograd witness of tests/gatv2_witness.py, over H in {1, 2, 3, 5, 8, 12, 24, 41, 64, 65, 128, 129, 256} with
every head count of {1, 2, 3, 4, 6, 8} that divides H (F = 2 and 3 straddle float4 groups), on a symmetric graph with
heavy rows cut across chunks and one row that takes a whole CTA's fix-up (the same-CSR backward is exact there), and on
a directed multigraph for the exact backward.  Rows live in NaN-padded buffers.  Also xl is xr, repeat calls and three
SM budgets byte-identical, the launch lists, and the refusals.

Models: build_gatv2 over three Adam steps against the witness (each step from the product's weights), at 1 head and
8 heads of 8, share_weights both ways, exact_backward on a directed graph, activation="elu" and loss="sigmoid"; norm,
bf16 features, infer mode, parameter_shape, op_info and set_bf16_aggregation.

Bounds: each output against fp64 with |got - want| <= 2e-4 |want| + 2e-5 max|want| (the bar of test_opgraph_gpu.py);
da, a column sum over every edge, at 1e-3 |want| + 1e-4 max|want|."""
import numpy as np
import pytest
import torch

import sg_matrix as sgm

from gatv2_witness import kernel_witness, model_witness
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_gatv2
from witness_gat import train_loss

pytestmark = pytest.mark.gpu

HS = [1, 2, 3, 5, 8, 12, 24, 41, 64, 65, 128, 129, 256]
# 192, 200 and 224 reach J = ceil(H / 32) = 6 and 7, so that with the list above every J = 1..8 runs
SHAPES = [(h, k) for h in HS for k in (1, 2, 3, 4, 6, 8) if h % k == 0] + [(192, 6), (200, 8), (224, 7)]
SLOPE = 0.2


def close(name, got, want, rtol=2e-4, atol_scale=2e-5):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.isfinite(got).all(), name
    scale = np.abs(want).max() if want.size else 0.0
    bound = rtol * np.abs(want) + atol_scale * scale + 1e-30
    r = float((np.abs(got - want) / bound).max()) if want.size else 0.0
    assert r <= 1.0, (name, r)


def sym_graph():
    """a symmetric graph with self loops, heavy rows (degree > 64) and one hub whose row spans > 32 chunks"""
    rng = np.random.RandomState(7)
    n = 3000
    pairs = {(i, i) for i in range(n)}
    for _ in range(6000):
        u, v = rng.randint(0, n, 2)
        pairs |= {(u, v), (v, u)}
    for u in range(1, 2600):                       # hub 0: 2600 edges, 41 chunks
        pairs |= {(0, u), (u, 0)}
    for u in range(100, 300):                      # row 5: a heavy row of a few chunks
        pairs |= {(5, u), (u, 5)}
    return _csr(n, sorted(pairs))


def directed_multigraph():
    rng = np.random.RandomState(8)
    n = 2000
    pairs = [(i, i) for i in range(n)]
    pairs += [tuple(rng.randint(0, n, 2)) for _ in range(9000)]
    pairs += [(3, u) for u in range(0, 1500)] + [(3, 7)] * 3     # a big row and duplicate edges
    return _csr(n, sorted(pairs))


def _csr(n, pairs):
    """pairs (dst, src) sorted by dst -> (row_end u64, col u32)"""
    dst = np.array([p[0] for p in pairs], dtype=np.int64)
    col = np.array([p[1] for p in pairs], dtype=np.uint32)
    row_end = np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64)
    return row_end, col


GRAPHS = {}


def graph(name):
    if name not in GRAPHS:
        re_, col = {"sym": sym_graph, "directed": directed_multigraph}[name]()
        dre = torch.from_numpy(re_.astype(np.int64)).cuda()
        dcol = torch.from_numpy(col.astype(np.int32)).cuda()
        n = re_.shape[0]
        GRAPHS[name] = dict(row_end=re_, col=col, plan=K.SgPlan(0, n - 1, 0, dre, dcol), tr=K.SgTranspose(dre, dcol),
                            n=n)
    return GRAPHS[name]


def nan_rows(v):
    """v [rows][h] (numpy) in a NaN-filled buffer of pitch h + 3 rounded up to 4, on the GPU"""
    rows, h = v.shape
    buf = torch.full((rows, (h + 3 + 3) // 4 * 4), float("nan"), device="cuda")
    buf[:, :h] = torch.from_numpy(np.asarray(v, dtype=np.float32))
    return buf[:, :h]


def inputs(n, h, heads, seed):
    rng = np.random.RandomState(seed)
    xl = rng.standard_normal((n, h)).astype(np.float32)
    xr = rng.standard_normal((n, h)).astype(np.float32)
    a = rng.uniform(-1, 1, (heads, h // heads)).astype(np.float32)
    gy = rng.standard_normal((n, h)).astype(np.float32)
    return xl, xr, a, gy


def run(g, xl, xr, a, gy, heads, exact=False, shared=False):
    dxl_, xr_ = nan_rows(xl), None
    xr_ = dxl_ if shared else nan_rows(xr)
    xl_ = dxl_
    ta = torch.from_numpy(a).cuda()
    out, stats = g["plan"].attn_v2_forward(xl_, xr_, ta, heads, SLOPE)
    gy_ = nan_rows(gy)
    if exact:
        dxl, dxr, da = g["tr"].attn_v2_backward(g["plan"], xl_, xr_, ta, out, stats, gy_, heads, SLOPE)
    else:
        dxl, dxr, da = g["plan"].attn_v2_backward(xl_, xr_, ta, out, stats, gy_, heads, SLOPE)
    torch.cuda.synchronize()
    return dict(out=out.cpu().numpy(), stats=stats.cpu().numpy(), dxl=dxl.cpu().numpy(), dxr=dxr.cpu().numpy(),
                da=da.cpu().numpy())


def check(got, want, heads, what, shared=False):
    close(what + " out", got["out"], want["out"])
    close(what + " m", got["stats"][:, :heads], want["m"])
    close(what + " 1/Z", got["stats"][:, heads:2 * heads], want["iz"])
    if shared:
        close(what + " dx", got["dxl"] + got["dxr"], want["dxl"])
    else:
        close(what + " dxl", got["dxl"], want["dxl"])
        close(what + " dxr", got["dxr"], want["dxr"])
    close(what + " da", got["da"], want["da"], rtol=1e-3, atol_scale=1e-4)


@pytest.mark.parametrize("h,heads", SHAPES)
def test_kernels_against_fp64_on_a_symmetric_graph(h, heads):
    g = graph("sym")
    xl, xr, a, gy = inputs(g["n"], h, heads, seed=h * 10 + heads)
    want = kernel_witness(g["row_end"], g["col"], xl, xr, a, gy, heads, SLOPE)
    got = run(g, xl, xr, a, gy, heads)
    check(got, want, heads, "H=%d heads=%d" % (h, heads))
    info = g["plan"].info()
    assert info["heavy_rows"] > 0


@pytest.mark.parametrize("h,heads", [(1, 1), (12, 3), (24, 8), (64, 8), (129, 3), (256, 4)])
def test_exact_backward_on_a_directed_multigraph(h, heads):
    g = graph("directed")
    xl, xr, a, gy = inputs(g["n"], h, heads, seed=h + heads)
    want = kernel_witness(g["row_end"], g["col"], xl, xr, a, gy, heads, SLOPE)
    check(run(g, xl, xr, a, gy, heads, exact=True), want, heads, "exact H=%d heads=%d" % (h, heads))


@pytest.mark.parametrize("h,heads", [(8, 4), (64, 1), (65, 5)])
def test_shared_input(h, heads):
    g = graph("sym")
    xl, _, a, gy = inputs(g["n"], h, heads, seed=3)
    want = kernel_witness(g["row_end"], g["col"], xl, xl, a, gy, heads, SLOPE)
    check(run(g, xl, xl, a, gy, heads, shared=True), want, heads, "shared", shared=True)
    g2 = graph("directed")
    xl, _, a, gy = inputs(g2["n"], h, heads, seed=4)
    want = kernel_witness(g2["row_end"], g2["col"], xl, xl, a, gy, heads, SLOPE)
    check(run(g2, xl, xl, a, gy, heads, exact=True, shared=True), want, heads, "shared exact", shared=True)


def _bits(r):
    return {k: v.view(np.int32).copy() for k, v in r.items()}


@pytest.mark.parametrize("h,heads", [(3, 3), (64, 8), (129, 3), (256, 8)])
def test_repeats_and_sm_budgets_are_byte_identical(h, heads):
    for name, exact in (("sym", False), ("directed", True)):
        g = graph(name)
        xl, xr, a, gy = inputs(g["n"], h, heads, seed=11)
        ref = _bits(run(g, xl, xr, a, gy, heads, exact=exact))
        assert all(np.array_equal(v, ref[k]) for k, v in _bits(run(g, xl, xr, a, gy, heads, exact=exact)).items())
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        prev = _lib.lib.roc_set_sm_reserve(0)
        try:
            for reserve in (sms - 8, sms // 2 + 1):     # 8 SMs and an odd count, beside the whole chip above
                _lib.lib.roc_set_sm_reserve(int(reserve))
                got = _bits(run(g, xl, xr, a, gy, heads, exact=exact))
                assert all(np.array_equal(v, ref[k]) for k, v in got.items()), (name, reserve)
        finally:
            _lib.lib.roc_set_sm_reserve(prev)


# The launch lists, restated (kind, red, vec, lanes, nch, grid), on a plan of schedule s and, for the source pass, sB
# (s itself, or the transposed plan's).  J = ceil(H / 32); (L, NCH) the sum's row shape for H scalar columns.
def v2_forward_launches(s, h):
    j, (lanes, nch) = sgm.cdiv(h, 32), sgm.shape(h)
    out = [("main", 64, 1, 32, j, sgm.cdiv(s.chunks, 8))]
    if s.heavy + s.big:
        out.append(("stat_fixup", 64, 1, 32, 1, sgm.cdiv(s.heavy + s.big, 8)))
    return out + [("main", 65, 1, 32, j, sgm.cdiv(s.chunks, 8))] + sgm.fixups(s, 0, 1, lanes, nch)


def v2_backward_launches(s, sb, n, h):
    j, (lanes, nch) = sgm.cdiv(h, 32), sgm.shape(h)
    out = [("record", -1, 1, 32, j, sgm.cdiv(n, 8))] if n else []
    out += [("main", 66, 1, 32, j, sgm.cdiv(s.chunks, 8))] + 2 * sgm.fixups(s, 0, 1, lanes, nch)   # dxr, then R
    out += [("main", 67, 1, 32, j, sgm.cdiv(sb.chunks, 8))] + sgm.fixups(sb, 0, 1, lanes, nch)
    if n:
        out += [("colsum", -1, 1, 256, 1, sgm.cdiv(n, 512)), ("colsum", -1, 1, 256, 1, 1)]
    return out


def launched():
    return [(l["kind"], l["red"], l["vec"], l["lanes"], l["nch"], l["grid"]) for l in K.sg_launches()]


SEEN = set()     # (red, J) of every main launch the file made


def run_matrix(g, h, heads, seed):
    """forward, same-CSR backward and exact backward of one sg_matrix graph, each launch list checked"""
    xl, xr, a, gy = inputs(g.n, h, heads, seed)
    xl_, xr_, gy_, ta = nan_rows(xl), nan_rows(xr), nan_rows(gy), torch.from_numpy(a).cuda()
    def check(want, what):
        got = launched()
        assert got == want, (g.name, h, what, got, want)
        SEEN.update((l[1], l[4]) for l in got if l[0] == "main")
    out, stats = g.plan.attn_v2_forward(xl_, xr_, ta, heads, SLOPE)
    check(v2_forward_launches(g.sched, h), "forward")
    got = dict(out=out, stats=stats)
    got["dxl"], got["dxr"], got["da"] = g.plan.attn_v2_backward(xl_, xr_, ta, out, stats, gy_, heads, SLOPE)
    check(v2_backward_launches(g.sched, g.sched, g.n, h), "backward")
    ex = g.tr.attn_v2_backward(g.plan, xl_, xr_, ta, out, stats, gy_, heads, SLOPE)
    check(v2_backward_launches(g.sched, g.sched_t, g.n, h), "exact backward")
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in got.items()}
    got["exact"] = [v.cpu().numpy() for v in ex]
    return got, kernel_witness(g.row_end, g.col, xl, xr, a, gy, heads, SLOPE)


@pytest.mark.parametrize("h,heads", [(3, 3), (64, 8), (200, 8)])
@pytest.mark.parametrize("name", ["empty", "single", "tiny", "aligned", "straddle", "carry32", "ragged", "directed",
                                  "hub", "fanout"])
def test_sg_matrix_graphs(name, h, heads):
    """The whole graphs of tests/sg_matrix.py: rows of degree 0 (no self loops), rows ending on chunk boundaries,
    32 and 33 carries, heavy and big rows, directed multigraphs.  The forward and the exact backward against the
    witness in full; the same-CSR backward's dxr and da, which come from the forward plan's rows and so are exact on
    any graph (its dxl is exact only on a symmetric graph)."""
    g = sgm.xgraphs()[name]
    got, want = run_matrix(g, h, heads, seed=h + heads)
    what = "%s H=%d heads=%d" % (name, h, heads)
    close(what + " out", got["out"], want["out"])
    close(what + " m", got["stats"][:, :heads], want["m"])
    close(what + " 1/Z", got["stats"][:, heads:2 * heads], want["iz"])
    deg0 = g.deg == 0
    if deg0.any():    # a row of degree 0: out 0 and stats 0 | 0, and zero gradients where nothing reaches it
        assert not got["out"][deg0].any() and not got["stats"][deg0, :2 * heads].any(), what
        assert not got["dxr"][deg0].any(), what
    close(what + " dxr", got["dxr"], want["dxr"])
    close(what + " da", got["da"], want["da"], rtol=1e-3, atol_scale=1e-4)
    dxl, dxr, da = got["exact"]
    close(what + " exact dxl", dxl, want["dxl"])
    close(what + " exact dxr", dxr, want["dxr"])
    close(what + " exact da", da, want["da"], rtol=1e-3, atol_scale=1e-4)
    no_out = np.ones(g.n, bool)
    no_out[g.col.astype(np.int64)] = False
    assert not dxl[no_out].any(), what                  # a node with no out-edge gets no dxl


@pytest.mark.parametrize("h", [1, 33, 65, 97, 129, 161, 193, 225])
def test_every_instantiation(h):
    """J = 1..8: the four passes' main kernels and the record kernel launched, with their lists, on the ragged graph
    (heavy and big rows), against the witness"""
    g = sgm.xgraphs()["ragged"]
    got, want = run_matrix(g, h, 1, seed=h)
    close("J=%d out" % sgm.cdiv(h, 32), got["out"], want["out"])
    close("J=%d exact dxl" % sgm.cdiv(h, 32), got["exact"][0], want["dxl"])
    j = sgm.cdiv(h, 32)
    assert {(r, j) for r in (64, 65, 66, 67)} <= SEEN


def test_refusals():
    g = graph("sym")
    n = g["n"]
    x = torch.zeros((n, 8), device="cuda")
    st = torch.zeros((n, 16), device="cuda")
    a = torch.zeros((8 * 1,), device="cuda")
    p = g["plan"].handle
    f = _lib.lib.roc_sg_attn_v2_forward_planned

    def fw(heads=1, H=8, slope=0.2, xl=x, xr=x, aa=a, out=x, stats=st, ld=8, lds=16):
        return f(p, heads, H, slope, K._ptr(xl), ld, K._ptr(xr), ld, K._ptr(aa), K._ptr(out), ld, K._ptr(stats), lds,
                 None)
    assert fw() == 0
    assert fw(xl=None) == _lib.ROC_ERR_INVALID and fw(aa=None) == _lib.ROC_ERR_INVALID
    assert fw(heads=0) == _lib.ROC_ERR_INVALID and fw(H=0) == _lib.ROC_ERR_INVALID
    assert fw(ld=7, H=8) == _lib.ROC_ERR_INVALID and fw(lds=1) == _lib.ROC_ERR_INVALID
    assert fw(slope=float("nan")) == _lib.ROC_ERR_INVALID and fw(slope=-1.0) == _lib.ROC_ERR_INVALID
    assert fw(heads=3) == _lib.ROC_ERR_UNSUPPORTED
    wide = torch.zeros((n, 260), device="cuda")
    assert fw(H=257, xl=wide, xr=wide, out=wide, ld=260) == _lib.ROC_ERR_UNSUPPORTED
    assert fw(heads=16, H=256, xl=wide, xr=wide, out=wide, ld=260, lds=32) == _lib.ROC_ERR_UNSUPPORTED
    # a plan over a graph slice names ids outside its rows
    sl = sgm.graphs()["slice"]
    xs, ss = torch.zeros((sl.n, 8), device="cuda"), torch.zeros((sl.n, 16), device="cuda")
    assert f(sl.plan.handle, 1, 8, 0.2, K._ptr(xs), 8, K._ptr(xs), 8, K._ptr(a), K._ptr(xs), 8, K._ptr(ss), 16,
             None) == _lib.ROC_ERR_UNSUPPORTED
    b = _lib.lib.roc_sg_attn_v2_backward_planned
    d1, d2 = torch.zeros_like(x), torch.zeros_like(x)

    def bw(dxl=d1, dxr=d2, da=a, H=8):
        return b(p, 1, H, 0.2, K._ptr(x), 8, K._ptr(x), 8, K._ptr(a), K._ptr(x), 8, K._ptr(st), 16, K._ptr(x), 8,
                 K._ptr(dxl), 8, K._ptr(dxr), 8, K._ptr(da), None)
    assert bw() == 0
    assert bw(dxr=d1) == _lib.ROC_ERR_INVALID and bw(da=None) == _lib.ROC_ERR_INVALID
    e = _lib.lib.roc_sg_attn_v2_backward_exact
    other = graph("directed")
    assert e(p, other["tr"].handle, 1, 8, 0.2, K._ptr(x), 8, K._ptr(x), 8, K._ptr(a), K._ptr(x), 8, K._ptr(st), 16,
             K._ptr(x), 8, K._ptr(d1), 8, K._ptr(d2), 8, K._ptr(a), None) == _lib.ROC_ERR_INVALID
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------- the models ---
def sym_model_graph():
    re_, col = datasets.rmat_graph(9, 2500, seed=3)
    return re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


def directed_model_graph():
    re_, col = datasets.rmat_graph(9, 2500, seed=4, directed=True)
    return re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


def bce_loss(logits, labels, mask):
    train = torch.from_numpy(mask == 0)
    x, y = logits[train], torch.from_numpy(np.asarray(labels, dtype=np.float64))[train]
    return torch.nn.functional.binary_cross_entropy_with_logits(x, y, reduction="sum")


def train(layers, heads, graph_, steps=3, loss="softmax", **kw):
    row_end, col = graph_
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    h = build_gatv2(m, layers, 0.0, heads=heads, loss=loss, **kw)
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


def check_model(run, graph_, layers, heads, loss="softmax", **kw):
    row_end, col = graph_
    hs = list(heads) if isinstance(heads, list) else [heads] * (len(layers) - 2)
    for k, st in enumerate(run["steps"]):
        logits, dw = model_witness(row_end, col, run["feats"], run["labels"], run["mask"], layers, st["w0"], hs,
                                   loss_fn=bce_loss if loss == "sigmoid" else train_loss, **kw)
        close("step %d logits" % k, st["logits"], logits)
        for p, (a, b) in enumerate(zip(st["dw"], dw)):
            close("step %d dW%d" % (k, p), a, b, rtol=1e-3, atol_scale=1e-4)


@pytest.mark.parametrize("layers,heads,share", [([24, 16, 12], 1, False), ([24, 64, 12], 8, False),
                                                 ([24, 64, 12], 8, True), ([24, 16, 12], 1, True)])
def test_build_gatv2_against_the_witness(layers, heads, share):
    g = sym_model_graph()
    r = train(layers, heads, g, share_weights=share)
    check_model(r, g, layers, heads, share_weights=share)
    per_layer = 2 if share else 3
    assert len(r["shapes"]) == per_layer * (len(layers) - 1)
    hs = [heads] * (len(layers) - 2) + [1]
    for i, hh in enumerate(hs):
        assert r["shapes"][per_layer * i + per_layer - 1] == (hh, layers[i + 1] // hh)
    kinds = [o["kind"] for o in r["info"]]
    assert kinds.count("attention_gather") == len(layers) - 1 and "attention_scores" not in kinds
    # infer mode: the same logits as the last trained forward would give from the same weights
    m, h = r["m"], r["h"]
    m.infer_mode(); m.forward()
    logits, _ = model_witness(g[0], g[1], r["feats"], r["labels"], r["mask"], layers,
                              [m.get_parameter(p) for p in range(m.num_parameters())], [heads] * (len(layers) - 2),
                              share_weights=share)
    close("infer logits", m.get_tensor(h["logits"]), logits)
    r["host"].close()


def test_exact_backward_on_a_directed_graph():
    g = directed_model_graph()
    r = train([24, 16, 12], 4, g, exact_backward=True)
    check_model(r, g, [24, 16, 12], 4)
    r["host"].close()


def test_elu_and_sigmoid_loss():
    g = sym_model_graph()
    r = train([24, 16, 12], 2, g, activation="elu", loss="sigmoid")
    check_model(r, g, [24, 16, 12], 2, loss="sigmoid", activation="elu")
    r["host"].close()


@pytest.mark.parametrize("kw,wkw", [(dict(norm="batch"), dict(norm="batch")),
                                    (dict(features="bfloat16"), dict(bf16_features=True)),
                                    (dict(norm="batch", share_weights=True), dict(norm="batch", share_weights=True))])
def test_norm_and_bf16_features_against_the_witness(kw, wkw):
    g = sym_model_graph()
    r = train([24, 16, 12], 2, g, **kw)
    check_model(r, g, [24, 16, 12], 2, **wkw)
    r["host"].close()


def test_bf16_aggregation_leaves_the_inputs_fp32():
    g = sym_model_graph()
    host = Host(0, 0, 1)
    host.graph_from_arrays(*g)
    m = Model(host, seed=1)
    m.set_bf16_aggregation(True)
    h = build_gatv2(m, [24, 16, 12], 0.0, heads=2)
    for xl, xr in h["attn_ins"]:
        assert m.tensor_dtype(xl) == "float32" and m.tensor_dtype(xr) == "float32"
    host.close()


def test_repeat_training_is_byte_identical():
    g = sym_model_graph()
    a = train([24, 64, 12], 8, g)
    b = train([24, 64, 12], 8, g)
    for sa, sb in zip(a["steps"], b["steps"]):
        assert np.array_equal(sa["logits"].view(np.int32), sb["logits"].view(np.int32))
        assert all(np.array_equal(x.view(np.int32), y.view(np.int32)) for x, y in zip(sa["dw"], sb["dw"]))
    a["host"].close(); b["host"].close()
