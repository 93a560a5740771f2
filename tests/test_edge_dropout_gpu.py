"""Edge dropout of the sum ScatterGather on the GPU (roc_sg_forward_dropout_planned,
roc_sg_forward_teleport_dropout_planned, roc_sg_transpose_sum_backward_dropout; Model.scatter_gather(dropout=),
build_gcn / build_appnp(edge_dropout=)).

The bit contract: on finite inputs each call's bytes equal the weighted sum with w[e] = keep ? s : 0 followed by the
unfused kernels its epilogue replaces.  That is checked on the graphs test_teleport_gpu.py uses (heavy and big fix-ups,
rows of degree 0, a slice with global ids), on float4 and scalar rows up to 2,051 columns, at rates 0.1, 0.5 and 0.9,
with an fp64 bound beside it; the backward over the same CSR against the weighted sum with reverse-pair weights, and
the exact backward against SgTranspose.backward; source rows only dropped edges read hold NaN and are never read.  The
models train three Adam steps against the fp64 witness of edge_dropout_witness.py, fused and unfused byte-identical."""
import numpy as np
import pytest
import torch

import sg_matrix as M
from edge_dropout_witness import drop_scale, edge_keep, witness
from opgraph import Recorder
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_appnp, build_gcn
from test_batchnorm_gpu import close, directed_graph, sym_graph

pytestmark = pytest.mark.gpu
DROP = _lib.SG_RED_DROP
SUM, TSUM, TELE = 0, 10, _lib.SG_RED_TELE
NORM, RELU, NORM_OUT = _lib.SG_EPI_NORM, _lib.SG_EPI_RELU, _lib.SG_EPI_NORM_OUT
ALPHA, BETA = float(np.float32(0.9)), float(np.float32(0.1))
RATES = (0.1, 0.5, 0.9)
GRAPHS = ("single", "tiny", "aligned", "straddle", "carry32", "ragged", "slice")
VEC_WIDTHS = sorted({w for qc, _, _ in M.RUNGS for w in (4 * qc - 3, 4 * qc)} | {1025, 2051})
KEY, STEP = (7 << 32) | 3, 5
U = 2.0 ** -24


# ------------------------------------------------------------------------------------------------ helpers ---
def want_launches(s, red, fix, vec, h):
    """per column block of the sum's width (1,024 floats on float4 rows, 256 scalar): the dropped main kernel on the
    register kernel, then the fix-ups of the form without dropout"""
    vw = 4 if vec else 1
    block = vw * 256
    out = []
    for c0 in range(0, h, block):
        lanes, nch = M.shape(M.cdiv(min(h - c0, block), vw))
        out.append(("main", red, vw, lanes, nch, M.cdiv(s.chunks, 256 // lanes)))
        out += M.fixups(s, fix, vw, lanes, nch)
    return out


def rows(rng, n, h):
    a = rng.standard_normal((n, h)).astype(np.float32)
    a[rng.random_sample((n, h)) < 0.05] = 0.0
    return a


def weights(keep, rate):
    """the weighted sum's w = keep ? s : 0 (bit 0 of each keep byte), on the device"""
    k = (keep & 1).bool()
    return torch.where(k, torch.tensor(drop_scale(rate), device=M.DEV), torch.tensor(0.0, device=M.DEV)).float()


def epilogue_chain(g_re, g, y, epi, vec, h, row_left=0, row_right=None, col_left=0):
    """NORM: roc_indegree_norm; RELU: then relu, each into a fresh output laid out like y"""
    if epi & NORM:
        z = M.guarded(y.shape[0], h, vec)
        K.indegree_norm(row_left, row_right if row_right is not None else y.shape[0] - 1, col_left, g_re, y,
                        out=z.view)
        y = z.view
    if epi & RELU:
        y = K.activation_fwd(y, _lib.AC_MODE_RELU)
    return y


def bits(t):
    return t.cpu().contiguous().view(torch.int32).numpy()


def fp64_sum(g, x, keep, rate, epi):
    """the dropped sum in fp64 and the same sum over |terms|, with the norm"""
    c = g.col.astype(np.int64)
    dst = np.repeat(np.arange(g.nloc), g.deg)
    w = np.where(keep & 1, drop_scale(rate), 0.0)[:, None]
    xs = x.astype(np.float64)[c]
    out, mag = np.zeros((g.nloc, x.shape[1])), np.zeros((g.nloc, x.shape[1]))
    np.add.at(out, dst, w * xs)
    np.add.at(mag, dst, np.abs(w * xs))
    if epi & NORM:
        d = np.sqrt(g.deg.astype(np.float64))[:, None]
        with np.errstate(invalid="ignore", divide="ignore"):
            out, mag = out / d, mag / d
    if epi & RELU:
        out = np.maximum(out, 0)
    return out, mag


def within_fp64(g, got, x, keep, rate, epi, what):
    want, mag = fp64_sum(g, x, keep, rate, epi)
    ok = np.isfinite(want)
    M.close_terms(got[ok], want[ok], mag[ok], what, (int(g.deg.max()) + 4) * U)


# ------------------------------------------------------------------------------------------- kernel matrix ---
@pytest.mark.parametrize("name", GRAPHS)
@pytest.mark.parametrize("vec", [True, False], ids=["vec", "scalar"])
def test_forward_is_the_weighted_chain(name, vec):
    g = M.graphs()[name]
    rng = np.random.RandomState(len(name) * 5 + vec)
    seen = set()
    for h in (VEC_WIDTHS if vec else M.SCALAR):
        xh = rows(rng, g.n, h)
        x = M.dev_in(xh, vec)
        t = M.dev_in(rows(rng, g.nloc, h), vec)
        for rate in RATES:
            keep = g.plan.attn_keep_mask(rate, KEY, STEP, self_base=g.self_base)
            w = weights(keep, rate)
            keep_h = keep.cpu().numpy()[:g.E]
            ws = M.guarded(g.nloc, h, vec)
            g.plan.weighted_forward(x, w, out=ws.view)
            for epi in (0, NORM, NORM | RELU):
                what = "%s %s H=%d rate=%g epi=%d" % (name, "vec" if vec else "scalar", h, rate, epi)
                out = M.guarded(g.nloc, h, vec)
                g.plan.forward_dropout(x, keep, rate, out=out.view, epilogue=epi)
                M.launches(what, want_launches(g.sched, DROP + SUM, SUM, vec, h), seen)
                out.check_guards(what)
                ref = epilogue_chain(g.d_re, g, ws.view, epi, vec, h, g.row_left, g.row_right, g.col_left)
                assert np.array_equal(bits(out.view), bits(ref)), what
                if h in (1, 5, 41, 129, 300, 1025) or h == max(VEC_WIDTHS):
                    within_fp64(g, out.host(), xh, keep_h, rate, epi, what)
                again = M.guarded(g.nloc, h, vec)
                g.plan.forward_dropout(x, keep, rate, out=again.view, epilogue=epi)
                M.same_bits(out, again, what)
            for epi in (NORM, NORM | NORM_OUT):
                what = "%s %s H=%d rate=%g teleport epi=%d" % (name, "vec" if vec else "scalar", h, rate, epi)
                out = M.guarded(g.nloc, h, vec)
                g.plan.teleport_forward_dropout(x, t, ALPHA, BETA, keep, rate, epilogue=epi, out=out.view)
                M.launches(what, want_launches(g.sched, DROP + TELE, TELE, vec, h), seen)
                s = epilogue_chain(g.d_re, g, ws.view, NORM, vec, h, g.row_left, g.row_right, g.col_left)
                y = M.guarded(g.nloc, h, vec)
                K.scaled_add_fwd(s, t, ALPHA, BETA, out=y.view)
                ref = y.view
                if epi & NORM_OUT:
                    ref = epilogue_chain(g.d_re, g, ref, NORM, vec, h, g.row_left, g.row_right, g.col_left)
                assert np.array_equal(bits(out.view), bits(ref)), what


@pytest.mark.parametrize("name", GRAPHS)
def test_backward_over_the_same_csr(name):
    """the dropped sum over gy with the reverse pairs' bytes, against the weighted sum with reverse-pair weights"""
    g = M.graphs()[name]
    rng = np.random.RandomState(11)
    for vec in (True, False):
        for h in (7, 64, 300):
            gy = M.dev_in(rows(rng, g.n, h), vec)
            for rate in RATES:
                rev = g.plan.attn_keep_mask(rate, KEY, STEP, self_base=g.self_base, row_is_source=True)
                ref = g.plan.weighted_forward(gy, weights(rev, rate))
                ref = epilogue_chain(g.d_re, g, ref, NORM, vec, h, g.row_left, g.row_right, g.col_left)
                got = g.plan.forward_dropout(gy, rev, rate, epilogue=NORM)
                assert np.array_equal(bits(got), bits(ref)), (name, vec, h, rate)


def test_exact_backward_is_the_weighted_transpose():
    """TSUM with dropout over the transposed plan against SgTranspose.backward(gy, w) and the norm"""
    seen = set()
    for name, g in M.xgraphs().items():
        rng = np.random.RandomState(len(name))
        for vec in (True, False):
            for h in (5, 64, 129, 1025) if vec else (1, 33, 257):
                gy = M.dev_in(rows(rng, g.n, h), vec)
                for rate in RATES:
                    keep_t = g.tr.attn_keep_mask(rate, KEY, STEP)
                    w = weights(g.plan.attn_keep_mask(rate, KEY, STEP), rate)
                    ws = g.tr.backward(gy, w)
                    for epi in (0, NORM):
                        what = "%s %s H=%d rate=%g epi=%d" % (name, vec, h, rate, epi)
                        got = M.guarded(g.n, h, vec)
                        g.tr.sum_backward_dropout(gy, keep_t, rate, epilogue=epi, row_end=g.d_re, out=got.view)
                        red, fix = (DROP + TSUM, TSUM) if epi else (DROP + SUM, SUM)
                        M.launches(what, want_launches(g.sched_t, red, fix, vec, h), seen)
                        ref = epilogue_chain(g.d_re, g, ws, epi, vec, h)
                        assert np.array_equal(bits(got.view), bits(ref)), what


def test_dropped_rows_are_never_read():
    """source rows that only dropped edges read hold NaN; the output stays finite and equal to the finite oracle"""
    for name in ("ragged", "carry32", "slice"):
        g = M.graphs()[name]
        rng = np.random.RandomState(2)
        for vec, h in ((True, 64), (False, 33), (True, 1030)):
            rate = 0.9
            keep = g.plan.attn_keep_mask(rate, KEY, STEP, self_base=g.self_base)
            k = keep.cpu().numpy()[:g.E] & 1
            read = np.zeros(g.n, bool)
            read[g.col[k == 1]] = True
            skipped = np.zeros(g.n, bool)
            skipped[g.col] = True
            skipped &= ~read
            assert skipped.sum() > 0, name
            xh = rows(rng, g.n, h)
            want = g.plan.forward_dropout(M.dev_in(xh, vec), keep, rate, epilogue=NORM).cpu().numpy()
            xh[skipped] = np.nan
            got = g.plan.forward_dropout(M.dev_in(xh, vec), keep, rate, epilogue=NORM).cpu().numpy()
            ok = g.deg > 0
            assert np.isfinite(got[ok]).all() and np.array_equal(got.view(np.int32), want.view(np.int32)), name


def test_every_new_instantiation_launched():
    """every (main, 32 + r, VEC, L, NCH) of the three dropped sums at every rung, and nothing else with dropout"""
    g = M.xgraphs()["carry32"]
    rng = np.random.RandomState(9)
    seen = set()
    for vec, vw in ((True, 4), (False, 1)):
        for qc, _, _ in M.RUNGS:
            h = vw * qc
            x = M.dev_in(rows(rng, g.n, h), vec)
            t = M.dev_in(rows(rng, g.n, h), vec)
            keep = g.plan.attn_keep_mask(0.5, KEY, STEP)
            g.plan.forward_dropout(x, keep, 0.5)
            seen |= {(l["kind"], l["red"], l["vec"], l["lanes"], l["nch"]) for l in K.sg_launches()}
            g.plan.teleport_forward_dropout(x, t, ALPHA, BETA, keep, 0.5, epilogue=NORM)
            seen |= {(l["kind"], l["red"], l["vec"], l["lanes"], l["nch"]) for l in K.sg_launches()}
            g.tr.sum_backward_dropout(x, g.tr.attn_keep_mask(0.5, KEY, STEP), 0.5, epilogue=NORM, row_end=g.d_re)
            seen |= {(l["kind"], l["red"], l["vec"], l["lanes"], l["nch"]) for l in K.sg_launches()}
    want = {("main", DROP + r, vw, lanes, nch) for r in (SUM, TSUM, TELE) for vw in (4, 1)
            for _, lanes, nch in M.RUNGS}
    assert {s for s in seen if s[1] >= DROP} == want
    assert all(s[0] == "main" for s in seen if s[1] >= DROP)
    assert {s[1] for s in seen if s[0] != "main"} <= {SUM, TSUM, TELE}


def test_rate_zero_and_no_mask_are_the_plain_calls():
    g = M.xgraphs()["ragged"]
    rng = np.random.RandomState(4)
    for vec, h in ((True, 96), (False, 17)):
        x = M.dev_in(rows(rng, g.n, h), vec)
        t = M.dev_in(rows(rng, g.n, h), vec)
        keep = g.plan.attn_keep_mask(0.5, KEY, STEP)
        plain = g.plan.forward(x, epilogue=NORM)
        want = [(l["kind"], l["red"]) for l in K.sg_launches()]
        for k, rate in ((keep, 0.0), (None, 0.5)):
            got = g.plan.forward_dropout(x, k, rate, epilogue=NORM)
            assert np.array_equal(bits(got), bits(plain)) and [(l["kind"], l["red"]) for l in K.sg_launches()] == want
        tp = g.plan.teleport_forward(x, t, ALPHA, BETA, epilogue=NORM)
        assert np.array_equal(bits(g.plan.teleport_forward_dropout(x, t, ALPHA, BETA, keep, 0.0, epilogue=NORM)),
                              bits(tp))
        bp = g.tr.sum_backward(x, epilogue=NORM, row_end=g.d_re)
        assert np.array_equal(bits(g.tr.sum_backward_dropout(x, None, 0.5, epilogue=NORM, row_end=g.d_re)), bits(bp))


def test_refusals():
    g = M.xgraphs()["tiny"]
    x = M.dev_in(np.ones((g.n, 8), np.float32), True)
    keep = g.plan.attn_keep_mask(0.5, KEY, STEP)
    for rate in (1.0, -0.25, float("nan")):
        for call in (lambda: g.plan.forward_dropout(x, keep, rate),
                     lambda: g.plan.teleport_forward_dropout(x, x, ALPHA, BETA, keep, rate, epilogue=NORM),
                     lambda: g.tr.sum_backward_dropout(x, keep, rate)):
            with pytest.raises(RuntimeError):
                call()
    with pytest.raises(RuntimeError):   # NORM without the graph's row ends
        g.tr.sum_backward_dropout(x, keep, 0.5, epilogue=NORM)


# -------------------------------------------------------------------------------------------------- models ---
BUILDERS = {
    "gcn": lambda m, **kw: build_gcn(m, [24, 16, 12], 0.5, **kw),
    "appnp": lambda m, **kw: build_appnp(m, [24, 16, 12], 0.5, K=10, alpha=0.1, **kw),
}


def train(name, graph, fuse, steps=3, edge_dropout=0.5, infer=False, **kw):
    row_end, col = graph
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    ir = Recorder(m)
    h = BUILDERS[name](ir, edge_dropout=edge_dropout, **kw)
    feats, labels, mask = (t.numpy() for t in datasets.node_data(n, 24, 12, seed=5))
    m.set_labels(h["label"], labels)
    m.set_tensor(h["input"], feats)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    relu_of = {nd["layer"]: nd["out"] for nd in ir.nodes if nd["kind"] == "relu"}
    out = dict(ir=ir, h=h, feats=feats, labels=labels, mask=mask, info=m.op_info(), steps=[], graph=graph)
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
    m.infer_mode(); m.forward()
    out["infer_logits"] = m.get_tensor(h["logits"])
    host.close()
    return out


def check_witness(run):
    for k, st in enumerate(run["steps"]):
        wt = witness(run["ir"], run["graph"], run["feats"], run["labels"], run["mask"], st["w0"], step=k + 1,
                     relu_masks=st["relu"])
        close("step %d logits" % k, st["logits"], wt["logits"])
        for p, (a, b) in enumerate(zip(st["dw"], wt["dW"])):
            close("step %d dW%d" % (k, p), a, b)


def check_identical(a, b, keys=("logits", "dw", "w1")):
    for sa, sb in zip(a["steps"], b["steps"]):
        for k in keys:
            xs, ys = (sa[k], sb[k]) if k != "logits" else ([sa[k]], [sb[k]])
            for x, y in zip(xs, ys):
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), k


def check_fusion(name, run):
    """the GCN block (forward NORM | RELU, backward NORM into the Linear's gradient) and the teleport still fuse"""
    ir, info = run["ir"], run["info"]
    sgs = [nd for nd in ir.nodes if nd["kind"] == "scatter_gather"]
    assert sgs and all(nd["attrs"]["dropout"] == 0.5 for nd in sgs)
    for i, sg in enumerate(sgs):
        e, be = info[sg["layer"]]["epilogue"], info[sg["layer"]]["bwdEpilogue"]
        if name == "gcn":
            assert e == (NORM | RELU if i != len(sgs) - 1 else NORM) and be == NORM, (i, e, be)
        else:
            assert e == (NORM | NORM_OUT if i != len(sgs) - 1 else NORM), (i, e)
            sa = [nd for nd in ir.nodes if nd["kind"] == "scaled_add"][i]
            assert info[sa["layer"]]["fusedInto"] == sg["layer"]


@pytest.mark.parametrize("name", list(BUILDERS))
def test_model_matches_the_witness(name):
    g = sym_graph()
    fused, unfused = train(name, g, True), train(name, g, False)
    check_witness(fused)
    check_identical(fused, unfused)
    check_fusion(name, fused)
    # two identical runs give the same bits
    check_identical(fused, train(name, g, True))
    # and the dropout changes every training step's logits
    plain = train(name, g, True, edge_dropout=0.0)
    assert all(not np.array_equal(a["logits"], b["logits"]) for a, b in zip(fused["steps"], plain["steps"]))


@pytest.mark.parametrize("name", list(BUILDERS))
def test_model_with_exact_backward_on_a_directed_multigraph(name):
    re_, col = directed_graph()
    deg = np.diff(np.concatenate([[0], re_.astype(np.int64)]))
    rows_ = np.split(col, np.cumsum(deg)[:-1])
    rows_ = [np.concatenate([r, r[::7]]) for r in rows_]
    g = (np.cumsum([len(r) for r in rows_]).astype(np.uint64), np.concatenate(rows_).astype(np.uint32))
    fused, unfused = train(name, g, True, exact_backward=True), train(name, g, False, exact_backward=True)
    check_witness(fused)
    check_identical(fused, unfused)


@pytest.mark.parametrize("name", list(BUILDERS))
def test_rate_zero_and_infer_mode_are_todays_model(name):
    """edge_dropout=0 builds today's model (same bits); infer mode runs the plain sums (same logits as a model
    without edge dropout holding the same weights)"""
    g = sym_graph()
    a = train(name, g, True, edge_dropout=0.0)
    row_end, col = g
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    h = BUILDERS[name](m)
    m.set_labels(h["label"], a["labels"])
    m.set_tensor(h["input"], a["feats"])
    m.set_tensor(h["mask"], a["mask"].astype(np.int32))
    for st in a["steps"]:
        m.train_mode(); m.zero_gradients(); m.forward()
        assert np.array_equal(m.get_tensor(h["logits"]).view(np.int32), st["logits"].view(np.int32))
        m.backward(); m.update()
    host.close()
    b = train(name, g, True, edge_dropout=0.5, steps=1)
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    h = BUILDERS[name](m)
    m.set_tensor(h["input"], b["feats"])
    for p, w in enumerate(b["steps"][-1]["w1"]):
        m.set_parameter(p, w)
    m.infer_mode(); m.forward()
    assert np.array_equal(m.get_tensor(h["logits"]).view(np.int32), b["infer_logits"].view(np.int32))
    host.close()


def test_masks_differ_between_hops_and_steps():
    """each hop draws its own mask every step: the witness's masks of the recorded APPNP are all distinct, and they
    are what the product used (the model matches the witness above)"""
    re_, col = sym_graph()
    ir = Recorder(None)
    build_appnp(ir, [24, 16, 12], 0.5, K=10, edge_dropout=0.5)
    keys = [nd["attrs"]["key"] for nd in ir.nodes if nd["kind"] == "scatter_gather"]
    masks = {(k, s): edge_keep(re_, col, 0.5, k, s).tobytes() for k in keys for s in (1, 2, 3)}
    assert len(set(masks.values())) == len(masks) == 30
    # and the device generator is that mask
    d_re, d_col = torch.from_numpy(re_.astype(np.int64)).cuda(), torch.from_numpy(col.astype(np.int32)).cuda()
    plan = K.SgPlan(0, re_.shape[0] - 1, 0, d_re, d_col)
    got = (plan.attn_keep_mask(0.5, keys[3], 2).cpu().numpy()[:col.shape[0]] & 1).astype(bool)
    assert np.array_equal(got, edge_keep(re_, col, 0.5, keys[3], 2))
