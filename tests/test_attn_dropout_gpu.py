"""Attention dropout on the GPU.

Kernels: roc_sg_attn_keep_mask bit-equal to the numpy restatement (attn_dropout_oracle) in all three edge orders, on
every matrix graph (slices with global ids among them), a directed multigraph and their transposes; the dropout
forward and both backwards at every new main-kernel instantiation (fp32 against the fp64 oracle with sg_matrix's bounds,
bf16 byte-equal to fp32 on the widened rows, planned and exact); rate 0 and NULL masks give the calls without dropout
bit for bit; repeats give the same bits; bad arguments give ROC_ERR_INVALID.

Models: build_gat(scores="per_head", activation="elu", attn_dropout=0.6) against a torch fp64 witness whose masks come
from the numpy restatement, for one and for three steps; with the exact backward on a directed graph with duplicate
edges; with bf16 aggregation; infer mode; attn_dropout=0 against no keyword; and the refusals."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import attn_dropout_oracle as ado
import attn_oracle as ao
from conftest import ROOT
from opgraph import Recorder, _relu_with_mask
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_gat
from sg_matrix import (SLOPE, Guarded, close_terms, dev_in, exact, graphs, guarded, no_new_nan, same_bits,
                       valid_heads, wgraphs, xgraphs)
from test_gat_heads_gpu import _bce_train_loss, close, directed_graph, sym_graph
from witness_gat import edge_lists, train_loss

pytestmark = pytest.mark.gpu
RATE, SEED, STEP = 0.6, (5 << 32) | 9, 3
# every row shape of the dropout passes: the rung ends on float4 rows (up to 128 T-columns) and on scalar rows
VEC_H = [16, 32, 64, 128, 256, 512]
SCALAR_H = [4, 8, 16, 32, 64, 128, 256]


def _u8(t):
    return t.cpu().numpy().astype(np.uint8)


# ------------------------------------------------------------------------------------------------ the generator ---
def test_keep_mask_matches_the_restatement_in_every_order():
    for g in graphs().values():
        for rev in (False, True):
            got = _u8(g.plan.attn_keep_mask(RATE, SEED, STEP, self_base=g.self_base, row_is_source=rev))[:g.E]
            want = ado.edge_keep(g.row_end, g.col, RATE, SEED, STEP, g.col_left, g.self_base, row_is_source=rev)
            assert np.array_equal(got, want), (g.name, rev)
    for g in xgraphs().values():                      # whole graphs, the directed multigraph among them
        info = g.tr.info()
        got = _u8(g.tr.attn_keep_mask(RATE, SEED, STEP))[:g.E]
        re_t, col_t = info["row_end"].cpu().numpy().astype(np.uint64), info["col"].cpu().numpy().astype(np.uint32)
        assert np.array_equal(got, ado.edge_keep(re_t, col_t, RATE, SEED, STEP, row_is_source=True)), g.name
        # the same pairs as the forward order, permuted
        fwd = ado.edge_keep(g.row_end, g.col, RATE, SEED, STEP)
        assert np.array_equal(got, fwd[info["perm"].cpu().numpy()]), g.name


def test_keep_mask_refusals():
    g = graphs()["aligned"]
    lib, E = _lib.lib, _lib.ROC_ERR_INVALID
    buf = torch.empty(g.E, dtype=torch.uint8, device="cuda")
    assert lib.roc_sg_attn_keep_mask(None, 0, 0, 0.5, 1, 1, buf.data_ptr(), None) == E
    assert lib.roc_sg_attn_keep_mask(g.plan.handle, 0, 0, 0.5, 1, 1, None, None) == E
    assert lib.roc_sg_attn_keep_mask(g.plan.handle, 0, 2, 0.5, 1, 1, buf.data_ptr(), None) == E
    for rate in (-0.1, 1.0, float("nan")):
        assert lib.roc_sg_attn_keep_mask(g.plan.handle, 0, 0, rate, 1, 1, buf.data_ptr(), None) == E


# ------------------------------------------------------------------------------------------------ the passes ---
def _masks(g, heads, rate=RATE):
    kf = ado.edge_keep(g.row_end, g.col, rate, SEED, STEP, g.col_left, g.self_base)
    kr = ado.edge_keep(g.row_end, g.col, rate, SEED, STEP, g.col_left, g.self_base, row_is_source=True)
    return kf, kr, ado.multipliers(kf, heads, rate), ado.multipliers(kr, heads, rate)


def _dev_u8(a):
    return torch.from_numpy(np.concatenate([a, [0]]).astype(np.uint8)).cuda()


def _fwd(plan, x, sd, keep, rate, heads, h, vec, rows, self_base):
    o, st = guarded(rows, h, vec), Guarded(rows, 2 * heads, 2 * heads + 4, 2 * heads)
    plan.attn_forward_dropout(x, sd, keep, rate, heads, SLOPE, self_base=self_base, out=o.view, stats=st.view)
    return o, st


def _bwd(plan, x, sd, o_all, st_all, gd, keep, keep2, rate, heads, h, vec, rows, self_base):
    ig, sg = guarded(rows, h, vec), Guarded(rows, 2 * heads, 2 * heads + 4, 2 * heads)
    plan.attn_backward_dropout(x, sd, o_all, st_all, gd, keep, keep2, rate, heads, SLOPE, self_base=self_base,
                               in_grad=ig.view, score_grad=sg.view)
    return ig, sg


def _bf16_rows(x, vec):
    """x rounded to bf16 in bf16_padded-style storage, and the widened fp32 rows in the fp32 call's layout."""
    xb = K.bf16_padded(x.shape[0], x.shape[1])
    xb.copy_(torch.from_numpy(x).cuda().bfloat16())
    return xb, dev_in(xb.float().cpu().numpy(), vec)


def run_passes(vec, h):
    for g in graphs().values():
        for heads in valid_heads(h):
            rng = np.random.RandomState(h * 17 + heads + g.nloc)
            x, gy = exact(rng, g.n, h), exact(rng, g.n, h)
            s = rng.randn(g.n, 2 * heads).astype(np.float32)
            xd, gd, sd = dev_in(x, vec), dev_in(gy, vec), dev_in(s, False, ld=2 * heads + 3)
            what = "%s H=%d heads=%d %s" % (g.name, h, heads, "vec" if vec else "scalar")
            kw = dict(self_base=g.self_base, col_left=g.col_left)
            kf, kr, m1, m2 = _masks(g, heads)
            kfd, krd = _dev_u8(kf), _dev_u8(kr)
            fw = [_fwd(g.plan, xd, sd, kfd, RATE, heads, h, vec, g.nloc, g.self_base) for _ in range(2)]
            assert [l["red"] for l in K.sg_launches() if l["kind"] == "main"][-1] == 37
            out, stats = fw[0]
            want, wstats = ado.forward(g.row_end, g.col, x, s, heads, SLOPE, m1, **kw)
            mag = ado.forward(g.row_end, g.col, np.abs(x), s, heads, SLOPE, m1, **kw)[0]
            no_new_nan(out.host(), want, what)
            close_terms(out.host(), want, mag, what + " forward", 0.0)
            assert np.array_equal(stats.bits(), _fwd(g.plan, xd, sd, None, 0.0, heads, h, vec, g.nloc,
                                                     g.self_base)[1].bits()), what + ": stats change with dropout"
            for b in fw:
                b[0].check_guards(what)
            same_bits(fw[0][0], fw[1][0], what)
            # the backward reads out / stats of every id: the forward's own for a whole graph, else the whole graph's
            if g.full is None:
                o_all, st_all, o_np = out.view, stats.view, want
            else:
                f = g.full
                fk = _dev_u8(ado.edge_keep(f.row_end, f.col, RATE, SEED, STEP))
                o_all, st_all = (b.view for b in _fwd(f.plan, xd, sd, fk, RATE, heads, h, vec, f.n, 0))
            bw = [_bwd(g.plan, xd, sd, o_all, st_all, gd, kfd, krd, RATE, heads, h, vec, g.nloc, g.self_base)
                  for _ in range(2)]
            assert [l["red"] for l in K.sg_launches() if l["kind"] == "main"][-2:] == [38, 39]
            ig, sg = bw[0]
            args = (g.row_end, g.col, x, s, o_all.cpu().numpy(), st_all.cpu().numpy())
            wig, wsg = ado.backward(*args, gy, heads, SLOPE, m1, m2, **kw)
            mig = ado.backward(*args, np.abs(gy), heads, SLOPE, m1, m2, **kw)[0]
            msg = ado.backward(*args, gy, heads, SLOPE, m1, m2, magnitude=True, **kw)[1]
            no_new_nan(ig.host(), wig, what)
            close_terms(ig.host(), wig, mig, what + " input gradient", 0.0)
            sgh = sg.host()
            close_terms(sgh[:, :heads], wsg[:, :heads], msg[:, :heads], what + " d s_dst", 1e-6)
            close_terms(sgh[:, heads:], wsg[:, heads:], msg[:, heads:], what + " d s_src", 1e-6)
            for b in bw:
                b[0].check_guards(what)
                b[1].check_guards(what)
            same_bits(bw[0][0], bw[1][0], what)
            same_bits(bw[0][1], bw[1][1], what)
            # bf16 rows: the bytes of the fp32 call on the widened rows
            xb, xw = _bf16_rows(x, vec)
            ob = _fwd(g.plan, xb, sd, kfd, RATE, heads, h, vec, g.nloc, g.self_base)
            assert [l["red"] for l in K.sg_launches() if l["kind"] == "main"][-1] == 53
            same_bits(ob[0], _fwd(g.plan, xw, sd, kfd, RATE, heads, h, vec, g.nloc, g.self_base)[0], what + " bf16")
            bb = _bwd(g.plan, xb, sd, o_all, st_all, gd, kfd, krd, RATE, heads, h, vec, g.nloc, g.self_base)
            assert [l["red"] for l in K.sg_launches() if l["kind"] == "main"][-2:] == [54, 55]
            bw32 = _bwd(g.plan, xw, sd, o_all, st_all, gd, kfd, krd, RATE, heads, h, vec, g.nloc, g.self_base)
            same_bits(bb[0], bw32[0], what + " bf16 input gradient")
            same_bits(bb[1], bw32[1], what + " bf16 score gradient")
            # rate 0 with an all-keep mask, and NULL masks at any rate: the calls without dropout, bit for bit
            ones = torch.full_like(kfd, 255)
            plain = guarded(g.nloc, h, vec), Guarded(g.nloc, 2 * heads, 2 * heads + 4, 2 * heads)
            g.plan.attn_forward(xd, sd, heads, SLOPE, self_base=g.self_base, out=plain[0].view, stats=plain[1].view)
            for keep, rate in ((ones, 0.0), (None, RATE)):
                same_bits(_fwd(g.plan, xd, sd, keep, rate, heads, h, vec, g.nloc, g.self_base)[0], plain[0], what)
            pb = guarded(g.nloc, h, vec), Guarded(g.nloc, 2 * heads, 2 * heads + 4, 2 * heads)
            g.plan.attn_backward(xd, sd, o_all, st_all, gd, heads, SLOPE, self_base=g.self_base, in_grad=pb[0].view,
                                 score_grad=pb[1].view)
            b0 = _bwd(g.plan, xd, sd, o_all, st_all, gd, ones, ones, 0.0, heads, h, vec, g.nloc, g.self_base)
            same_bits(b0[0], pb[0], what)
            same_bits(b0[1], pb[1], what)


@pytest.mark.parametrize("h", VEC_H, ids=str)
def test_passes_vector(h):
    run_passes(True, h)


@pytest.mark.parametrize("h", SCALAR_H, ids=str)
def test_passes_scalar(h):
    run_passes(False, h)


def _exact_ref(g, x, s, o, stats, gy, heads, m1, absolute=False):
    """The true adjoint, per forward edge e = (i <- j): d s_dst[i] and d s_src[j] take dz(i<-j), inGrad[j] takes
    a'(i<-j) G[i].  absolute: the same sums over the terms' magnitudes."""
    re_, deg, r, j, i = ao._edges(g.row_end, g.col, 0, 0)
    n = g.n
    F = x.shape[1] // heads
    if absolute:
        x, gy = np.abs(x), np.abs(gy)
    D = (gy * o).reshape(n, heads, F).sum(-1)
    if absolute:
        D = np.abs(D)
    m, iz = stats[:, :heads], stats[:, heads:]
    z = s[i, :heads] + s[j, heads:]
    a = np.where(iz[i] == 0, 0.0, np.exp(ao._leaky(z, SLOPE) - m[i]) * iz[i])
    l = np.where(z > 0, 1.0, SLOPE)
    dot = ao._per_head_dot(gy, i, x, j, heads)
    dz = a * (m1 * dot + D[i]) * l if absolute else a * (m1 * dot - D[i]) * l
    ig = ao._weighted_gather(j, i, a * m1, n, gy, heads, n)
    return ig, np.concatenate([ao._row_sum(i, dz, n), ao._row_sum(j, dz, n)], axis=1)


@pytest.mark.parametrize("h,vec", [(16, True), (64, True), (256, True), (8, False), (33, False), (128, False)])
def test_exact_backward(h, vec):
    """Over the transposed plan, against the true adjoint on every whole graph (a directed multigraph, a hub, a
    fan-out); on a symmetric graph with increasing sources the transpose is the CSR and the planned call's bits."""
    for g in xgraphs().values():
        for heads in valid_heads(h):
            rng = np.random.RandomState(h + heads + g.n)
            x, gy = exact(rng, g.n, h), exact(rng, g.n, h)
            s = rng.randn(g.n, 2 * heads).astype(np.float32)
            xd, gd, sd = dev_in(x, vec), dev_in(gy, vec), dev_in(s, False, ld=2 * heads + 3)
            what = "%s exact H=%d heads=%d" % (g.name, h, heads)
            kf, _, m1, _ = _masks(g, heads)
            kfd = _dev_u8(kf)
            kt = g.tr.attn_keep_mask(RATE, SEED, STEP)
            o, st = _fwd(g.plan, xd, sd, kfd, RATE, heads, h, vec, g.n, 0)
            res = []
            for _ in range(2):
                ig, sg = guarded(g.n, h, vec), Guarded(g.n, 2 * heads, 2 * heads + 4, 2 * heads)
                g.tr.attn_backward_dropout(g.plan, xd, sd, o.view, st.view, gd, kfd, kt, RATE, heads, SLOPE,
                                           in_grad=ig.view, score_grad=sg.view)
                res.append((ig, sg))
            on, stn = o.host().astype(np.float64), st.host().astype(np.float64)
            wig, wsg = _exact_ref(g, x.astype(np.float64), s.astype(np.float64), on, stn, gy.astype(np.float64),
                                  heads, m1)
            mig, msg = _exact_ref(g, x.astype(np.float64), s.astype(np.float64), on, stn, gy.astype(np.float64),
                                  heads, m1, absolute=True)
            ig, sg = res[0]
            no_new_nan(ig.host(), wig, what)
            close_terms(ig.host(), wig, mig, what + " input gradient", 0.0)
            close_terms(sg.host(), wsg, msg, what + " score gradient", 1e-6)
            same_bits(res[0][0], res[1][0], what)
            same_bits(res[0][1], res[1][1], what)
            xb, xw = _bf16_rows(x, vec)
            b16 = guarded(g.n, h, vec), Guarded(g.n, 2 * heads, 2 * heads + 4, 2 * heads)
            g.tr.attn_backward_dropout(g.plan, xb, sd, o.view, st.view, gd, kfd, kt, RATE, heads, SLOPE,
                                       in_grad=b16[0].view, score_grad=b16[1].view)
            b32 = guarded(g.n, h, vec), Guarded(g.n, 2 * heads, 2 * heads + 4, 2 * heads)
            g.tr.attn_backward_dropout(g.plan, xw, sd, o.view, st.view, gd, kfd, kt, RATE, heads, SLOPE,
                                       in_grad=b32[0].view, score_grad=b32[1].view)
            same_bits(b16[0], b32[0], what + " bf16")
            same_bits(b16[1], b32[1], what + " bf16")


def test_invalid_arguments():
    g = wgraphs()["directed"]
    h, heads = 16, 2
    x = K.padded(g.n, h)
    s = torch.zeros((g.n, 2 * heads), device="cuda")
    keep = torch.full((g.E,), 255, dtype=torch.uint8, device="cuda")
    for rate in (-0.5, 1.0, float("nan")):
        with pytest.raises(_lib.RocError, match="ROC_ERR_INVALID"):
            g.plan.attn_forward_dropout(x, s, keep, rate, heads)
    o, st = g.plan.attn_forward_dropout(x, s, keep, 0.5, heads)
    for k1, k2 in ((keep, None), (None, keep)):
        with pytest.raises(_lib.RocError, match="ROC_ERR_INVALID"):
            g.plan.attn_backward_dropout(x, s, o, st, x, k1, k2, 0.5, heads)
        with pytest.raises(_lib.RocError, match="ROC_ERR_INVALID"):
            g.tr.attn_backward_dropout(g.plan, x, s, o, st, x, k1, k2, 0.5, heads)
    with pytest.raises(_lib.RocError, match="ROC_ERR_INVALID"):
        g.plan.attn_backward_dropout(x, s, o, st, x, keep, keep, 1.0, heads)


# ------------------------------------------------------------------------------------------------- the models ---
def witness(ir, graph, feats, labels, mask, weights, step, relu_masks, loss_fn=train_loss, rounded=None):
    """The recorded GAT graph in torch fp64 with autograd for one training step, as test_gat_heads_gpu.witness, with
    each attention_gather's dropout taken from the numpy restatement of its mask at `step`."""
    row_end, col = np.asarray(graph[0]), np.asarray(graph[1])
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    rounded = rounded or {}
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(True) for w in weights]
    val = {ir.leaves[0]: torch.from_numpy(np.asarray(feats, dtype=np.float64))}
    loss = logits = None
    for nd in ir.nodes:
        k, a, ins, what = nd["kind"], nd["attrs"], nd["ins"], "layer %d (%s)" % (nd["layer"], nd["kind"])
        x = val.get(ins[0])
        if k == "linear":
            y = x @ ws[a["param"]].T
        elif k == "attention_scores":
            hd, w = a["heads"], ws[a["param"]]
            xv = x.reshape(n, hd, -1)
            y = torch.cat([(xv * w[:hd]).sum(2), (xv * w[hd:]).sum(2)], 1)
        elif k == "attention_gather":
            hd, sc = a["heads"], val[ins[1]]
            z = sc[dst, :hd] + sc[src, hd:]
            yv = torch.where(z > 0, z, a["slope"] * z)
            m = torch.full((n, hd), -np.inf, dtype=torch.float64).scatter_reduce(
                0, dst.unsqueeze(1).expand(-1, hd), yv.detach(), "amax", include_self=True)
            ex = torch.exp(yv - m[dst])
            den = torch.zeros((n, hd), dtype=torch.float64).index_add(0, dst, ex)
            al = ex / den[dst]
            if a["dropout"] > 0:
                keep = ado.edge_keep(row_end, col, a["dropout"], a["key"], step)
                al = al * torch.from_numpy(ado.multipliers(keep, hd, a["dropout"]))
            f = x.shape[1] // hd
            msg = (al.unsqueeze(2) * x[src].reshape(-1, hd, f)).reshape(-1, x.shape[1])
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, msg)
        elif k == "relu":
            y = _relu_with_mask(x, relu_masks.get(nd["layer"]), what)
        elif k == "elu":
            y = torch.nn.functional.elu(x)
        elif k == "dropout":
            if a["rate"] > 0:
                from oracle import oracle
                keep = oracle.dropout_mask(0, n, x.shape[1], a["rate"], a["key"], step)
                scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(a["rate"])))
                y = x * torch.from_numpy(keep.astype(np.float64) * scale)
            else:
                y = x
        elif k in ("softmax_cross_entropy", "sigmoid_cross_entropy"):
            loss, logits = loss_fn(x, np.asarray(labels), np.asarray(mask)), x
            continue
        else:
            raise AssertionError("op not in these models: " + k)
        if nd["out"] in rounded:
            r, p = torch.from_numpy(np.asarray(rounded[nd["out"]], dtype=np.float64)), y.detach()
            assert ((r - p).abs() <= 2.0 ** -8 * 1.001 * p.abs() + 1e-5 * p.abs().max()).all(), what
            y = y + (r - p)
        val[nd["out"]] = y
    loss.backward()
    return logits.detach().numpy(), [w.grad.numpy() if w.grad is not None else np.zeros(w.shape) for w in ws]


LAYERS, HEADS = [24, 16, 32, 12], [2, 8]
PAPER = dict(scores="per_head", activation="elu")


def train(graph, steps=3, fuse=True, infer=False, **kw):
    row_end, col = graph
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    ir = Recorder(m)
    h = build_gat(ir, LAYERS, 0.5, heads=HEADS, **kw)
    feats, labels, mask = (t.numpy() for t in datasets.node_data(n, LAYERS[0], LAYERS[-1], seed=5))
    m.set_labels(h["label"], labels)
    m.set_tensor(h["input"], feats)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    relu_of = {nd["layer"]: nd["out"] for nd in ir.nodes if nd["kind"] == "relu"}
    out = dict(ir=ir, h=h, feats=feats, labels=labels, mask=mask, steps=[], graph=graph)
    dtypes = {t: m.tensor_dtype(t) for t in ir.width}
    bf16 = [t for t in h["attn_ins"] if dtypes[t] == "bfloat16"]
    for _ in range(steps):
        st = dict(w0=[m.get_parameter(p) for p in range(m.num_parameters())])
        m.train_mode(); m.zero_gradients(); m.forward()
        st["logits"] = m.get_tensor(h["logits"])
        st["relu"] = {l: m.get_tensor(t) > 0 for l, t in relu_of.items()}
        st["rounded"] = {t: m.get_tensor(t) for t in bf16}
        m.backward()
        st["dw"] = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
        st["w1"] = [m.get_parameter(p) for p in range(m.num_parameters())]
        out["steps"].append(st)
    if infer:
        m.infer_mode(); m.forward()
        out["infer"] = m.get_tensor(h["logits"])
    host.close()
    return out


def check_witness(run):
    for k, st in enumerate(run["steps"]):
        logits, dw = witness(run["ir"], run["graph"], run["feats"], run["labels"], run["mask"], st["w0"], k + 1,
                             st["relu"], rounded=st["rounded"])
        close("step %d logits" % k, st["logits"], logits)
        for p, (a, b) in enumerate(zip(st["dw"], dw)):
            close("step %d dW%d" % (k, p), a, b)


def identical(a, b):
    for sa, sb in zip(a["steps"], b["steps"]):
        for key in ("logits", "dw", "w1"):
            xs, ys = (sa[key], sb[key]) if key != "logits" else ([sa[key]], [sb[key]])
            for x, y in zip(xs, ys):
                if not np.array_equal(np.asarray(x).view(np.int32), np.asarray(y).view(np.int32)):
                    return False
    return True


def test_paper_gat_one_step_matches_the_witness():
    check_witness(train(sym_graph(), steps=1, attn_dropout=RATE, **PAPER))


def test_paper_gat_three_steps_match_the_witness_with_new_masks():
    run = train(sym_graph(), steps=3, attn_dropout=RATE, **PAPER)
    check_witness(run)
    g = sym_graph()
    assert not np.array_equal(ado.edge_keep(*g, RATE, 2, 1), ado.edge_keep(*g, RATE, 2, 2))
    unfused = train(sym_graph(), steps=3, fuse=False, attn_dropout=RATE, **PAPER)
    assert identical(run, unfused)


def test_paper_gat_with_exact_backward_on_a_directed_multigraph():
    g = directed_graph()
    dst = np.repeat(np.arange(g[0].shape[0]), np.diff(np.concatenate([[0], g[0].astype(np.int64)])))
    pairs = dst * g[0].shape[0] + g[1]
    if np.unique(pairs).shape[0] == pairs.shape[0]:           # give it duplicate edges
        re_, col = g
        col = col.copy()
        starts = np.concatenate([[0], re_[:-1].astype(np.int64)])
        multi = np.nonzero(np.diff(np.concatenate([starts, [col.shape[0]]])) >= 2)[0][:50]
        for r in multi:
            col[starts[r] + 1] = col[starts[r]]
        g = (re_, col)
    check_witness(train(g, exact_backward=True, attn_dropout=RATE, **PAPER))


def test_paper_gat_with_bf16_aggregation():
    run = train(sym_graph(), aggregation="bfloat16", attn_dropout=RATE, **PAPER)
    check_witness(run)


def test_infer_mode_is_the_rate_zero_model():
    a = train(sym_graph(), steps=1, infer=True, attn_dropout=RATE, **PAPER)
    b = train(sym_graph(), steps=1, infer=True, **PAPER)
    # the same weights after the step would need the same masks; infer on the weights each model reached is checked
    # against a model of rate 0 given those weights
    host = Host(0, 0, 1)
    host.graph_from_arrays(*sym_graph())
    m = Model(host, seed=1)
    h = build_gat(m, LAYERS, 0.5, heads=HEADS, **PAPER)
    for p, w in enumerate(a["steps"][-1]["w1"]):
        m.set_parameter(p, w)
    m.set_tensor(h["input"], a["feats"])
    m.infer_mode(); m.forward()
    assert np.array_equal(m.get_tensor(h["logits"]).view(np.int32), a["infer"].view(np.int32))
    host.close()
    assert b["infer"].shape == a["infer"].shape


def test_rate_zero_is_the_model_without_the_keyword():
    a = train(sym_graph(), steps=2, attn_dropout=0.0, **PAPER)
    b = train(sym_graph(), steps=2, **PAPER)
    assert identical(a, b)


def run_prog(lines):
    prog = "\n".join(["import numpy as np", "from roc_b200 import _lib", "from roc_b200.model import Host, Model"] +
                     lines + ["host.synchronize()", "print('NO REFUSAL')"])
    return subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True, timeout=300, cwd=ROOT,
                          env=dict(os.environ))


@pytest.mark.parametrize("rate", ["1.0", "-0.25", "float('nan')"])
def test_host_refuses_a_rate_outside_the_unit_interval(rate):
    p = run_prog(["host = Host(0, 0, 1)",
                  "host.graph_from_arrays(np.arange(1, 101, dtype=np.uint64), np.arange(100, dtype=np.uint32))",
                  "m = Model(host, seed=1)",
                  "x = m.create_node_tensor(8); s = m.create_node_tensor(4)",
                  "_lib.lib.roc_host_attention_gather_dropout(m.h, x, s, 2, 0.2, %s, 0)" % rate])
    assert p.returncode != 0 and "NO REFUSAL" not in p.stdout
    assert "attention_gather: the dropout rate must be in [0, 1)" in p.stderr, p.stderr[-2000:]


def test_more_than_one_partition_is_refused():
    p = run_prog(["host = Host(0, 0, 2)",
                  "host.graph_from_arrays(np.arange(1, 101, dtype=np.uint64), np.arange(100, dtype=np.uint32))",
                  "m = Model(host, seed=1)",
                  "x = m.create_node_tensor(8); s = m.create_node_tensor(4)",
                  "m.attention_gather(x, s, 2, 0.2, dropout=0.5)"])
    assert p.returncode != 0 and "NO REFUSAL" not in p.stdout
    assert "one partition only" in p.stderr, p.stderr[-2000:]
