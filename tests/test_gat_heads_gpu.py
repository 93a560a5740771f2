"""Per-head GAT scores and ELU on the GPU.

Kernels: roc_attn_scores_fwd / _bwd (and their _bf16 forms) against the fp64 references of tests/test_gat_heads_cpu.py
over rows x (heads, F) with dense and NaN-padded pitches, accumulation on and off, dX == NULL, byte-identical repeats,
the bf16 forms byte-equal to the fp32 call on the widened rows, and the error codes; ELU forward and backward over the
same widths with +-0, +-inf, NaN, subnormals and x < -20.

Models: build_gat(scores="per_head", activation="elu") over three Adam steps against an fp64 autograd interpreter of
the recorded op graph (witness below), fused and unfused byte-identical; the heads = 1 cross-check against the dense
score Linear; each option alone; composition with the exact backward, bf16 features, bf16 aggregation, the sigmoid
loss and batch_norm; and the refusals.

Bounds, U = 2^-24:
  S:   |s - s64| <= gamma_F sum_f |a x|, gamma_F = F U / (1 - F U)       (F fmas in order)
  dX:  |dx - dx64| <= 3 U (|gd ad| + |gs as|)  [+ 2 U (|old| + |dx64|) accumulating]
  dA:  |da - da64| <= 2 U sum_v |g x|                                     (fp64 sums, one rounding)
  ELU: |y - y64| <= 2 U |y64| + 2^-149 (CUDA's expm1f: 1 ulp); the backward, from the product's y,
       |dx - dx64| <= 4 U |g| (|y| + 1), absolute because y + 1 cancels for very negative x."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from opgraph import Recorder, _relu_with_mask
from oracle import oracle
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_gat
from test_gat_heads_cpu import elu_bwd_ref, elu_ref, scores_bwd_ref, scores_ref
from witness_gat import attend, edge_lists, train_loss

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
K_DX = 3
K_DA = 2
ROWS = [1, 2, 1000, 65537, 4194304]
# (2, 1), (3, 1), (6, 1) and (7, 1): F < H % 4, so a row's last column group spans several heads and padding
SHAPES = [(1, 1), (1, 3), (1, 41), (1, 64), (2, 4), (3, 5), (4, 16), (8, 8), (8, 32), (8, 64), (1, 602), (2, 1), (3, 1),
          (6, 1), (7, 1)]


# ------------------------------------------------------------------------------------------------- the kernels ---
def _nan_rows(v, ld):
    """v [rows][h] copied into a NaN-filled [rows][ld] buffer; returns the [rows][h] view"""
    rows, h = v.shape
    buf = torch.full((rows, ld), float("nan"), device=v.device, dtype=v.dtype)
    buf[:, :h] = v
    return buf[:, :h]


def _bits(t):
    """every element of t's storage window, padding included, as integer bits"""
    rows, h = t.shape
    full = torch.as_strided(t, (rows, t.stride(0)), (t.stride(0), 1))
    return full.view(torch.int32 if t.element_size() == 4 else torch.int16)


def _pad_untouched(t):
    rows, h = t.shape
    full = torch.as_strided(t, (rows, t.stride(0)), (t.stride(0), 1))
    return bool(torch.isnan(full[:, h:]).all()) if full.shape[1] > h else True


def _chunks(rows, h):
    step = max(1, (1 << 24) // max(h, 1))
    return [(r, min(r + step, rows)) for r in range(0, rows, step)]


def _worst(got, want, bound):
    return float(((got.double() - want).abs() / (bound + 1e-300)).max()) if want.numel() else 0.0


def _check_scores(rows, heads, f, padded, seed):
    h = heads * f
    what = "rows=%d heads=%d F=%d padded=%s" % (rows, heads, f, padded)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    ldx = (h + 3) // 4 * 4 + 4 if padded else h
    lds = (2 * heads + 3) // 4 * 4 + 4 if padded else 2 * heads
    x = _nan_rows(torch.randn((rows, h), generator=gen, device="cuda"), ldx)
    a = torch.randn((2 * heads, f), generator=gen, device="cuda") / math.sqrt(f)
    ds = _nan_rows(torch.randn((rows, 2 * heads), generator=gen, device="cuda"), lds)
    s = K.attn_scores_fwd(x, a, heads, out=_nan_rows(torch.zeros((rows, 2 * heads), device="cuda"), lds))
    assert _pad_untouched(s), what
    gamma = f * U / (1 - f * U)
    for r0, r1 in _chunks(rows, h):
        want, b = scores_ref(x[r0:r1], a, heads)
        assert _worst(s[r0:r1], want, gamma * b) <= 1.0, what
    s2 = K.attn_scores_fwd(x, a, heads, out=_nan_rows(torch.zeros((rows, 2 * heads), device="cuda"), lds))
    assert torch.equal(_bits(s), _bits(s2)), what
    # backward: overwrite and accumulate
    base = torch.randn((rows, h), generator=gen, device="cuda")
    da_want = torch.zeros((2 * heads, f), device="cuda", dtype=torch.float64)
    da_abs = torch.zeros_like(da_want)
    dxs = {}
    for acc in (False, True):
        dx = _nan_rows(base.clone() if acc else torch.zeros_like(base), ldx)
        dx, da = K.attn_scores_bwd(x, a, ds, heads, dx=dx, accumulate=acc)
        assert _pad_untouched(dx), what
        dxs[acc] = (dx, da)
    for r0, r1 in _chunks(rows, h):
        ref = scores_bwd_ref(x[r0:r1], a, ds[r0:r1], heads)
        da_want += ref["da"]
        da_abs += ref["da_abs"]
        bound = K_DX * U * ref["dx_abs"]
        assert _worst(dxs[False][0][r0:r1], ref["dx"], bound) <= 1.0, (what, "dx")
        old = base[r0:r1].double()
        bound_acc = bound + 2 * U * (old.abs() + ref["dx"].abs())
        assert _worst(dxs[True][0][r0:r1], old + ref["dx"], bound_acc) <= 1.0, (what, "dx accumulate")
    for acc in (False, True):
        assert _worst(dxs[acc][1], da_want, K_DA * U * da_abs) <= 1.0, (what, "da")
    assert torch.equal(dxs[False][1].view(torch.int32), dxs[True][1].view(torch.int32)), what
    # dX == NULL: dA alone, the same bytes; a repeat: the same bytes everywhere
    _, da_only = K.attn_scores_bwd(x, a, ds, heads, need_dx=False)
    assert torch.equal(da_only.view(torch.int32), dxs[False][1].view(torch.int32)), what
    dx2, da2 = K.attn_scores_bwd(x, a, ds, heads, dx=_nan_rows(torch.zeros_like(base), ldx))
    assert torch.equal(_bits(dx2), _bits(dxs[False][0])) and torch.equal(da2.view(torch.int32),
                                                                          dxs[False][1].view(torch.int32)), what
    del dxs, dx2, base
    # bf16 rows: the bytes of the fp32 call on the widened rows
    ldb = (h + 7) // 8 * 8 + 8 if padded else h
    xb = _nan_rows(x.bfloat16(), ldb)
    xw = _nan_rows(xb.float(), ldx)
    sb = K.attn_scores_fwd_bf16(xb, a, heads, out=_nan_rows(torch.zeros((rows, 2 * heads), device="cuda"), lds))
    sw = K.attn_scores_fwd(xw, a, heads, out=_nan_rows(torch.zeros((rows, 2 * heads), device="cuda"), lds))
    assert torch.equal(_bits(sb), _bits(sw)), what
    dxb, dab = K.attn_scores_bwd_bf16(xb, a, ds, heads, dx=_nan_rows(torch.zeros((rows, h), device="cuda"), ldx))
    dxw, daw = K.attn_scores_bwd(xw, a, ds, heads, dx=_nan_rows(torch.zeros((rows, h), device="cuda"), ldx))
    assert torch.equal(_bits(dxb), _bits(dxw)) and torch.equal(dab.view(torch.int32), daw.view(torch.int32)), what


@pytest.mark.parametrize("heads,f", SHAPES)
@pytest.mark.parametrize("rows", ROWS)
def test_scores_kernel_matches_fp64(rows, heads, f):
    for padded in (False, True):
        _check_scores(rows, heads, f, padded, seed=rows * 31 + heads * 7 + f + padded)
    torch.cuda.empty_cache()


def test_scores_kernel_error_codes():
    rows, heads, f = 8, 2, 4
    h = heads * f
    x, s = K.padded(rows, h), K.padded(rows, 2 * heads)
    a = torch.zeros((2 * heads, f), device="cuda")
    ws_bytes = _lib.lib.roc_attn_scores_workspace_bytes(rows, h, heads)
    ws = torch.empty(ws_bytes + 16, device="cuda", dtype=torch.uint8)
    p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    ok = dict(rows=rows, h=h, heads=heads, x=x, ldx=8, a=a, s=s, lds=4, dx=x, lddx=8, da=a, ws=ws, wsb=ws_bytes)

    def fwd(**kw):
        c = dict(ok, **kw)
        rc = _lib.lib.roc_attn_scores_fwd(c["rows"], c["h"], c["heads"], p(c["x"]), c["ldx"], p(c["a"]), p(c["s"]),
                                          c["lds"], None)
        torch.cuda.synchronize()
        return rc

    def bwd(**kw):
        c = dict(ok, **kw)
        rc = _lib.lib.roc_attn_scores_bwd(c["rows"], c["h"], c["heads"], p(c["x"]), c["ldx"], p(c["a"]), p(c["s"]),
                                          c["lds"], p(c["dx"]), c["lddx"], 0, p(c["da"]), p(c["ws"]), c["wsb"], None)
        torch.cuda.synchronize()
        return rc

    assert fwd() == _lib.ROC_OK and bwd() == _lib.ROC_OK and bwd(dx=None, lddx=0) == _lib.ROC_OK
    for bad in (dict(x=None), dict(a=None), dict(s=None), dict(rows=-1), dict(h=0), dict(heads=0), dict(heads=-2),
                dict(ldx=7), dict(lds=3)):
        assert fwd(**bad) == _lib.ROC_ERR_INVALID, bad
    for bad in (dict(x=None), dict(a=None), dict(s=None), dict(da=None), dict(ws=None), dict(heads=0), dict(ldx=7),
                dict(lds=3), dict(lddx=7), dict(wsb=ws_bytes - 1)):
        assert bwd(**bad) == _lib.ROC_ERR_INVALID, bad
    assert bwd(ws=ws[8:]) == _lib.ROC_ERR_INVALID                     # a misaligned workspace
    for bad in (dict(heads=3, lds=8), dict(h=1028, ldx=1028, lddx=1028)):
        assert fwd(**bad) == _lib.ROC_ERR_UNSUPPORTED, bad
        assert bwd(**bad) == _lib.ROC_ERR_UNSUPPORTED, bad


def _elu_inputs(rows, h, gen):
    x = torch.randn((rows, h), generator=gen, device="cuda") * 4
    specials = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-40, -1e-40, -3e-39, -20.5, -30.0,
                             -88.0, -104.0, 1e-30, -1e-30, 3e38, -3e38], device="cuda")
    flat = x.view(-1)
    k = min(flat.numel(), specials.numel() * 8)
    flat[:k] = specials.repeat(8)[:k]
    return x


@pytest.mark.parametrize("h", sorted({hd * f for hd, f in SHAPES}))
@pytest.mark.parametrize("rows", [1, 1000, 65537])
def test_elu_kernel_matches_fp64(rows, h):
    _check_elu(rows, h, rows * 3 + h)


def test_elu_kernel_at_production_rows():
    _check_elu(4194304, 64, 5)


def _check_elu(rows, h, seed):
    what = "rows=%d H=%d" % (rows, h)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    for ld in (h, (h + 3) // 4 * 4 + 4):
        x = _nan_rows(_elu_inputs(rows, h, gen), ld)
        y = K.activation_fwd(x, _lib.AC_MODE_ELU)
        want = elu_ref(x)
        assert torch.equal(torch.isnan(y), torch.isnan(want)), what
        inf = torch.isinf(want)
        assert torch.equal(y[inf].double(), want[inf]), what
        fin = torch.isfinite(want)
        err = (y.double() - want).abs()[fin]
        assert bool((err <= 2 * U * want.abs()[fin] + 2.0 ** -149).all()), (what, float(err.max()))
        zero = x == 0
        assert torch.equal(torch.signbit(y[zero]), torch.signbit(x[zero])), what      # +-0 keep their sign
        g = torch.randn((rows, h), generator=gen, device="cuda")
        yd = elu_ref(x)                                                                 # exact derivative's y
        for acc in (False, True):
            base = torch.randn((rows, h), generator=gen, device="cuda") if acc else None
            dx = K.activation_bwd(y, g, _lib.AC_MODE_ELU, dx=base.clone() if acc else None)
            ref = elu_bwd_ref(yd, g) + (base.double() if acc else 0)
            assert torch.equal(torch.isnan(dx), torch.isnan(ref)), what
            ok = ~torch.isnan(ref)
            bound = 4 * U * g.double().abs() * (yd.abs().nan_to_num(posinf=0) + 1)
            if acc:
                bound = bound + 2 * U * (base.double().abs() + ref.abs())
            assert bool(((dx.double() - ref).abs()[ok] <= bound[ok]).all()), (what, acc)
    # the bf16-output forms stay relu only
    xb = K.padded(4, 8)
    assert _lib.lib.roc_activation_fwd_y_bf16(4, 8, _lib.AC_MODE_ELU, xb.data_ptr(), 8, K.bf16_padded(4, 8).data_ptr(),
                                              8, None) == _lib.ROC_ERR_UNSUPPORTED


# ------------------------------------------------------------------------------------------------- the models ---
def witness(ir, graph, feats, labels, mask, weights, step=1, relu_masks=None, loss_fn=train_loss, rounded=None):
    """The recorded GAT graph in torch fp64 with autograd for one training step: dropout (the product's Philox masks
    of `step`), linear, attention_scores, attention_gather, relu (the product's masks where fp32 and fp64 tie), elu,
    batch_norm on the batch statistics, and the loss.  rounded: {tensor: the product's bf16 values}, taken in the
    forward with the gradient passed straight through.  Returns logits and dW."""
    row_end, col = np.asarray(graph[0]), np.asarray(graph[1])
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    relu_masks, rounded = relu_masks or {}, rounded or {}
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
            y = attend(x, val[ins[1]], dst, src, n, a["heads"], a["slope"])
        elif k == "relu":
            y = _relu_with_mask(x, relu_masks.get(nd["layer"]), what)
        elif k == "elu":
            y = torch.nn.functional.elu(x)
        elif k == "batch_norm":
            y = torch.nn.functional.batch_norm(x, None, None, ws[a["gamma"]][0], ws[a["beta"]][0], training=True,
                                               eps=a["eps"])
        elif k == "dropout":
            if a["rate"] > 0:
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
            assert ((r - p).abs() <= 2.0 ** -8 * 1.001 * p.abs() + 1e-5 * p.abs().max()).all(), \
                "%s: the product's bf16 value is not a rounding of the fp64 one" % what
            y = y + (r - p)
        val[nd["out"]] = y
    loss.backward()
    return logits.detach().numpy(), [w.grad.numpy() if w.grad is not None else np.zeros(w.shape) for w in ws]


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


CONFIGS = {   # layers, heads
    "heads1": ([24, 16, 12], 1),
    "heads4": ([24, 16, 12], 4),
    "heads2_8": ([24, 16, 32, 12], [2, 8]),
}


def train(config, graph, fuse, steps=3, loss="softmax", **kw):
    layers, heads = CONFIGS[config]
    row_end, col = graph
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    ir = Recorder(m)
    h = build_gat(ir, layers, 0.5, heads=heads, loss=loss, **kw)
    if loss == "sigmoid":
        feats, labels, mask = (t.numpy() for t in datasets.multilabel_node_data(n, layers[0], layers[-1], seed=5))
        m.set_multilabels(h["label"], labels)
    else:
        feats, labels, mask = (t.numpy() for t in datasets.node_data(n, layers[0], layers[-1], seed=5))
        m.set_labels(h["label"], labels)
    m.set_tensor(h["input"], feats)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    relu_of = {nd["layer"]: nd["out"] for nd in ir.nodes if nd["kind"] == "relu"}
    out = dict(ir=ir, h=h, feats=feats, labels=labels, mask=mask, info=m.op_info(), steps=[], graph=graph, loss=loss)
    out["dtypes"] = {t: m.tensor_dtype(t) for t in ir.width}
    bf16 = [t for t in h["attn_ins"] if out["dtypes"][t] == "bfloat16"]
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
    host.close()
    return out


def close(name, got, want, rtol=2e-4, atol_scale=2e-5):
    """test_opgraph_gpu.py's bar; a dW row that vanishes in fp64 (a head's a_dst when each row's edges all sit on one
    side of the LeakyReLU: the softmax ignores a common shift) holds only rounding of cancelling terms and is held to
    1e-4 of the matrix's largest entry"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    scale = np.abs(want).max() if want.size else 0.0
    bound = rtol * np.abs(want) + atol_scale * scale + 1e-30
    if want.ndim == 2 and want.size:
        bound[np.abs(want).max(axis=1) <= 1e-12 * scale] = 1e-4 * scale + 1e-30
    r = float((np.abs(got - want) / bound).max()) if want.size else 0.0
    assert r <= 1.0, (name, r)


def check_witness(run, feats=None):
    ir = run["ir"]
    feats = run["feats"] if feats is None else feats
    loss_fn = _bce_train_loss if run["loss"] == "sigmoid" else train_loss
    for k, st in enumerate(run["steps"]):
        logits, dw = witness(ir, run["graph"], feats, run["labels"], run["mask"], st["w0"], step=k + 1,
                             relu_masks=st["relu"], loss_fn=loss_fn, rounded=st["rounded"])
        close("step %d logits" % k, st["logits"], logits)
        for p, (a, b) in enumerate(zip(st["dw"], dw)):
            close("step %d dW%d" % (k, p), a, b)
    assert [i["kind"] for i in run["info"]] == [nd["kind"] for nd in ir.nodes]


def check_identical(a, b):
    for sa, sb in zip(a["steps"], b["steps"]):
        assert np.array_equal(sa["logits"].view(np.int32), sb["logits"].view(np.int32))
        for k in ("dw", "w1"):
            for x, y in zip(sa[k], sb[k]):
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), k


PAPER = dict(scores="per_head", activation="elu")


@pytest.mark.parametrize("config", list(CONFIGS))
def test_paper_gat_matches_the_witness(config):
    g = sym_graph()
    fused, unfused = train(config, g, True, **PAPER), train(config, g, False, **PAPER)
    check_witness(fused)
    check_identical(fused, unfused)
    # the ELU is never fused, and each A has the shape (2 * heads, F)
    ir = fused["ir"]
    for nd in ir.nodes:
        if nd["kind"] == "elu":
            assert fused["info"][nd["layer"]]["fusedInto"] == -1
        if nd["kind"] == "attention_scores":
            hd = nd["attrs"]["heads"]
            assert fused["steps"][0]["w0"][nd["attrs"]["param"]].shape == (2 * hd, ir.width[nd["ins"][0]] // hd)


@pytest.mark.parametrize("kw", [dict(scores="per_head"), dict(activation="elu")])
def test_each_option_alone_matches_the_witness(kw):
    run = train("heads4", sym_graph(), True, **kw)
    check_witness(run)


def test_per_head_scores_equal_the_dense_linear_at_one_head():
    """With one head, attention_scores is the score Linear F -> 2: A is drawn as that Linear's W (the same values, in
    creation order), and one step gives the same logits and dW to fp32 rounding."""
    g = sym_graph()
    dense = train("heads1", g, True, steps=1, activation="elu")
    per = train("heads1", g, True, steps=1, **PAPER)
    for a, b in zip(dense["steps"][0]["w0"], per["steps"][0]["w0"]):
        assert np.array_equal(a, b)
    close("logits", per["steps"][0]["logits"], dense["steps"][0]["logits"])
    for p, (a, b) in enumerate(zip(per["steps"][0]["dw"], dense["steps"][0]["dw"])):
        close("dW%d" % p, a, b)


def test_paper_gat_with_exact_backward_on_a_directed_graph():
    g = directed_graph()
    fused = train("heads4", g, True, exact_backward=True, **PAPER)
    unfused = train("heads4", g, False, exact_backward=True, **PAPER)
    check_witness(fused)
    check_identical(fused, unfused)


def test_paper_gat_with_bf16_features():
    run = train("heads4", sym_graph(), True, features="bfloat16", **PAPER)
    assert run["dtypes"][run["h"]["input"]] == "bfloat16"
    check_witness(run, feats=torch.from_numpy(run["feats"]).bfloat16().float().numpy())


@pytest.mark.parametrize("config", ["heads1", "heads2_8"])
def test_paper_gat_with_bf16_aggregation(config):
    """wh, read by the attention_gather and the attention_scores, is stored in bf16; the witness takes the product's
    rounded wh with a straight-through gradient"""
    a = train(config, sym_graph(), True, aggregation="bfloat16", **PAPER)
    for wh in a["h"]["attn_ins"]:
        assert a["dtypes"][wh] == "bfloat16"
    for t in a["h"]["scores"] + a["h"]["relu_outs"]:
        assert a["dtypes"][t] == "float32"
    check_witness(a)
    check_identical(a, train(config, sym_graph(), False, aggregation="bfloat16", **PAPER))


def test_paper_gat_with_sigmoid_loss():
    check_witness(train("heads4", sym_graph(), True, loss="sigmoid", **PAPER))


def test_paper_gat_with_batch_norm():
    g = sym_graph()
    fused, unfused = train("heads2_8", g, True, norm="batch", **PAPER), train("heads2_8", g, False, norm="batch", **PAPER)
    check_witness(fused)
    check_identical(fused, unfused)


REFUSALS = {
    "bf16_leaf": ("x = m.create_node_tensor(8, dtype='bfloat16'); y = m.create_node_tensor(4);"
                  " mk = m.create_node_tensor(1, True); m.softmax_cross_entropy(m.attention_scores(x, 2), y, mk);"
                  " m.adam(); m.init()", "attention_scores cannot read a bf16 tensor"),
    "heads": ("x = m.create_node_tensor(8); m.attention_scores(x, 3)",
              "attention_scores: the input width must be heads * F"),
    "linear_elu": ("x = m.create_node_tensor(8); m.linear(x, 4, 3)", "linear: a Linear cannot apply AC_MODE_ELU"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_refusals(name):
    body, message = REFUSALS[name]
    prog = "\n".join([
        "import numpy as np",
        "from roc_b200.model import Host, Model",
        "host = Host(0, 0, 1)",
        "host.graph_from_arrays(np.arange(1, 101, dtype=np.uint64), np.arange(100, dtype=np.uint32))",
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
