"""Attention ScatterGather on the GPU: the kernels against the fp64 oracle (tests/attn_oracle.py) at every width
class and head layout, on the vector and scalar paths, bitwise reproducible; and GAT through the Model API against
an independent torch fp64 autograd witness."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import attn_oracle as ao
from conftest import ROOT, rel_close
from oracle import oracle
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_gat
from sg_graphs import graph, to_dev
from sg_matrix import close_terms, valid_heads
import witness_gat as wg
from witness_gat import gat_witness

pytestmark = pytest.mark.gpu
DEV = "cuda"
SLOPE = 0.2


def bits(t):
    return t.contiguous().cpu().view(torch.int32).numpy()


def feature_buf(rows, h, vec):
    """A [rows][h] feature view: ld = round_up(h, 4) (the vector path), or ld = h + 1 with h + 1 not a multiple of 4,
    so that no feature row is 16-byte aligned past row 0 and the kernels must take the scalar path."""
    if vec:
        return K.padded(rows, h, DEV)
    ld = h + 1 if (h + 1) % 4 else h + 2
    return torch.zeros((rows, ld), device=DEV)[:, :h]


def dev(a, vec):
    t = feature_buf(a.shape[0], a.shape[1], vec)
    t.copy_(torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)))
    assert (t.stride(0) % 4 == 0) == vec
    return t


def check(plan, row_end, col, x, s, g, heads, vec, what, self_base=0, col_left=0, full=None, eps_a=0.0):
    """Forward and backward against the oracle; the oracle's backward takes the kernel's own out and stats, so both
    sides compute the same function of the same inputs.  eps_a: the relative error the inputs' fp32 rounding leaves
    in each a (0 at ordinary score magnitudes).  Returns the device results."""
    xd, gd = dev(x, vec), dev(g, vec)
    sd = torch.from_numpy(np.ascontiguousarray(s, dtype=np.float32)).to(DEV)
    nloc = row_end.shape[0]
    out, stats = plan.attn_forward(xd, sd, heads, SLOPE, self_base=self_base, out=feature_buf(nloc, x.shape[1], vec))
    want, wstats = ao.forward(row_end, col, x, s, heads, SLOPE, self_base=self_base, col_left=col_left)
    mag = ao.forward(row_end, col, np.abs(x), s, heads, SLOPE, self_base=self_base, col_left=col_left)[0]
    close_terms(out.cpu().numpy(), want, mag, "%s forward" % what, eps_a)
    rel_close(stats.cpu().numpy(), wstats, rtol=1e-4 + eps_a, what="%s stats" % what)
    if full is None:
        o_all, st_all = out, stats
    else:
        o_all, st_all = full
    ig, sg = plan.attn_backward(xd, sd, o_all, st_all, gd, heads, SLOPE, self_base=self_base,
                                in_grad=feature_buf(nloc, x.shape[1], vec))
    args = (row_end, col, x, s, o_all.cpu().numpy(), st_all.cpu().numpy())
    kw = dict(self_base=self_base, col_left=col_left)
    wig, wsg = ao.backward(*args, g, heads, SLOPE, **kw)
    mig = ao.backward(*args, np.abs(g), heads, SLOPE, **kw)[0]
    msg = ao.score_grad_magnitude(*args, g, heads, SLOPE, **kw)
    close_terms(ig.cpu().numpy(), wig, mig, "%s input gradient" % what, eps_a)
    sgh = sg.cpu().numpy()
    close_terms(sgh[:, :heads], wsg[:, :heads], msg[:, :heads], "%s d s_dst" % what, 1e-6 + eps_a)
    close_terms(sgh[:, heads:], wsg[:, heads:], msg[:, heads:], "%s d s_src" % what, 1e-6 + eps_a)
    return xd, sd, gd, out, stats, ig, sg


@pytest.mark.parametrize("kind", ["uniform", "rmat", "dense", "ragged", "single"])
@pytest.mark.parametrize("h", [1, 4, 16, 41, 64, 100, 128, 256, 512])
def test_attn_planned_vs_oracle_and_reproducible(kind, h):
    row_end, col = graph(kind)
    n = row_end.shape[0]
    d_re, d_col = to_dev(row_end, col)
    plan = K.SgPlan(0, n - 1, 0, d_re, d_col)
    for heads in valid_heads(h):
        rng = np.random.RandomState(h * 10 + heads)
        x = rng.randn(n, h).astype(np.float32)
        s = rng.randn(n, 2 * heads).astype(np.float32)
        g = rng.randn(n, h).astype(np.float32)
        for vec in ((True, False) if h <= 256 else (True,)):
            what = "%s H=%d heads=%d %s" % (kind, h, heads, "padded" if vec else "ld=H")
            xd, sd, gd, out, stats, ig, sg = check(plan, row_end, col, x, s, g, heads, vec, what)
            out2, stats2 = plan.attn_forward(xd, sd, heads, SLOPE, out=feature_buf(n, h, vec))
            ig2, sg2 = plan.attn_backward(xd, sd, out, stats, gd, heads, SLOPE, in_grad=feature_buf(n, h, vec))
            torch.cuda.synchronize()
            for a, b in ((out, out2), (stats, stats2), (ig, ig2), (sg, sg2)):
                assert np.array_equal(bits(a), bits(b)), "%s: not bitwise reproducible" % what


def test_attn_partition_slice_with_global_ids():
    row_end, col = graph("rmat")
    n, h, heads = row_end.shape[0], 32, 2
    rng = np.random.RandomState(2)
    x, s, g = rng.randn(n, h), rng.randn(n, 2 * heads), rng.randn(n, h)
    x, s, g = (a.astype(np.float32) for a in (x, s, g))
    d_re, d_col = to_dev(row_end, col)
    whole = K.SgPlan(0, n - 1, 0, d_re, d_col)
    full = whole.attn_forward(dev(x, True), torch.from_numpy(s).to(DEV), heads, SLOPE)   # out / stats of every id
    for parts in (2, 4):
        k, vb, eb = oracle.partition(row_end, parts)
        for c in range(k):
            rl, rr, cl, cr = int(vb[c, 0]), int(vb[c, 1]), int(eb[c, 0]), int(eb[c, 1])
            s_re, s_col = row_end[rl:rr + 1], col[cl:cr + 1]
            plan = K.SgPlan(rl, rr, cl, *to_dev(s_re, s_col))
            check(plan, s_re, s_col, x, s, g, heads, True, "slice %d/%d" % (c, parts), self_base=rl, col_left=cl,
                  full=full)


def test_attn_large_scores_do_not_overflow():
    row_end, col = graph("uniform")
    n, h, heads = row_end.shape[0], 64, 4
    rng = np.random.RandomState(4)
    x = rng.randn(n, h).astype(np.float32)
    s = (rng.randn(n, 2 * heads) * 1000).astype(np.float32)
    g = rng.randn(n, h).astype(np.float32)
    assert not np.isfinite(np.exp(np.float32(np.abs(s).max())))
    plan = K.SgPlan(0, n - 1, 0, *to_dev(row_end, col))
    # fp32 rounds s_dst + s_src to half an ulp of its magnitude, and a = exp(y - m) / Z inherits that absolute error
    # in y as a relative one: two ulps at the largest |y|
    eps_a = 2.0 * float(np.spacing(np.float32(2 * np.abs(s).max())))
    _, _, _, out, stats, ig, sg = check(plan, row_end, col, x, s, g, heads, True, "scores x1000", eps_a=eps_a)
    for t in (out, stats, ig, sg):
        assert torch.isfinite(t).all()


def test_attn_zero_scores_give_the_mean():
    row_end, col = graph("rmat")
    n, h = row_end.shape[0], 48
    x = torch.from_numpy(np.random.RandomState(5).randn(n, h).astype(np.float32)).to(DEV)
    plan = K.SgPlan(0, n - 1, 0, *to_dev(row_end, col))
    out, stats = plan.attn_forward(x, torch.zeros((n, 2), device=DEV), 1, SLOPE)
    deg = torch.from_numpy(np.diff(np.concatenate([[0], row_end.astype(np.int64)]))).to(DEV).float()
    mean = plan.forward(x) / deg.clamp(min=1).unsqueeze(1)
    rel_close(out.cpu().numpy(), mean.cpu().numpy(), what="zero scores vs AGGR_AVG")
    assert torch.equal(stats[:, 0], torch.zeros_like(stats[:, 0]))


def test_attn_at_scale_20():
    """Hub rows spanning hundreds of chunks go through the big-row fix-ups of both passes."""
    re_t, col_t = datasets.rmat_graph(20, 1 << 23, seed=1, device=DEV)
    row_end = re_t.cpu().numpy().astype(np.uint64)
    col = col_t.cpu().numpy().astype(np.uint32)
    n, h, heads = row_end.shape[0], 64, 8
    plan = K.SgPlan(0, n - 1, 0, re_t, col_t)
    assert plan.info()["heavy_rows"] > 0
    rng = np.random.RandomState(20)
    x, s, g = rng.rand(n, h) - 0.5, rng.randn(n, 2 * heads), rng.rand(n, h) - 0.5
    check(plan, row_end, col, *(a.astype(np.float32) for a in (x, s, g)), heads, True, "scale 20")


def test_attn_invalid_and_unsupported_arguments():
    row_end, col = graph("uniform")
    plan = K.SgPlan(0, row_end.shape[0] - 1, 0, *to_dev(row_end, col))
    x = torch.zeros((1000, 600), device=DEV)
    f, b = _lib.lib.roc_sg_attn_forward_planned, _lib.lib.roc_sg_attn_backward_planned
    p = x.data_ptr()
    INV, UNS = _lib.ROC_ERR_INVALID, _lib.ROC_ERR_UNSUPPORTED

    def fwd(heads=1, H=16, slope=0.2, ptrs=(p, p, p, p), ld=(16, 16, 16, 16), plan_h=plan.handle):
        return f(plan_h, heads, H, slope, 0, ptrs[0], ld[0], ptrs[1], ld[1], ptrs[2], ld[2], ptrs[3], ld[3], None)

    def bwd(heads=1, H=16, slope=0.2, ptrs=(p,) * 7, ld=(16,) * 7):
        return b(plan.handle, heads, H, slope, 0, ptrs[0], ld[0], ptrs[1], ld[1], ptrs[2], ld[2], ptrs[3], ld[3],
                 ptrs[4], ld[4], ptrs[5], ld[5], ptrs[6], ld[6], None)

    assert fwd(plan_h=None) == INV
    for i in range(4):
        assert fwd(ptrs=tuple(None if k == i else p for k in range(4))) == INV
    for i in (0, 2):
        assert fwd(ld=tuple(15 if k == i else 16 for k in range(4))) == INV          # ld < H
    for i in (1, 3):
        assert fwd(heads=8, H=64, ld=tuple(15 if k == i else 64 for k in range(4))) == INV   # ld < 2 heads
    for heads in (0, -1):
        assert fwd(heads=heads) == INV
    assert fwd(H=0) == INV
    for slope in (-0.1, float("nan"), float("inf")):
        assert fwd(slope=slope) == INV
    for i in range(7):
        assert bwd(ptrs=tuple(None if k == i else p for k in range(7))) == INV
        assert bwd(ld=tuple(1 if k == i else 16 for k in range(7))) == INV
    assert bwd(slope=-1.0) == INV and bwd(heads=0) == INV
    # head layouts and widths the kernels do not take
    assert fwd(heads=3, H=12) == UNS                         # heads not in {1, 2, 4, 8}
    assert fwd(heads=16, H=64, ld=(64, 32, 64, 32)) == UNS
    assert fwd(heads=2, H=18, ld=(20, 4, 20, 4)) == UNS      # F = 9, not a power of two
    assert fwd(heads=4, H=8, ld=(8, 8, 8, 8)) == UNS         # F = 2 < 4
    assert fwd(heads=2, H=24, ld=(24, 4, 24, 4)) == UNS      # F = 12
    assert fwd(H=516, ld=(516, 4, 516, 4)) == UNS            # vector path: H > 512
    assert fwd(H=257, ld=(257, 4, 257, 4)) == UNS            # scalar path: H > 256
    assert bwd(heads=3, H=12) == UNS
    assert bwd(H=600, ld=(600, 4, 600, 4, 600, 600, 4)) == UNS


# ------------------------------------------------------------------- model ---
def small_case(layers, seed=9):
    re_t, col_t = datasets.rmat_graph(8, 1500, seed=31)
    row_end, col = re_t.numpy().astype(np.uint64), col_t.numpy().astype(np.uint32)
    feats, labels, mask = datasets.node_data(row_end.shape[0], layers[0], layers[-1], seed=seed)
    return row_end, col, feats.numpy(), labels.numpy(), mask.numpy()


def run_model(case, layers, heads, dropout=0.0, epochs=1, fuse=True):
    row_end, col, feats, labels, mask = case
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    hd = build_gat(m, list(layers), dropout, heads=heads)
    m.set_tensor(hd["input"], feats)
    m.set_labels(hd["label"], labels)
    m.set_tensor(hd["mask"], mask.astype(np.int32))
    res = {"w0": [m.get_parameter(p) for p in range(m.num_parameters())]}
    for ep in range(epochs):
        m.train_mode(); m.zero_gradients(); m.forward()
        if ep == 0:
            res["logits"] = m.get_tensor(hd["logits"])
        m.backward()
        if ep == 0:
            res["dW"] = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
    res["w"] = [m.get_parameter(p) for p in range(m.num_parameters())]
    host.close()
    return res


@pytest.mark.parametrize("layers,heads", [((12, 16, 5), (1,)), ((12, 32, 16, 5), (4, 1))])
def test_gat_against_torch_fp64_witness(layers, heads):
    case = small_case(layers)
    row_end, col, feats, labels, mask = case
    got = run_model(case, layers, list(heads))
    wl, wdw = gat_witness(row_end, col, feats, labels, mask, layers, got["w0"], heads)
    rel_close(got["logits"], wl, what="GAT logits vs torch fp64")
    for p, (a, b) in enumerate(zip(got["dW"], wdw)):
        rel_close(a, b, rtol=2e-4, atol_scale=2e-5, what="GAT dW[%d] vs torch autograd" % p)


def test_gat_fused_and_unfused_schedules_agree_bitwise():
    layers = (12, 32, 16, 5)
    case = small_case(layers)
    a = run_model(case, layers, [4, 1], dropout=0.5, epochs=3, fuse=True)
    b = run_model(case, layers, [4, 1], dropout=0.5, epochs=3, fuse=False)
    assert np.array_equal(a["logits"], b["logits"])
    for x, y in zip(a["dW"] + a["w"], b["dW"] + b["w"]):
        assert np.array_equal(x, y)


def build_attn_residual(model, dropout_rate, heads=4):
    """attention_gather where the two scratch paths of its backward run: on the raw features (a leaf: no input
    gradient), and on a tensor that also feeds a residual add, whose backward runs first (the gradient accumulates).

        a0 = attention_gather(x, linear(x, 2), 1)
        t  = linear(a0, 16)
        t  = relu(add(attention_gather(t, linear(t, 2 * heads), heads), t))
        logits = linear(t, 5)
    """
    x = model.create_node_tensor(12)
    label = model.create_node_tensor(5)
    mask = model.create_node_tensor(1, is_int=True)
    a0 = model.attention_gather(x, model.linear(x, 2), 1)
    t = model.linear(model.dropout(a0, dropout_rate), 16)
    t = model.relu(model.add(model.attention_gather(t, model.linear(t, 2 * heads), heads), t))
    logits = model.linear(t, 5)
    model.softmax_cross_entropy(logits, label, mask)
    model.adam(0.01, 0.05)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": logits}


def test_attention_gather_accumulating_and_leaf_inputs_against_witness():
    row_end, col, feats, labels, mask = small_case((12, 5))
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    hd = build_attn_residual(m, 0.0)
    m.set_tensor(hd["input"], feats)
    m.set_labels(hd["label"], labels)
    m.set_tensor(hd["mask"], mask.astype(np.int32))
    w0 = [m.get_parameter(p) for p in range(m.num_parameters())]
    m.train_mode(); m.zero_gradients(); m.forward()
    logits = m.get_tensor(hd["logits"])
    m.backward()
    dw = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
    host.close()
    # the witness, in torch fp64: parameters in creation order (score 0, feature 1, score 1, output)
    ws = [torch.from_numpy(w.astype(np.float64)).requires_grad_(True) for w in w0]
    dst, src = wg.edge_lists(row_end, col)
    n = row_end.shape[0]
    x = torch.from_numpy(feats.astype(np.float64))
    a0 = wg.attend(x, x @ ws[0].T, dst, src, n, 1, SLOPE)
    t = a0 @ ws[1].T
    t = torch.relu(wg.attend(t, t @ ws[2].T, dst, src, n, 4, SLOPE) + t)
    want = t @ ws[3].T
    wg.train_loss(want, labels, mask).backward()
    rel_close(logits, want.detach().numpy(), what="logits vs torch fp64")
    for p, (a, w) in enumerate(zip(dw, ws)):
        rel_close(a, w.grad.numpy(), rtol=2e-4, atol_scale=2e-5, what="dW[%d] vs torch autograd" % p)


@pytest.mark.parametrize("width,heads,message", [(12, 3, "heads must be 1, 2, 4 or 8"),
                                                 (24, 2, "power of two"), (8, 4, "power of two"),
                                                 (516, 1, "at most 512")])
def test_attention_gather_refuses_an_unsupported_layout_at_build(width, heads, message):
    prog = "\n".join([
        "import sys; sys.path.insert(0, %r)" % ROOT,
        "import numpy as np",
        "from roc_b200.model import Host, Model",
        "host = Host(0, 0, 1)",
        "host.graph_from_arrays(np.array([2, 4], dtype=np.uint64), np.array([0, 1, 0, 1], dtype=np.uint32))",
        "m = Model(host, seed=1)",
        "x = m.create_node_tensor(%d)" % width,
        "m.attention_gather(x, m.linear(x, %d), %d)" % (2 * heads, heads),
        "print('built')",
    ])
    p = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ))
    assert p.returncode != 0 and "built" not in p.stdout
    assert message in p.stderr, p.stderr[-2000:]


def test_attention_gather_refuses_more_than_one_partition():
    prog = "\n".join([
        "import sys; sys.path.insert(0, %r)" % ROOT,
        "import numpy as np",
        "from roc_b200.model import Host, Model, build_gat",
        "host = Host(0, 0, 2)",
        "host.graph_from_arrays(np.array([2, 4, 6, 8], dtype=np.uint64), np.array([0, 1, 0, 1, 2, 3, 2, 3], dtype=np.uint32))",
        "m = Model(host, seed=1)",
        "build_gat(m, [4, 4, 2], 0.0)",
        "print('initialised')",
    ])
    p = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ))
    assert p.returncode != 0 and "initialised" not in p.stdout
    assert "one partition only" in p.stderr, p.stderr[-2000:]
