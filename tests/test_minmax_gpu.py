"""Max / min ScatterGather on the GPU: the kernels against the oracle's definition (values and indices bit-exact,
backward within the parity tolerance and bitwise reproducible), and GraphSAGE-pool through the Model API against an
independent torch fp64 autograd witness."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import minmax_oracle as mmo
from conftest import ROOT, rel_close
from oracle import oracle
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_sage_mean, build_sage_pool
from sg_graphs import graph, to_dev
from witness_pool import sage_pool_witness

pytestmark = pytest.mark.gpu
DEV = "cuda"
AGGRS = (_lib.AGGR_MAX, _lib.AGGR_MIN)


def bits(t):
    return t.contiguous().cpu().view(torch.int32).numpy() if isinstance(t, torch.Tensor) else t.view(np.int32)


def check_forward(plan, x_dev, want, warg, aggr, what):
    out, arg = plan.minmax_forward(x_dev, aggr)
    torch.cuda.synchronize()
    assert np.array_equal(bits(out), bits(want)), "%s: values differ from the oracle" % what
    assert np.array_equal(bits(arg), bits(warg)), "%s: indices differ from the oracle" % what
    return out, arg


@pytest.mark.parametrize("kind", ["uniform", "rmat", "dense", "ragged", "single"])
@pytest.mark.parametrize("h", [1, 4, 16, 41, 64, 100, 128, 256, 602])
def test_minmax_planned_vs_oracle(kind, h):
    row_end, col = graph(kind)
    n = row_end.shape[0]
    rng = np.random.RandomState(h)
    x = rng.randn(n, h).astype(np.float32)
    gy = rng.randn(n, h).astype(np.float32)
    d_re, d_col = to_dev(row_end, col)
    plan = K.SgPlan(0, n - 1, 0, d_re, d_col)
    xp = K.padded(n, h, DEV, fill=torch.from_numpy(x).to(DEV))        # ld = round_up(h, 4): vector path
    xd = torch.from_numpy(x).to(DEV)                                 # ld = h: scalar path when h % 4
    gp = K.padded(n, h, DEV, fill=torch.from_numpy(gy).to(DEV))
    gd = torch.from_numpy(gy).to(DEV)
    for aggr in AGGRS:
        want, warg = mmo.forward(0, n - 1, 0, row_end, col, x, aggr)
        wgrad = mmo.backward(0, n - 1, 0, row_end, col, gy, warg)
        _, arg_p = check_forward(plan, xp, want, warg, aggr, "%s H=%d aggr %d padded" % (kind, h, aggr))
        _, arg_d = check_forward(plan, xd, want, warg, aggr, "%s H=%d aggr %d dense" % (kind, h, aggr))
        g1 = plan.minmax_backward(gp, arg_p)
        rel_close(g1.cpu().numpy(), wgrad, what="%s H=%d aggr %d backward padded" % (kind, h, aggr))
        g2 = plan.minmax_backward(gd, arg_d)
        rel_close(g2.cpu().numpy(), wgrad, what="%s H=%d aggr %d backward dense" % (kind, h, aggr))
        assert torch.equal(plan.minmax_backward(gp, arg_p), g1), "backward must be bitwise reproducible"


def test_minmax_partition_slice_with_global_ids():
    row_end, col = graph("rmat")
    n, h = row_end.shape[0], 24
    rng = np.random.RandomState(2)
    x = rng.randn(n, h).astype(np.float32)
    gy = rng.randn(n, h).astype(np.float32)
    _, warg_all = mmo.forward(0, n - 1, 0, row_end, col, x, _lib.AGGR_MAX)
    xd, gd = torch.from_numpy(x).to(DEV), torch.from_numpy(gy).to(DEV)
    arg_all = torch.from_numpy(warg_all.view(np.int32)).to(DEV)
    for parts in (2, 4):
        k, vb, eb = oracle.partition(row_end, parts)
        for c in range(k):
            rl, rr, cl, cr = int(vb[c, 0]), int(vb[c, 1]), int(eb[c, 0]), int(eb[c, 1])
            assert rl > 0 or c == 0
            d_re, d_col = to_dev(row_end[rl:rr + 1], col[cl:cr + 1])
            plan = K.SgPlan(rl, rr, cl, d_re, d_col)
            want, warg = mmo.forward(rl, rr, cl, row_end[rl:rr + 1], col[cl:cr + 1], x, _lib.AGGR_MAX)
            check_forward(plan, xd, want, warg, _lib.AGGR_MAX, "slice %d/%d" % (c, parts))
            wgrad = mmo.backward(rl, rr, cl, row_end[rl:rr + 1], col[cl:cr + 1], gy, warg_all, self_base=rl)
            got = plan.minmax_backward(gd, arg_all, self_base=rl)
            rel_close(got.cpu().numpy(), wgrad, what="slice %d/%d backward" % (c, parts))


def test_minmax_propagates_nan():
    row_end, col = graph("rmat")
    n, h = row_end.shape[0], 64
    rng = np.random.RandomState(7)
    x = rng.randn(n, h).astype(np.float32)
    x[rng.rand(n, h) < 0.01] = np.nan
    x[rng.rand(n, h) < 0.01] = -np.inf
    d_re, d_col = to_dev(row_end, col)
    plan = K.SgPlan(0, n - 1, 0, d_re, d_col)
    for aggr in AGGRS:
        want, warg = mmo.forward(0, n - 1, 0, row_end, col, x, aggr)
        assert np.isnan(want).any()
        check_forward(plan, torch.from_numpy(x).to(DEV), want, warg, aggr, "NaN input aggr %d" % aggr)


def test_minmax_invalid_arguments():
    row_end, col = graph("uniform")
    d_re, d_col = to_dev(row_end, col)
    plan = K.SgPlan(0, row_end.shape[0] - 1, 0, d_re, d_col)
    x = torch.zeros((1000, 8), device=DEV)
    a = torch.zeros((1000, 8), device=DEV, dtype=torch.int32)
    f = _lib.lib.roc_sg_minmax_forward_planned
    xp, ap = x.data_ptr(), a.data_ptr()
    for aggr in (0, 3, 4, -1):
        assert f(plan.handle, aggr, 8, xp, 8, xp, 8, ap, 8, None) == _lib.ROC_ERR_INVALID
    assert f(plan.handle, 1, 0, xp, 8, xp, 8, ap, 8, None) == _lib.ROC_ERR_INVALID
    assert f(plan.handle, 1, 8, None, 8, xp, 8, ap, 8, None) == _lib.ROC_ERR_INVALID
    assert f(plan.handle, 1, 8, xp, 8, xp, 8, None, 8, None) == _lib.ROC_ERR_INVALID
    assert f(plan.handle, 1, 8, xp, 8, xp, 8, ap, 4, None) == _lib.ROC_ERR_INVALID
    assert f(None, 1, 8, xp, 8, xp, 8, ap, 8, None) == _lib.ROC_ERR_INVALID
    b = _lib.lib.roc_sg_minmax_backward_planned
    assert b(plan.handle, 8, 0, xp, 8, None, 8, xp, 8, None) == _lib.ROC_ERR_INVALID
    assert b(plan.handle, 8, 0, xp, 4, ap, 8, xp, 8, None) == _lib.ROC_ERR_INVALID
    assert b(plan.handle, -1, 0, xp, 8, ap, 8, xp, 8, None) == _lib.ROC_ERR_INVALID
    assert plan.rows_sorted()


def test_minmax_at_scale_20():
    """Hub rows spanning hundreds of chunks go through the big-row fix-up."""
    re_t, col_t = datasets.rmat_graph(20, 1 << 23, seed=1, device=DEV)
    row_end = re_t.cpu().numpy().astype(np.uint64)
    col = col_t.cpu().numpy().astype(np.uint32)
    n, h = row_end.shape[0], 64
    rng = np.random.RandomState(20)
    x = rng.rand(n, h).astype(np.float32) - 0.5
    gy = rng.rand(n, h).astype(np.float32) - 0.5
    plan = K.SgPlan(0, n - 1, 0, re_t, col_t)
    assert plan.info()["heavy_rows"] > 0
    want, warg = mmo.forward(0, n - 1, 0, row_end, col, x, _lib.AGGR_MAX)
    _, arg = check_forward(plan, torch.from_numpy(x).to(DEV), want, warg, _lib.AGGR_MAX, "scale 20")
    got = plan.minmax_backward(torch.from_numpy(gy).to(DEV), arg).cpu().numpy()
    rel_close(got, mmo.backward(0, n - 1, 0, row_end, col, gy, warg), what="scale 20 backward")


# ------------------------------------------------------------------- model ---
def small_case(layers, seed=9):
    re_t, col_t = datasets.rmat_graph(8, 1500, seed=31)
    row_end, col = re_t.numpy().astype(np.uint64), col_t.numpy().astype(np.uint32)
    feats, labels, mask = datasets.node_data(row_end.shape[0], layers[0], layers[-1], seed=seed)
    return row_end, col, feats.numpy(), labels.numpy(), mask.numpy()


def run_model(builder, case, layers, dropout=0.0, epochs=1, fuse=True):
    row_end, col, feats, labels, mask = case
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    h = builder(m, list(layers), dropout)
    m.set_tensor(h["input"], feats)
    m.set_labels(h["label"], labels)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    res = {"w0": [m.get_parameter(p) for p in range(m.num_parameters())]}
    for ep in range(epochs):
        m.train_mode(); m.zero_gradients(); m.forward()
        if ep == 0:
            res["logits"] = m.get_tensor(h["logits"])
            res["args"] = [m.get_aggr_index(t) for t in h.get("pools", [])]
        m.backward()
        if ep == 0:
            res["dW"] = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
    res["w"] = [m.get_parameter(p) for p in range(m.num_parameters())]
    host.close()
    return res


@pytest.mark.parametrize("aggr,layers", [(_lib.AGGR_MAX, (12, 16, 5)), (_lib.AGGR_MAX, (12, 24, 16, 5)),
                                         (_lib.AGGR_MIN, (12, 24, 16, 5))])
def test_sage_pool_against_torch_fp64_witness(aggr, layers):
    case = small_case(layers)
    row_end, col, feats, labels, mask = case
    got = run_model(lambda m, l, d: build_sage_pool(m, l, d, aggr=aggr), case, layers)
    is_max = aggr == _lib.AGGR_MAX
    wl, wdw, chosen, pools = sage_pool_witness(row_end, col, feats, labels, mask, layers, got["w0"], is_max)
    # Where fp32 and fp64 pick different sources, the candidates must be equal to within rounding; the witness then
    # takes the product's choice (the policy DESIGN §4 uses for ReLU sign flips).
    flips = 0
    for pa, wa, p64 in zip(got["args"], chosen, pools):
        diff = pa.astype(np.int64) != wa
        if diff.any():
            cols = np.nonzero(diff)[1]
            a, b = p64[pa[diff].astype(np.int64), cols], p64[wa[diff], cols]
            assert np.abs(a - b).max() <= 1e-5 * np.abs(p64).max(), "argmax differs away from a tie"
            flips += int(diff.sum())
    if flips:
        wl, wdw, _, _ = sage_pool_witness(row_end, col, feats, labels, mask, layers, got["w0"], is_max,
                                          args=[a.astype(np.int64) for a in got["args"]])
    rel_close(got["logits"], wl, what="sage-pool logits vs torch fp64")
    for p, (a, b) in enumerate(zip(got["dW"], wdw)):
        rel_close(a, b, rtol=2e-4, atol_scale=2e-5, what="sage-pool dW[%d] vs torch autograd" % p)


def test_sage_pool_fused_and_unfused_schedules_agree_bitwise():
    layers = (12, 24, 16, 5)
    case = small_case(layers)
    a = run_model(build_sage_pool, case, layers, dropout=0.5, epochs=3, fuse=True)
    b = run_model(build_sage_pool, case, layers, dropout=0.5, epochs=3, fuse=False)
    assert np.array_equal(a["logits"], b["logits"])
    for x, y in zip(a["dW"] + a["w"], b["dW"] + b["w"]):
        assert np.array_equal(x, y)


def build_sage_avg(model, layers, dropout_rate):
    """build_sage_mean with the aggregation spelled scatter_gather(t, AGGR_AVG)."""
    L = len(layers)
    x = model.create_node_tensor(layers[0])
    label = model.create_node_tensor(layers[-1])
    mask = model.create_node_tensor(1, is_int=True)
    t = x
    for i in range(1, L):
        d = model.dropout(t, dropout_rate)
        nb = model.scatter_gather(model.linear(d, layers[i], _lib.AC_MODE_NONE), _lib.AGGR_AVG)
        t = model.add(nb, model.linear(d, layers[i], _lib.AC_MODE_NONE))
        if i != L - 1:
            t = model.relu(t)
    model.softmax_cross_entropy(t, label, mask)
    model.adam(0.01, 0.05)
    model.init()
    return {"input": x, "label": label, "mask": mask, "logits": t}


def test_avg_aggregation_is_the_sage_mean_wiring_bitwise():
    layers = (12, 24, 16, 5)
    case = small_case(layers)
    a = run_model(build_sage_avg, case, layers, dropout=0.5, epochs=2)
    b = run_model(build_sage_mean, case, layers, dropout=0.5, epochs=2)
    assert np.array_equal(a["logits"], b["logits"])
    for x, y in zip(a["dW"] + a["w"], b["dW"] + b["w"]):
        assert np.array_equal(x, y)


def test_init_refuses_a_graph_with_an_unsorted_row():
    prog = "\n".join([
        "import sys; sys.path.insert(0, %r)" % ROOT,
        "import numpy as np",
        "from roc_b200.model import Host, Model, build_sage_pool",
        "host = Host(0, 0, 1)",
        # row 1 lists source 2 before source 0
        "host.graph_from_arrays(np.array([2, 4, 6], dtype=np.uint64), np.array([0, 1, 2, 0, 1, 2], dtype=np.uint32))",
        "m = Model(host, seed=1)",
        "build_sage_pool(m, [4, 4, 2], 0.0)",
        "print('initialised')",
    ])
    p = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ))
    assert p.returncode != 0 and "initialised" not in p.stdout
    assert "strictly increasing" in p.stderr, p.stderr[-2000:]
