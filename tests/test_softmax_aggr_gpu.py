"""The softmax aggregation on the GPU.

Kernels: roc_sg_softmax_forward_planned, roc_sg_softmax_backward_planned and roc_sg_softmax_backward_exact against the
fp64 autograd witness of tests/softmax_aggr_witness.py, over H in {1, 3, 4, 5, 8, 16, 17, 32, 33, 41, 64, 65, 100, 128,
129, 200, 256, 300} (every J = ceil(H / 32) up to 8, and one column block past the widest), with and without dt, on a
symmetric graph with heavy rows and a hub whose row takes the big-row fix-up (the same-CSR backward is exact there and
equals the exact one within the bar), on a directed multigraph for the exact backward, and on the whole graphs of
tests/sg_matrix.py.  Rows live in NaN-padded buffers, outputs in sentinel-padded ones.  Also t = 0 against the mean, a
large t against the max aggregation, a negative t, |x| up to 1e3, repeat calls and three SM budgets byte-identical,
the launch lists, and the refusals.

Models: build_deepergcn at depth 3 over three Adam steps against the witness (each step from the product's weights):
logits, every dW, dt and t after Adam; learn_temperature on and off, norm None and "batch", loss="sigmoid",
exact_backward on a directed graph, infer-mode logits, set_fusion(False) bit-identical to fusion on; op_info,
parameter_shape and the refusal of a bf16 input.

Bounds: each output against fp64 with |got - want| <= 2e-4 |want| + 2e-5 max|want| (the bar of test_gatv2_gpu.py);
dt, a sum over every edge and column, at 1e-3 |want| + 1e-4 max|want|, as GATv2's da."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import sg_matrix as sgm

from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_deepergcn
from softmax_aggr_witness import kernel_witness, model_witness
from witness_gat import train_loss

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HS = [1, 3, 4, 5, 8, 16, 17, 32, 33, 41, 64, 65, 100, 128, 129, 200, 256, 300]
SENTINEL = 12345.0


def close(name, got, want, rtol=2e-4, atol_scale=2e-5):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.isfinite(got).all(), name
    scale = np.abs(want).max() if want.size else 0.0
    bound = rtol * np.abs(want) + atol_scale * scale + 1e-30
    r = float((np.abs(got - want) / bound).max()) if want.size else 0.0
    assert r <= 1.0, (name, r)


def _csr(n, pairs):
    dst = np.array([p[0] for p in pairs], dtype=np.int64)
    col = np.array([p[1] for p in pairs], dtype=np.uint32)
    return np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64), col


def sym_graph():
    """a symmetric graph with self loops, heavy rows (degree > 64) and one hub whose row spans > 32 chunks"""
    rng = np.random.RandomState(7)
    n = 3000
    pairs = {(i, i) for i in range(n)}
    for _ in range(6000):
        u, v = rng.randint(0, n, 2)
        pairs |= {(u, v), (v, u)}
    for u in range(1, 2600):
        pairs |= {(0, u), (u, 0)}
    for u in range(100, 300):
        pairs |= {(5, u), (u, 5)}
    return _csr(n, sorted(pairs))


def directed_multigraph():
    rng = np.random.RandomState(8)
    n = 2000
    pairs = [(i, i) for i in range(n)] + [tuple(rng.randint(0, n, 2)) for _ in range(9000)]
    pairs += [(3, u) for u in range(0, 1500)] + [(3, 7)] * 3
    return _csr(n, sorted(pairs))


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
    buf = torch.full((rows, (h + 6) // 4 * 4), float("nan"), device="cuda")
    buf[:, :h] = torch.from_numpy(np.asarray(v, dtype=np.float32))
    return buf[:, :h]


def out_rows(rows, h):
    """an output [rows][h] in a sentinel-filled buffer with pad columns"""
    return torch.full((rows, (h + 6) // 4 * 4), SENTINEL, device="cuda")[:, :h]


def inputs(n, h, seed, scale=1.0):
    rng = np.random.RandomState(seed)
    x = (scale * rng.standard_normal((n, h))).astype(np.float32)
    gy = rng.standard_normal((n, h)).astype(np.float32)
    return x, gy


def run(plan, tr, n, x, gy, t, exact=False, want_dt=True):
    x_, gy_ = nan_rows(x), nan_rows(gy)
    h = x.shape[1]
    y, stats = plan.softmax_forward(x_, t, out=out_rows(n, h), stats=out_rows(n, 2 * h))
    dx = out_rows(n, h)
    if exact:
        dx, dt = tr.softmax_backward(plan, x_, t, y, stats, gy_, dx=dx, want_dt=want_dt)
    else:
        dx, dt = plan.softmax_backward(x_, t, y, stats, gy_, dx=dx, want_dt=want_dt)
    torch.cuda.synchronize()
    pads = [v.as_strided((v.shape[0], v.stride(0)), (v.stride(0), 1))[:, v.shape[1]:] for v in (y, stats, dx)]
    assert all(bool((p == SENTINEL).all()) for p in pads), "a store past the row"
    return dict(out=y.cpu().numpy(), stats=stats.cpu().numpy(), dx=dx.cpu().numpy(),
                dt=None if dt is None else dt.cpu().numpy())


def check(got, want, h, what, dx=True):
    close(what + " out", got["out"], want["out"])
    close(what + " m", got["stats"][:, :h], want["m"])
    close(what + " 1/Z", got["stats"][:, h:2 * h], want["iz"])
    if dx:
        close(what + " dx", got["dx"], want["dx"])
        if got["dt"] is not None:
            close(what + " dt", got["dt"], [want["dt"]], rtol=1e-3, atol_scale=1e-4)


@pytest.mark.parametrize("h", HS)
def test_kernels_against_fp64_on_a_symmetric_graph(h):
    g = graph("sym")
    x, gy = inputs(g["n"], h, seed=h)
    want = kernel_witness(g["row_end"], g["col"], x, 0.7, gy)
    planned = run(g["plan"], g["tr"], g["n"], x, gy, 0.7)
    check(planned, want, h, "H=%d" % h)
    exact = run(g["plan"], g["tr"], g["n"], x, gy, 0.7, exact=True)
    check(exact, want, h, "H=%d exact" % h)
    close("H=%d same-CSR vs exact dx" % h, planned["dx"], exact["dx"])
    no_dt = run(g["plan"], g["tr"], g["n"], x, gy, 0.7, want_dt=False)
    assert no_dt["dt"] is None and np.array_equal(no_dt["dx"].view(np.int32), planned["dx"].view(np.int32))


@pytest.mark.parametrize("h", [1, 17, 64, 129, 300])
@pytest.mark.parametrize("want_dt", [True, False])
def test_exact_backward_on_a_directed_multigraph(h, want_dt):
    g = graph("directed")
    x, gy = inputs(g["n"], h, seed=h + 1)
    want = kernel_witness(g["row_end"], g["col"], x, -0.4, gy)
    check(run(g["plan"], g["tr"], g["n"], x, gy, -0.4, exact=True, want_dt=want_dt), want, h, "H=%d" % h)


@pytest.mark.parametrize("h", [5, 64, 200])
def test_temperature_limits(h):
    """t = 0 against the mean, t = 1e4 against the max aggregation, and a negative t against the witness"""
    g = graph("sym")
    x, gy = inputs(g["n"], h, seed=3)
    x_ = nan_rows(x)
    mean = g["plan"].softmax_forward(x_, 0.0)[0]
    deg = torch.from_numpy(np.diff(np.concatenate([[0], g["row_end"].astype(np.int64)])).astype(np.float32)).cuda()
    summed = g["plan"].forward(x_)
    close("t=0", mean.cpu().numpy(), (summed / deg.clamp(min=1)[:, None]).cpu().numpy())
    # at t = 1e4 the weight of a value d below the row's max is exp(-1e4 d), so y is within 1 / (e 1e4) of the max
    mx = g["plan"].minmax_forward(x_, _lib.AGGR_MAX)[0]
    big = g["plan"].softmax_forward(x_, 1e4)[0]
    np.testing.assert_allclose(big.cpu().numpy(), mx.cpu().numpy(), rtol=0, atol=1e-3)
    check(run(g["plan"], g["tr"], g["n"], x, gy, -3.0), kernel_witness(g["row_end"], g["col"], x, -3.0, gy), h,
          "t=-3")


def test_large_inputs_are_finite():
    """|x| up to 1e3 at t = 1: z - m and t x - m never overflow (exp(t x) alone would)"""
    g = graph("sym")
    x, gy = inputs(g["n"], 64, seed=5, scale=300.0)
    x = np.clip(x, -1e3, 1e3)
    want = kernel_witness(g["row_end"], g["col"], x, 1.0, gy)
    got = run(g["plan"], g["tr"], g["n"], x, gy, 1.0)
    close("|x|<=1e3 out", got["out"], want["out"])
    assert np.isfinite(got["dx"]).all() and np.isfinite(got["dt"]).all()


def _bits(r):
    return {k: v.view(np.int32).copy() for k, v in r.items() if v is not None}


@pytest.mark.parametrize("h", [3, 64, 129, 300])
def test_repeats_and_sm_budgets_are_byte_identical(h):
    for name, exact in (("sym", False), ("directed", True)):
        g = graph(name)
        x, gy = inputs(g["n"], h, seed=11)
        ref = _bits(run(g["plan"], g["tr"], g["n"], x, gy, 0.9, exact=exact))
        assert all(np.array_equal(v, ref[k]) for k, v in _bits(run(g["plan"], g["tr"], g["n"], x, gy, 0.9,
                                                                   exact=exact)).items())
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        prev = _lib.lib.roc_set_sm_reserve(0)
        try:
            for reserve in (sms - 8, sms // 2 + 1):
                _lib.lib.roc_set_sm_reserve(int(reserve))
                got = _bits(run(g["plan"], g["tr"], g["n"], x, gy, 0.9, exact=exact))
                assert all(np.array_equal(v, ref[k]) for k, v in got.items()), (name, reserve)
        finally:
            _lib.lib.roc_set_sm_reserve(prev)


# The launch lists, restated (kind, red, vec, lanes, nch, grid), per column block of Hb <= 256 columns.
def blocks(h):
    return [min(256, h - c0) for c0 in range(0, h, 256)]


def forward_launches(s, h):
    out = []
    for hb in blocks(h):
        j = sgm.cdiv(hb, 32)
        out.append(("main", 72, 1, 32, j, sgm.cdiv(s.chunks, 8)))
        if s.heavy:
            out.append(("fixup", 72, 1, 32, j, sgm.cdiv(s.heavy, 8)))
        if s.big:
            out.append(("big_fixup", 72, 1, 32, j, s.big))
    return out


def backward_launches(sb, n, h, dt):
    out = []
    for hb in blocks(h):
        j, (lanes, nch) = sgm.cdiv(hb, 32), sgm.shape(hb)
        out += [("record", -1, 1, 32, j, sgm.cdiv(n, 8))] if n else []
        out += [("main", 74 if dt else 73, 1, 32, j, sgm.cdiv(sb.chunks, 8))]
        out += (2 if dt else 1) * sgm.fixups(sb, 0, 1, lanes, nch)
    if dt and n:
        out += [("colsum", -1, 1, 256, 1, sgm.cdiv(n, 512)), ("colsum", -1, 1, 32, 1, 1)]
    return out


def launched():
    return [(l["kind"], l["red"], l["vec"], l["lanes"], l["nch"], l["grid"]) for l in K.sg_launches()]


SEEN = set()


@pytest.mark.parametrize("h", [3, 64, 300])
@pytest.mark.parametrize("name", ["empty", "single", "tiny", "aligned", "straddle", "carry32", "ragged", "directed",
                                  "hub", "fanout"])
def test_sg_matrix_graphs(name, h):
    """rows of degree 0, rows ending on chunk boundaries, 32 and 33 carries, heavy and big rows, directed multigraphs:
    the forward and the exact backward against the witness, the launch lists of every call"""
    g = sgm.xgraphs()[name]
    x, gy = inputs(g.n, h, seed=h)
    x_, gy_ = nan_rows(x), nan_rows(gy)

    def seen(want, what):
        got = launched()
        assert got == want, (name, h, what, got, want)
        SEEN.update((l[1], l[4]) for l in got if l[0] == "main")
    y, stats = g.plan.softmax_forward(x_, 0.6)
    seen(forward_launches(g.sched, h), "forward")
    g.plan.softmax_backward(x_, 0.6, y, stats, gy_)
    seen(backward_launches(g.sched, g.n, h, True), "backward")
    g.plan.softmax_backward(x_, 0.6, y, stats, gy_, want_dt=False)
    seen(backward_launches(g.sched, g.n, h, False), "backward without dt")
    dx, dt = g.tr.softmax_backward(g.plan, x_, 0.6, y, stats, gy_)
    seen(backward_launches(g.sched_t, g.n, h, True), "exact backward")
    infer = g.plan.softmax_forward(x_, 0.6, keep_stats=False)[0]
    torch.cuda.synchronize()
    want = kernel_witness(g.row_end, g.col, x, 0.6, gy)
    what = "%s H=%d" % (name, h)
    y, stats = y.cpu().numpy(), stats.cpu().numpy()
    close(what + " out", y, want["out"])
    close(what + " m", stats[:, :h], want["m"])
    close(what + " 1/Z", stats[:, h:], want["iz"])
    assert np.array_equal(infer.cpu().numpy().view(np.int32), y.view(np.int32)), what
    deg0 = g.deg == 0
    assert not y[deg0].any() and not stats[deg0].any(), what
    close(what + " exact dx", dx.cpu().numpy(), want["dx"])
    close(what + " exact dt", dt.cpu().numpy(), [want["dt"]], rtol=1e-3, atol_scale=1e-4)


def test_every_instantiation():
    """J = 1..8 of the forward, both source passes and the record, with their fix-ups, on the ragged graph"""
    g = sgm.xgraphs()["ragged"]
    for h in (1, 33, 65, 97, 129, 161, 193, 225):
        x, gy = inputs(g.n, h, seed=h)
        x_, gy_ = nan_rows(x), nan_rows(gy)
        y, stats = g.plan.softmax_forward(x_, 1.3)
        SEEN.update((l["red"], l["nch"]) for l in K.sg_launches() if l["kind"] == "main")
        for want_dt in (True, False):
            g.tr.softmax_backward(g.plan, x_, 1.3, y, stats, gy_, want_dt=want_dt)
            SEEN.update((l["red"], l["nch"]) for l in K.sg_launches() if l["kind"] == "main")
        torch.cuda.synchronize()
        close("H=%d out" % h, y.cpu().numpy(), kernel_witness(g.row_end, g.col, x, 1.3, gy)["out"])
    assert {(r, j) for r in (72, 73, 74) for j in range(1, 9)} <= SEEN


def test_refusals():
    g = graph("sym")
    n = g["n"]
    x = torch.zeros((n, 8), device="cuda")
    y = torch.zeros((n, 8), device="cuda")
    st = torch.zeros((n, 16), device="cuda")
    t = torch.ones((1,), device="cuda")
    p = g["plan"].handle
    f = _lib.lib.roc_sg_softmax_forward_planned

    def fw(H=8, tt=t, xx=x, yy=y, stats=st, ld=8, lds=16):
        return f(p, H, K._ptr(tt), K._ptr(xx), ld, K._ptr(yy), ld, K._ptr(stats), lds, None)
    assert fw() == 0 and fw(stats=None, lds=0) == 0
    assert fw(tt=None) == _lib.ROC_ERR_INVALID and fw(xx=None) == _lib.ROC_ERR_INVALID
    assert fw(yy=None) == _lib.ROC_ERR_INVALID and fw(H=0) == _lib.ROC_ERR_INVALID
    assert fw(ld=7) == _lib.ROC_ERR_INVALID and fw(lds=15) == _lib.ROC_ERR_INVALID and fw(yy=x) == _lib.ROC_ERR_INVALID
    sl = sgm.graphs()["slice"]
    xs, ys = torch.zeros((sl.n, 8), device="cuda"), torch.zeros((sl.n, 8), device="cuda")
    assert f(sl.plan.handle, 8, K._ptr(t), K._ptr(xs), 8, K._ptr(ys), 8, None, 0, None) == _lib.ROC_ERR_UNSUPPORTED
    b = _lib.lib.roc_sg_softmax_backward_planned
    gy, dx, dt = torch.zeros_like(x), torch.zeros_like(x), torch.zeros((1,), device="cuda")

    def bw(dxx=dx, dtt=dt, stats=st, gyy=gy, tt=t):
        return b(p, 8, K._ptr(tt), K._ptr(x), 8, K._ptr(y), 8, K._ptr(stats), 16, K._ptr(gyy), 8, K._ptr(dxx), 8,
                 K._ptr(dtt), None)
    assert bw() == 0 and bw(dtt=None) == 0
    assert bw(stats=None) == _lib.ROC_ERR_INVALID and bw(gyy=None) == _lib.ROC_ERR_INVALID
    assert bw(dxx=None) == _lib.ROC_ERR_INVALID and bw(tt=None) == _lib.ROC_ERR_INVALID
    for alias in (x, y, gy, st):
        assert bw(dxx=alias) == _lib.ROC_ERR_INVALID
    assert bw(dtt=t) == _lib.ROC_ERR_INVALID
    e = _lib.lib.roc_sg_softmax_backward_exact
    other = graph("directed")
    assert e(p, other["tr"].handle, 8, K._ptr(t), K._ptr(x), 8, K._ptr(y), 8, K._ptr(st), 16, K._ptr(gy), 8,
             K._ptr(dx), 8, K._ptr(dt), None) == _lib.ROC_ERR_INVALID
    assert e(p, None, 8, K._ptr(t), K._ptr(x), 8, K._ptr(y), 8, K._ptr(st), 16, K._ptr(gy), 8,
             K._ptr(dx), 8, K._ptr(dt), None) == _lib.ROC_ERR_INVALID
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------- the models ---
LAYERS = [24, 16, 12]
DEPTH = 3


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


def train(graph_, steps=3, loss="softmax", fusion=True, **kw):
    row_end, col = graph_
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    if not fusion:
        m.set_fusion(False)
    h = build_deepergcn(m, LAYERS, 0.0, DEPTH, loss=loss, **kw)
    if loss == "sigmoid":
        feats, labels, mask = (t.numpy() for t in datasets.multilabel_node_data(n, LAYERS[0], LAYERS[-1], seed=5))
        m.set_multilabels(h["label"], labels)
    else:
        feats, labels, mask = (t.numpy() for t in datasets.node_data(n, LAYERS[0], LAYERS[-1], seed=5))
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
        st["w1"] = [m.get_parameter(p) for p in range(m.num_parameters())]
        out["steps"].append(st)
    return out


def adam_t(t0, grads, lr=0.01, wd=0.05, b1=0.9, b2=0.999, eps=1e-8):
    """t after Adam steps from t0 with gradients `grads`, weight decay added to the gradient (the engine's Adam)"""
    t, m, v = float(t0), 0.0, 0.0
    for k, g in enumerate(grads, 1):
        g = g + wd * t
        m, v = b1 * m + (1 - b1) * g, b2 * v + (1 - b2) * g * g
        t -= lr * np.sqrt(1 - b2 ** k) / (1 - b1 ** k) * m / (np.sqrt(v) + eps)
    return t


def check_model(run, graph_, loss="softmax", **kw):
    row_end, col = graph_
    for k, st in enumerate(run["steps"]):
        logits, dw = model_witness(row_end, col, run["feats"], run["labels"], run["mask"], LAYERS, st["w0"], DEPTH,
                                   loss_fn=bce_loss if loss == "sigmoid" else train_loss, **kw)
        close("step %d logits" % k, st["logits"], logits)
        for p, (a, b) in enumerate(zip(st["dw"], dw)):
            close("step %d dW%d" % (k, p), a, b, rtol=1e-3, atol_scale=1e-4)
    temps = [p for p in run["h"]["temperatures"] if p is not None]
    for p in temps:
        grads = [float(st["dw"][p][0, 0]) for st in run["steps"]]
        t1 = float(run["steps"][-1]["w1"][p][0, 0])
        assert abs(t1 - adam_t(run["steps"][0]["w0"][p][0, 0], grads)) <= 1e-5, (p, t1)


# At t = 0.8, learn_temperature=False and norm=None, one input of the head's relu lands 8.7e-9 from 0 at the second
# step, where fp32 and fp64 take different sides of the kink: 0.9 keeps every case clear of such a tie.
T0 = 0.9


@pytest.mark.parametrize("learn", [True, False])
@pytest.mark.parametrize("norm", ["batch", None])
def test_build_deepergcn_against_the_witness(learn, norm):
    g = sym_model_graph()
    r = train(g, learn_temperature=learn, norm=norm, temperature=T0)
    check_model(r, g, learn_temperature=learn, norm=norm, temperature=T0)
    temps = r["h"]["temperatures"]
    assert len(temps) == DEPTH
    if learn:
        assert all(r["shapes"][p] == (1, 1) for p in temps)
        assert all(r["steps"][0]["w0"][p][0, 0] == np.float32(T0) for p in temps)
    else:
        assert temps == [None] * DEPTH
    kinds = [o["kind"] for o in r["info"]]
    assert kinds.count("attention_gather") == DEPTH
    # infer mode: the logits of the last weights, batch norm on its running statistics
    m, h = r["m"], r["h"]
    m.infer_mode(); m.forward()
    running = [m.batch_norm_stats(b) for b in h["bns"]]
    logits, _ = model_witness(g[0], g[1], r["feats"], r["labels"], r["mask"], LAYERS,
                              [m.get_parameter(p) for p in range(m.num_parameters())], DEPTH,
                              learn_temperature=learn, norm=norm, temperature=T0, training=False, bn_running=running)
    close("infer logits", m.get_tensor(h["logits"]), logits)
    r["host"].close()


def test_sigmoid_loss_and_exact_backward_on_a_directed_graph():
    g = sym_model_graph()
    r = train(g, loss="sigmoid")
    check_model(r, g, loss="sigmoid")
    r["host"].close()
    g = directed_model_graph()
    r = train(g, exact_backward=True)
    check_model(r, g)
    r["host"].close()


def test_fusion_off_is_bit_identical():
    g = sym_model_graph()
    a = train(g)
    b = train(g, fusion=False)
    for sa, sb in zip(a["steps"], b["steps"]):
        assert np.array_equal(sa["logits"].view(np.int32), sb["logits"].view(np.int32))
        assert all(np.array_equal(x.view(np.int32), y.view(np.int32)) for x, y in zip(sa["dw"], sb["dw"]))
        assert all(np.array_equal(x.view(np.int32), y.view(np.int32)) for x, y in zip(sa["w1"], sb["w1"]))
    a["host"].close(); b["host"].close()


def test_a_bf16_input_is_refused():
    """init() exits naming the op; run in a child, since the refusal ends the process"""
    code = """
import numpy as np
from roc_b200 import datasets
from roc_b200.model import Host, Model
re_, col = datasets.rmat_graph(7, 500, seed=3)
host = Host(0, 0, 1)
host.graph_from_arrays(re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32))
m = Model(host, seed=1)
x = m.create_node_tensor(16, dtype="bfloat16")
y = m.softmax_gather(x)
"""
    code = "import sys; sys.path.insert(0, %r)\n" % ROOT + code
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ))
    assert p.returncode != 0 and "softmax_gather" in p.stderr + p.stdout, (p.returncode, p.stderr[-500:])
