"""Layer normalisation on the GPU: roc_layernorm_fwd / roc_layernorm_bwd against the fp64 witness of
tests/layernorm_witness.py with bounds derived from rounding counts, over every (S, J) instantiation and the wide path,
NaN-padded columns and sentinel guard rows, special rows, repeats and SM budgets, and the refusals; then GCN, GAT,
GraphSAGE-mean and DeeperGCN with norm="layer_norm" over three Adam steps against the witness, fused and unfused.

The kernels' dispatch on H4 = ceil(H / 4), restated: H4 <= 32 runs S = the smallest power of two >= H4 lanes per row
with J = 1 float4 group per lane; 32 < H4 <= 224 runs S = 32, J = ceil(H4 / 32); H4 > 224 (H > 896) runs the wide
path.  H below reaches every one of these."""
import gc

import numpy as np
import pytest
import torch

from layernorm_witness import LN_EPS, deepergcn_witness, graph_witness, kernel_witness
from opgraph import Recorder
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K
from roc_b200.model import Host, Model, build_deepergcn, build_gat, build_gcn, build_sage_mean
from witness_gat import train_loss

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_gpu_memory():
    """The fp64 witnesses and bounds of the large cases take tens of GB; hand them back to the device after each test,
    so that later tests in the same process see the memory free (torch's caching allocator would keep it)."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
U = 2.0 ** -24          # fp32 unit roundoff
U64 = 2.0 ** -53
# rounding counts of the kernel's arithmetic, restated from include/roc_b200.h
R_DIV = 1               # mu = s / H, var = q / H, the means of gh and gh xhat: one correctly rounded division each
R_RSTD = 3              # var + eps, sqrt, 1 / sqrt: one rounding each
R_FMA = 1               # y = fma(xhat, gamma, beta); t = fma(-xhat, mb, gh - ma)
SAFETY = 1.0 + 1e-6     # for the second-order terms the first-order bounds below leave out

HS = [1, 2, 3, 4, 5, 12, 31, 41, 63, 64, 65, 127, 128, 129, 256, 257, 400, 602, 700, 800, 1023, 1024, 1025, 2051]


def shape(h):
    h4 = (h + 3) // 4
    if h4 > 224:
        return "wide"
    if h4 > 32:
        return (32, (h4 + 31) // 32)
    s = 1
    while s < h4:
        s *= 2
    return (s, 1)


def test_the_widths_reach_every_instantiation():
    assert {shape(h) for h in HS} == {(s, 1) for s in (1, 2, 4, 8, 16, 32)} | {(32, j) for j in range(2, 8)} | {"wide"}


def test_every_instantiation_runs_as_restated():
    """the kernel each width launches (torch.profiler's kernel names) is the restated dispatch's"""
    seen = {}
    for h in HS:
        x = K.padded(40, h)
        x[:, :h] = torch.randn(40, h, device="cuda")
        g, dx = K.padded(40, h), K.padded(40, h)
        g[:, :h], dx[:, :h] = torch.randn(40, h, device="cuda"), 0.0
        gm, bt = torch.ones(h, device="cuda"), torch.zeros(h, device="cuda")
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            K.layernorm_fwd(x, gm, bt, relu=True)
            K.layernorm_bwd(x, g, gm, bt, relu=False, accumulate=True, dx=dx)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if "k_ln_" in e.name and "finalize" not in e.name]
        s = shape(h)
        want = ("k_ln_fwd_wide<true>", "k_ln_bwd_wide<false, true>") if s == "wide" else \
            ("k_ln_fwd<%d, %d, true>" % s, "k_ln_bwd<%d, %d, false, true>" % s)
        assert any(want[0] in n for n in names) and any(want[1] in n for n in names), (h, want, sorted(set(names)))
        seen[s] = True
    assert len(seen) == 13


# ------------------------------------------------------------------------------------------------- the kernel ---
def _guarded(rows, h, fill):
    """a [rows][h] view into a NaN buffer of round_up4(h) columns with one sentinel row before and after"""
    buf = torch.full((rows + 2, (h + 3) // 4 * 4), float("nan"), device="cuda")
    v = buf[1:rows + 1, :h]
    if fill is not None:
        v.copy_(fill)
    return buf, v


def _untouched(buf, h, base=None):
    """the guard rows and the pad columns are still NaN (and the view equals base when it must be untouched)"""
    return bool(torch.isnan(buf[0]).all() and torch.isnan(buf[-1]).all() and torch.isnan(buf[1:-1, h:]).all())


def _inputs(rows, h, seed):
    """rows cycle through: plain normal, mean 1e4 with std 1, constant (var 0), a third +-0 values, normal scaled by 3"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((rows, h), generator=gen, device="cuda")
    kind = torch.arange(rows, device="cuda")[:, None] % 5
    x = torch.where(kind == 1, x + 1e4, x)
    x = torch.where(kind == 2, torch.full_like(x, 3.25), x)
    zeros = (torch.rand((rows, h), generator=gen, device="cuda") < 0.33) & (kind == 3)
    x = torch.where(zeros, torch.where(torch.rand((rows, h), generator=gen, device="cuda") < 0.5, 0.0, -0.0), x)
    x = torch.where(kind == 4, 3 * x, x)
    g = torch.randn((rows, h), generator=gen, device="cuda")
    gamma = torch.rand(h, generator=gen, device="cuda") + 0.5
    beta = torch.randn(h, generator=gen, device="cuda")
    return x, g, gamma, beta


def _bounds(x, g, gamma, beta, eps, relu_mask=None):
    """first-order fp64 bounds on |y - y64| and |dx - dx64| from the kernel's rounding counts, per element, and on
    dgamma / dbeta per column.  g is the (masked) output gradient."""
    x, g, gm, bt = x.double(), g.double(), gamma.double(), beta.double()
    n, h = x.shape
    mu = x.mean(1, keepdim=True)
    d = x - mu
    var = (d * d).mean(1, keepdim=True)
    s = var + eps
    rstd = 1.0 / torch.sqrt(s)
    xh = d * rstd
    # mu: H - 1 additions over the row, then the division
    e_mu = (h - 1) * U * x.abs().mean(1, keepdim=True) + R_DIV * U * mu.abs()
    e_d = e_mu + U * (d.abs() + e_mu)
    # var: the squares' errors, H fma roundings, the division
    e_q = (2 * d.abs() * e_d + e_d ** 2).mean(1, keepdim=True) + h * U * ((d.abs() + e_d) ** 2).mean(1, keepdim=True)
    e_var = e_q + R_DIV * U * var
    rel_rstd = (e_var + U * s) / (2 * s) + (R_RSTD - 1) * U
    e_xh = rstd * e_d + xh.abs() * rel_rstd + U * xh.abs()
    pre = xh * gm + bt
    e_y = SAFETY * (gm.abs() * e_xh + R_FMA * U * pre.abs()) + 1e-300
    gh = g * gm
    ma, mb = gh.mean(1, keepdim=True), (gh * xh).mean(1, keepdim=True)
    e_gh = U * gh.abs()
    e_ma = h * U * (gh.abs()).mean(1, keepdim=True) + e_gh.mean(1, keepdim=True) + R_DIV * U * ma.abs()
    e_mb = ((gh.abs() + e_gh) * e_xh + e_gh * xh.abs()).mean(1, keepdim=True) + \
        (h + 1) * U * (gh * xh).abs().mean(1, keepdim=True) + R_DIV * U * mb.abs()
    t = gh - ma - xh * mb
    e_t = e_gh + e_ma + U * (gh - ma).abs() + e_xh * mb.abs() + xh.abs() * e_mb + R_FMA * U * t.abs()
    dx = rstd * t
    e_dx = SAFETY * (rstd * e_t + dx.abs() * rel_rstd + U * dx.abs()) + 1e-300
    e_dgamma = SAFETY * ((g.abs() * e_xh).sum(0) + U * (g * xh).sum(0).abs() + 4 * n * U64 * (g * xh).abs().sum(0))
    e_dbeta = SAFETY * (U * g.sum(0).abs() + 4 * n * U64 * g.abs().sum(0)) + 1e-300
    return dict(y=e_y, dx=e_dx, dgamma=e_dgamma + 1e-300, dbeta=e_dbeta)


WORST = {}


def _ratio(what, got, want, bound):
    r = float(((got.double() - want).abs() / bound).max()) if got.numel() else 0.0
    WORST[what] = max(WORST.get(what, 0.0), r)
    return r


def _check_case(rows, h, seed, modes=((False, False), (True, False), (False, True), (True, True))):
    what = "rows=%d H=%d" % (rows, h)
    x0, g0, gamma, beta = _inputs(rows, h, seed)
    xb, x = _guarded(rows, h, x0)
    gb, g = _guarded(rows, h, g0)
    for relu in (False, True):
        yb, y = _guarded(rows, h, None)
        K.layernorm_fwd(x, gamma, beta, relu=relu, eps=LN_EPS, out=y)
        assert _untouched(yb, h), what
        mask = (y > 0) if relu else None      # the product's own relu test, which its backward recomputes
        gm = torch.where(mask, g0, 0.0) if relu else g0
        w = kernel_witness(x0, gm, gamma, beta, LN_EPS, relu=False)
        b = _bounds(x0, gm, gamma, beta, LN_EPS)
        want = torch.relu(w["y"]) if relu else w["y"]
        assert _ratio("y", y, want, b["y"]) <= 1.0, (what, relu)
        y2 = K.layernorm_fwd(x, gamma, beta, relu=relu, eps=LN_EPS)
        assert torch.equal(y.contiguous().view(torch.int32), y2[:, :h].contiguous().view(torch.int32)), what
        for r, acc in modes:
            if r != relu:
                continue
            base = torch.randn_like(x0) if acc else None
            db, dx = _guarded(rows, h, base)
            dx, dgam, dbet = K.layernorm_bwd(x, g, gamma, beta, relu=relu, eps=LN_EPS, dx=dx, accumulate=acc)
            assert _untouched(db, h), (what, relu, acc)
            want = w["dx"] + (base.double() if acc else 0)
            bnd = b["dx"] + (U * want.abs() if acc else 0)
            assert _ratio("dx", dx, want, bnd) <= 1.0, (what, relu, acc)
            assert _ratio("dgamma", dgam, w["dgamma"], b["dgamma"]) <= 1.0, (what, relu)
            assert _ratio("dbeta", dbet, w["dbeta"], b["dbeta"]) <= 1.0, (what, relu)
            dx2 = K.layernorm_bwd(x, g, gamma, beta, relu=relu, eps=LN_EPS, dx=_guarded(rows, h, base)[1],
                                  accumulate=acc)[0]
            assert torch.equal(dx.contiguous().view(torch.int32), dx2.contiguous().view(torch.int32)), what
            _, dg3, db3 = K.layernorm_bwd(x, g, gamma, beta, relu=relu, eps=LN_EPS, need_dx=False)
            assert torch.equal(dg3.view(torch.int32), dgam.view(torch.int32)), what
            assert torch.equal(db3.view(torch.int32), dbet.view(torch.int32)), what
    assert torch.isnan(xb[0]).all() and torch.isnan(gb[-1]).all()


@pytest.mark.parametrize("h", HS)
@pytest.mark.parametrize("rows", [1, 2, 33, 70001])
def test_kernel_matches_fp64(rows, h):
    _check_case(rows, h, seed=rows * 7 + h)


@pytest.mark.parametrize("h", [41, 64, 256])
def test_kernel_over_many_grid_passes(h):
    _check_case(1000003, h, seed=h, modes=((False, True), (True, False)))


def test_report_worst_ratios():
    """the worst |got - fp64| / bound over the cases above (printed with -s)"""
    print("worst ratios:", {k: round(v, 4) for k, v in sorted(WORST.items())})
    assert all(v <= 1.0 for v in WORST.values())


@pytest.mark.parametrize("h", [1, 5, 64, 2051])
def test_zero_rows(h):
    """rows = 0 writes nothing but zero dgamma / dbeta (called with real pointers: an empty torch view has none)"""
    ld = (h + 3) // 4 * 4
    buf = torch.full((4, ld), float("nan"), device="cuda")
    gm, bt = torch.ones(h, device="cuda"), torch.zeros(h, device="cuda")
    dg, db = torch.full((h,), 7.0, device="cuda"), torch.full((h,), 7.0, device="cuda")
    ws_bytes = _lib.lib.roc_layernorm_workspace_bytes(0, h)
    ws = torch.empty(ws_bytes, device="cuda", dtype=torch.uint8)
    p = buf.data_ptr()
    assert _lib.lib.roc_layernorm_fwd(0, h, p, ld, gm.data_ptr(), bt.data_ptr(), 1e-5, 1, p, ld, None) == _lib.ROC_OK
    assert _lib.lib.roc_layernorm_bwd(0, h, p, ld, p, ld, 1, gm.data_ptr(), bt.data_ptr(), 1e-5, dg.data_ptr(),
                                      db.data_ptr(), p, ld, 1, ws.data_ptr(), ws_bytes, None) == _lib.ROC_OK
    torch.cuda.synchronize()
    assert not dg.any() and not db.any() and torch.isnan(buf).all()


@pytest.mark.parametrize("h", [1, 3, 64, 300, 1025])
def test_special_rows(h):
    """a constant row (var 0) and a row of -0 give y = beta exactly; H = 1 gives y = beta and dx = 0 on every row; a
    NaN reaches only its own row's y and dx"""
    rows = 40
    x = torch.randn(rows, h, device="cuda")
    x[4] = 0.5                                  # 0.5 H / H is exact: mu = 0.5, var = 0
    x[7] = -0.0
    x[9, h // 2] = float("nan")
    gm, bt = torch.rand(h, device="cuda") + 0.5, torch.randn(h, device="cuda")
    xp, gp = K.padded(rows, h), K.padded(rows, h)
    xp[:, :h], gp[:, :h] = x, torch.randn(rows, h, device="cuda")
    y = K.layernorm_fwd(xp, gm, bt)[:, :h]
    dx = K.layernorm_bwd(xp, gp, gm, bt)[0][:, :h]
    assert torch.equal(y[4], bt) and torch.equal(y[7], bt)
    fin = ~torch.isnan(x).any(1)
    if h == 1:
        assert torch.equal(y[fin, 0], bt.expand(int(fin.sum()))) and not dx[fin].any()
    assert torch.isnan(y[9]).all() and torch.isnan(dx[9]).all()
    assert torch.isfinite(y[fin]).all() and torch.isfinite(dx[fin]).all()


@pytest.mark.parametrize("h", [5, 64, 129, 602, 2051])
def test_repeats_and_sm_budgets_are_byte_identical(h):
    rows = 50001
    x0, g0, gamma, beta = _inputs(rows, h, seed=5)
    x, g = K.padded(rows, h), K.padded(rows, h)
    x[:, :h], g[:, :h] = x0, g0

    def run():
        y = K.layernorm_fwd(x, gamma, beta, relu=True)
        dx, dg, db = K.layernorm_bwd(x, g, gamma, beta, relu=True)
        return [t.contiguous().view(torch.int32).clone() for t in (y[:, :h], dx[:, :h], dg, db)]

    ref = run()
    assert all(torch.equal(a, b) for a, b in zip(ref, run()))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    prev = _lib.lib.roc_set_sm_reserve(0)
    try:
        for reserve in (sms - 8, sms // 2 + (1 - (sms - sms // 2) % 2)):   # 8 SMs left, and an odd count
            _lib.lib.roc_set_sm_reserve(int(reserve))
            assert all(torch.equal(a, b) for a, b in zip(ref, run())), reserve
    finally:
        _lib.lib.roc_set_sm_reserve(prev)


def test_kernel_refuses_bad_arguments():
    rows, h = 8, 6
    x, y, g, dx = K.padded(rows, h), K.padded(rows, h), K.padded(rows, h), K.padded(rows, h)
    gm, bt = torch.ones(h, device="cuda"), torch.zeros(h, device="cuda")
    dgm, dbt = torch.empty(h, device="cuda"), torch.empty(h, device="cuda")
    wsb = _lib.lib.roc_layernorm_workspace_bytes(rows, h)
    ws = torch.empty(wsb + 16, device="cuda", dtype=torch.uint8)
    p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    ok = dict(rows=rows, H=h, x=x, ldX=8, g=g, ldG=8, gm=gm, bt=bt, eps=1e-5, y=y, ldY=8, dgm=dgm, dbt=dbt, dx=dx,
              ldDX=8, ws=ws, wsb=wsb, wsoff=0)

    def fwd(**kw):
        a = dict(ok, **kw)
        return _lib.lib.roc_layernorm_fwd(a["rows"], a["H"], p(a["x"]) and p(a["x"]) + a.get("xoff", 0), a["ldX"],
                                          p(a["gm"]), p(a["bt"]), a["eps"], 0, p(a["y"]), a["ldY"], None)

    def bwd(**kw):
        a = dict(ok, **kw)
        return _lib.lib.roc_layernorm_bwd(a["rows"], a["H"], p(a["x"]), a["ldX"], p(a["g"]) and p(a["g"]) +
                                          a.get("goff", 0), a["ldG"], 0, p(a["gm"]), p(a["bt"]), a["eps"], p(a["dgm"]),
                                          p(a["dbt"]), p(a["dx"]), a["ldDX"], 0, p(a["ws"]) and p(a["ws"]) + a["wsoff"],
                                          a["wsb"], None)

    assert fwd() == _lib.ROC_OK and bwd() == _lib.ROC_OK and bwd(dx=None) == _lib.ROC_OK
    assert fwd(rows=0) == _lib.ROC_OK and bwd(rows=0) == _lib.ROC_OK
    inf = float("inf")
    for bad in (dict(x=None), dict(gm=None), dict(bt=None), dict(y=None), dict(rows=-1), dict(H=0), dict(H=-3),
                dict(ldX=5), dict(ldY=6), dict(ldX=10), dict(ldY=9), dict(xoff=4), dict(eps=-1e-5), dict(eps=inf),
                dict(eps=float("nan"))):
        assert fwd(**bad) == _lib.ROC_ERR_INVALID, bad
    for bad in (dict(x=None), dict(g=None), dict(gm=None), dict(bt=None), dict(dgm=None), dict(dbt=None),
                dict(ws=None), dict(rows=-1), dict(H=0), dict(ldX=5), dict(ldG=5), dict(ldDX=5), dict(ldG=10),
                dict(ldDX=9), dict(goff=8), dict(eps=-1.0), dict(eps=inf), dict(eps=float("nan")), dict(wsb=wsb - 1),
                dict(wsoff=8)):
        assert bwd(**bad) == _lib.ROC_ERR_INVALID, bad
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------- the models ---
def sym_graph():
    re_, col = datasets.rmat_graph(9, 2500, seed=3)
    return re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


def directed_graph():
    re_, col = datasets.rmat_graph(9, 2500, seed=4, directed=True)
    return re_.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


def bce_loss(logits, labels, mask):
    train = torch.from_numpy(mask == _lib.MASK_TRAIN)
    y = torch.from_numpy(np.asarray(labels, dtype=np.float64))
    return torch.nn.functional.binary_cross_entropy_with_logits(logits[train], y[train], reduction="sum")


MODELS = {   # at dropout 0
    "gcn": lambda ir, **kw: build_gcn(ir, [24, 16, 16, 12], 0.0, **kw),
    "gat": lambda ir, **kw: build_gat(ir, [24, 16, 12], 0.0, heads=2, scores="per_head", activation="elu", **kw),
    "sage_mean": lambda ir, **kw: build_sage_mean(ir, [24, 16, 16, 12], 0.0, **kw),
}
DGCN = [24, 16, 12]


def train(build, graph, fuse=True, steps=3, loss="softmax", **kw):
    row_end, col = graph
    n = row_end.shape[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(row_end, col)
    m = Model(host, seed=1)
    m.set_fusion(fuse)
    ir = Recorder(m)
    h = build(ir, norm="layer_norm", dropout_rate=0.0, loss=loss, **kw) if build is build_dgcn else \
        build(ir, norm="layer_norm", **kw)
    gen = datasets.multilabel_node_data if loss == "sigmoid" else datasets.node_data
    feats, labels, mask = (t.numpy() for t in gen(n, 24, 12, seed=5))
    (m.set_multilabels if loss == "sigmoid" else m.set_labels)(h["label"], labels)
    m.set_tensor(h["input"], feats)
    m.set_tensor(h["mask"], mask.astype(np.int32))
    out = dict(ir=ir, h=h, feats=feats, labels=labels, mask=mask, info=m.op_info(), steps=[], graph=graph)
    for _ in range(steps):
        st = dict(w0=[m.get_parameter(p) for p in range(m.num_parameters())])
        m.train_mode(); m.zero_gradients(); m.forward()
        st["logits"] = m.get_tensor(h["logits"])
        m.backward()
        st["dw"] = [m.get_parameter(p, "grad") for p in range(m.num_parameters())]
        m.update()
        st["w1"] = [m.get_parameter(p) for p in range(m.num_parameters())]
        out["steps"].append(st)
    m.infer_mode(); m.forward()
    out["infer_logits"] = m.get_tensor(h["logits"])
    host.close()
    return out


def build_dgcn(ir, norm, dropout_rate, loss, **kw):
    return build_deepergcn(ir, DGCN, dropout_rate, 3, norm=norm, loss=loss, temperature=0.9, **kw)


def close(name, got, want, rtol=2e-4, atol_scale=2e-5):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    bound = rtol * np.abs(want) + atol_scale * np.abs(want).max() + 1e-30
    r = float((np.abs(got - want) / bound).max())
    assert r <= 1.0, (name, r)


def adam(w0, grads, lr=0.01, wd=0.05, b1=0.9, b2=0.999, eps=1e-8):
    """each step's parameters from w0 under the engine's Adam (weight decay added to the gradient)"""
    w, m, v, out = np.asarray(w0, dtype=np.float64), 0.0, 0.0, []
    for k, g in enumerate(grads, 1):
        g = g + wd * w
        m, v = b1 * m + (1 - b1) * g, b2 * v + (1 - b2) * g * g
        w = w - lr * np.sqrt(1 - b2 ** k) / (1 - b1 ** k) * m / (np.sqrt(v) + eps)
        out.append(w)
    return out


def check(run, witness):
    """each step's logits and every parameter's gradient against the witness, and every parameter (gamma / beta
    included) after each step against Adam on the witness's gradients"""
    wgrads = []
    for k, st in enumerate(run["steps"]):
        logits, dw = witness(st["w0"])
        close("step %d logits" % k, st["logits"], logits)
        for p, (a, b) in enumerate(zip(st["dw"], dw)):
            close("step %d dW%d" % (k, p), a, b, rtol=1e-3, atol_scale=1e-4)
        wgrads.append(dw)
    for p in range(len(run["steps"][0]["w0"])):
        want = adam(run["steps"][0]["w0"][p], [g[p] for g in wgrads])
        for k, st in enumerate(run["steps"]):
            assert np.abs(st["w1"][p] - want[k]).max() <= 1e-3 * 0.01 + 1e-5 * np.abs(want[k]).max(), (k, p)


def identical(a, b):
    for sa, sb in zip(a["steps"], b["steps"]):
        assert np.array_equal(sa["logits"].view(np.int32), sb["logits"].view(np.int32))
        for k in ("dw", "w1"):
            for x, y in zip(sa[k], sb[k]):
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), k
    assert np.array_equal(a["infer_logits"].view(np.int32), b["infer_logits"].view(np.int32))


def check_fusion(fused, unfused):
    """op_info: kind batch_norm, each relu after a layer_norm fused into it and left apart with fusion off"""
    BN = "batch_norm"
    for nd in fused["ir"].nodes:
        if nd["kind"] != "layer_norm":
            continue
        assert fused["info"][nd["layer"]]["kind"] == BN and unfused["info"][nd["layer"]]["kind"] == BN
        relu = [r for r in fused["ir"].nodes if r["ins"] == [nd["out"]]]
        if len(relu) == 1 and relu[0]["kind"] == "relu":
            assert fused["info"][relu[0]["layer"]]["fusedInto"] == nd["layer"]
            assert fused["info"][nd["layer"]]["fwdOut"] == relu[0]["out"]
        else:
            assert fused["info"][nd["layer"]]["fwdOut"] == -1
        assert unfused["info"][nd["layer"]]["fwdOut"] == -1


@pytest.mark.parametrize("name", list(MODELS))
def test_builders_with_layer_norm_match_the_witness(name):
    g = sym_graph()
    fused, unfused = train(MODELS[name], g, True), train(MODELS[name], g, False)
    ir = fused["ir"]
    check(fused, lambda w: (lambda r: (r["logits"], r["dW"]))(
        graph_witness(ir, g, fused["feats"], fused["labels"], fused["mask"], w)))
    identical(fused, unfused)
    identical(fused, train(MODELS[name], g, True))
    check_fusion(fused, unfused)
    if name == "gat":       # the elu after the norm is not a relu: nothing fused
        assert all(fused["info"][nd["layer"]]["fwdOut"] == -1 for nd in ir.nodes if nd["kind"] == "layer_norm")
    # infer mode runs the train-mode forward: at dropout 0 the logits are its bits, and match the witness
    ev = graph_witness(ir, g, fused["feats"], fused["labels"], fused["mask"], fused["steps"][-1]["w1"],
                       training=False)
    close("infer logits", fused["infer_logits"], ev["logits"])
    for nd in ir.nodes:   # gamma 1 and beta 0 at the start, shape (1, H)
        if nd["kind"] == "layer_norm":
            w = fused["steps"][0]["w0"]
            assert np.all(w[nd["attrs"]["gamma"]] == 1) and np.all(w[nd["attrs"]["beta"]] == 0)
            assert w[nd["attrs"]["gamma"]].shape == (1, ir.width[nd["out"]])


def test_infer_logits_are_the_train_forward_bits():
    g = sym_graph()
    run = train(MODELS["gcn"], g, True, steps=0)
    host = Host(0, 0, 1)
    host.graph_from_arrays(*g)
    m = Model(host, seed=1)
    h = MODELS["gcn"](Recorder(m), norm="layer_norm")
    m.set_labels(h["label"], run["labels"])
    m.set_tensor(h["input"], run["feats"])
    m.set_tensor(h["mask"], run["mask"].astype(np.int32))
    m.train_mode(); m.forward()
    t = m.get_tensor(h["logits"])
    host.close()
    assert np.array_equal(t.view(np.int32), run["infer_logits"].view(np.int32))


@pytest.mark.parametrize("learn", [True, False])
def test_deepergcn_with_layer_norm_matches_the_witness(learn):
    g = directed_graph()
    kw = dict(learn_temperature=learn, exact_backward=True)
    fused = train(build_dgcn, g, True, loss="sigmoid", **kw)
    unfused = train(build_dgcn, g, False, loss="sigmoid", **kw)
    re_, col = g
    check(fused, lambda w: deepergcn_witness(re_, col, fused["feats"], fused["labels"], fused["mask"], DGCN, w, 3,
                                             learn_temperature=learn, temperature=0.9, loss_fn=bce_loss))
    identical(fused, unfused)
    check_fusion(fused, unfused)
    assert len(fused["h"]["bns"]) == 3 + 2 + 1
