"""GPU suite: the bf16 forms of the max / min, edge-weighted and attention ScatterGathers (the roc_sg_*_bf16 calls)
against their fp32 calls on the widened rows, bit for bit, and the relu whose output is stored in bf16.

Each case runs the fp32 call on roc_bf16_to_f32 of the bf16 rows (16-byte aligned, a leading dimension that is a
multiple of 4) and the bf16 call on the rows themselves, into Guarded outputs whose sentinels must survive, on the
long-lived plans of the fp32 matrices: sg_matrix.graphs() for max / min and the attention gathers over the same CSR,
wgraphs() for the weighted sum and the edge dot, xgraphs() for the exact attention backward.  Widths: both ends of
every rung of the row-shape table on float4 rows, column blocks past the widest row, and every width of
sg_matrix.SCALAR.  The bf16 rows hold NaN in their pad columns; the max / min inputs also hold NaN values.  Each
call's launch list is the fp32 call's with 16 added to the reduction of its main kernels.  Then R-MAT scale 22
(config 2's graph) at H = 64 and 41, and a last test that every new instantiation ran."""
import numpy as np
import pytest
import torch

import sg_matrix as sm
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K

pytestmark = pytest.mark.gpu
BF = _lib.SG_RED_BF16
NEW = (sm.MAX, sm.MIN, sm.ATTN, sm.ADST, sm.ASRC, sm.WSUM, sm.EDOT)   # the reductions that have a bf16 form
SEEN = set()


def vec_widths(q4):
    """float4-row widths at both ends of every rung up to a widest row of q4 T-columns, and one column block past it"""
    out, lo = [], 1
    for qc, _, _ in sm.RUNGS:
        if qc <= q4:
            out += [lo, 4 * qc]
            lo = 4 * qc + 1
    return out + [4 * q4 + 8]


def bf16_rows(rng, rows, h, nan=False):
    """bf16 [rows][h] of both signs and many magnitudes, in rows of round_up(h, 8) + 8 elements whose pad columns hold
    NaN; with nan, some values are NaN too."""
    ld = (h + 7) // 8 * 8 + 8
    buf = torch.full((rows, ld), float("nan"), dtype=torch.bfloat16, device=sm.DEV)
    v = rng.standard_normal((rows, h)) * np.exp2(rng.randint(-6, 7, size=(rows, h)))
    if nan:
        v[rng.rand(rows, h) < 0.05] = np.nan
    buf[:, :h] = torch.from_numpy(v.astype(np.float32)).to(sm.DEV).to(torch.bfloat16)
    return buf[:, :h]


def widened(x):
    """the fp32 copy of bf16 rows, in 16-byte aligned rows of round_up(h, 4) + 4 floats"""
    h = x.shape[1]
    out = torch.full((x.shape[0], sm.r4(h) + 4), float("nan"), device=sm.DEV)[:, :h]
    return K.bf16_to_f32(x, out=out)


def bf16_form(want):
    """an fp32 call's launch list as its bf16 form reports it: 16 + r on the main kernels of the reductions r above"""
    return [(k, r + BF if k == "main" and r in NEW else r, v, ln, nch, g) for k, r, v, ln, nch, g in want]


def same(got, want, what):
    for a, b in zip(got, want):
        a.check_guards(what)
        assert np.array_equal(a.bits(), b.bits()), "%s: bits differ from the fp32 call on the widened rows" % what


def edge_buf(g, rng, accumulate):
    """[E + 1] edge outputs (the last one never written) between two sentinel guards; with accumulate, the first E
    hold random values to add to"""
    b = torch.full((g.E + 3,), sm.SENT_F, device=sm.DEV)
    if accumulate and g.E:
        b[1:g.E + 1] = torch.from_numpy(rng.standard_normal(g.E).astype(np.float32)).to(sm.DEV)
    return b


def stats_buf(rows, heads):
    return sm.Guarded(rows, 2 * heads, 2 * heads + 4, 2 * heads)


# ---------------------------------------------------------------------------------------------------- max / min ---
def run_minmax(vec, widths):
    for g in sm.graphs().values():
        rng = np.random.RandomState(g.nloc + len(widths))
        for h in widths:
            x = bf16_rows(rng, g.n, h, nan=True)
            xw = widened(x)
            for aggr, red in ((_lib.AGGR_MAX, sm.MAX), (_lib.AGGR_MIN, sm.MIN)):
                what = "%s %s H=%d %s" % (g.name, "max" if red == sm.MAX else "min", h, "vec" if vec else "scalar")
                outs = []
                for form in (0, 1):
                    o, a = sm.guarded(g.nloc, h, vec), sm.guarded(g.nloc, h, vec, index=True)
                    (g.plan.minmax_forward_bf16 if form else g.plan.minmax_forward)(x if form else xw, aggr,
                                                                                    out=o.view, arg=a.view)
                    want = sm.planned(g.sched, red, vec, h)
                    sm.launches(what, bf16_form(want) if form else want, SEEN)
                    outs.append((o, a))
                torch.cuda.synchronize()
                same(outs[1], outs[0], what)


@pytest.mark.parametrize("vec", [True, False], ids=["vec", "scalar"])
def test_minmax_bf16(vec):
    run_minmax(vec, vec_widths(sm.REDS[sm.MAX].q4) if vec else sm.SCALAR)


# --------------------------------------------------------------------------------- weighted sum and edge dot ---
def run_weighted(vec, widths):
    for g in sm.wgraphs().values():
        rng = np.random.RandomState(3 * g.nloc + len(widths))
        w = torch.from_numpy(rng.standard_normal(max(g.E, 1)).astype(np.float32)).to(sm.DEV)
        for h in widths:
            x = bf16_rows(rng, g.n, h)
            xw = widened(x)
            what = "%s H=%d %s" % (g.name, h, "vec" if vec else "scalar")
            outs = []
            for form in (0, 1):
                o = sm.guarded(g.nloc, h, vec)
                (g.plan.weighted_forward_bf16 if form else g.plan.weighted_forward)(x if form else xw, w, out=o.view)
                want = sm.planned(g.sched, sm.WSUM, vec, h)
                sm.launches(what + " weighted", bf16_form(want) if form else want, SEEN)
                outs.append(o)
            gd = sm.dev_in(rng.standard_normal((g.nloc, h)).astype(np.float32), vec)
            for acc in (False, True):
                dws = []
                for form in (0, 1):
                    dw = edge_buf(g, np.random.RandomState(h), acc)
                    (g.plan.edge_dot_bf16 if form else g.plan.edge_dot)(gd, x if form else xw, dw=dw[1:-1],
                                                                        accumulate=acc)
                    want = sm.planned(g.sched, sm.EDOT, vec, h)
                    sm.launches(what + " edge dot", bf16_form(want) if form else want, SEEN)
                    dws.append(dw)
                torch.cuda.synchronize()
                a, b = (d.cpu().view(torch.int32).numpy() for d in dws)
                sent = np.float32(sm.SENT_F).view(np.int32)
                assert a[0] == sent and a[-1] == sent, what + " edge dot: a guard changed"
                assert np.array_equal(a, b), "%s edge dot accumulate=%d: bits differ" % (what, acc)
            torch.cuda.synchronize()
            same(outs[1:], outs[:1], what + " weighted")


@pytest.mark.parametrize("vec", [True, False], ids=["vec", "scalar"])
def test_weighted_and_edge_dot_bf16(vec):
    run_weighted(vec, vec_widths(sm.REDS[sm.WSUM].q4) if vec else sm.SCALAR)


# --------------------------------------------------------------------------------------------------- attention ---
ATTN_V = [w for w in vec_widths(sm.REDS[sm.ATTN].q4) if w <= 512]      # the attention gathers take H <= 512
ATTN_S = [w for w in sm.SCALAR if w <= 256]                            # (256 on scalar rows)


def attn_inputs(rng, g, h, heads, vec):
    x = bf16_rows(rng, g.n, h)
    s = sm.scores_dev(rng.standard_normal((g.n, 2 * heads)).astype(np.float32))
    gd = sm.dev_in(rng.standard_normal((g.n, h)).astype(np.float32), vec)
    return x, widened(x), s, gd


def attn_forward(g, plan, x, s, heads, h, vec, rows, self_base, form):
    o, st = sm.guarded(rows, h, vec), stats_buf(rows, heads)
    (plan.attn_forward_bf16 if form else plan.attn_forward)(x, s, heads, sm.SLOPE, self_base=self_base, out=o.view,
                                                            stats=st.view)
    return o, st


def run_attn(vec, widths):
    for g in sm.graphs().values():
        for h in widths:
            for heads in sm.valid_heads(h):
                rng = np.random.RandomState(h * 13 + heads + g.nloc)
                x, xw, s, gd = attn_inputs(rng, g, h, heads, vec)
                what = "%s attention H=%d heads=%d %s" % (g.name, h, heads, "vec" if vec else "scalar")
                fw = []
                for form in (0, 1):
                    fw.append(attn_forward(g, g.plan, x if form else xw, s, heads, h, vec, g.nloc, g.self_base, form))
                    want = sm.attn_forward(g.sched, vec, h, heads)
                    sm.launches(what + " forward", bf16_form(want) if form else want, SEEN)
                torch.cuda.synchronize()
                same(fw[1], fw[0], what + " forward")
                if g.full is None:
                    o_all, st_all = fw[0][0].view, fw[0][1].view
                else:
                    o_all, st_all = (b.view for b in attn_forward(g.full, g.full.plan, xw, s, heads, h, vec,
                                                                  g.full.n, 0, 0))
                n = max(g.id_end, g.self_base + g.nloc)
                bw = []
                for form in (0, 1):
                    ig, sg = sm.guarded(g.nloc, h, vec), stats_buf(g.nloc, heads)
                    (g.plan.attn_backward_bf16 if form else g.plan.attn_backward)(
                        x if form else xw, s, o_all, st_all, gd, heads, sm.SLOPE, self_base=g.self_base,
                        in_grad=ig.view, score_grad=sg.view)
                    want = sm.attn_backward(g.sched, g.sched, vec, h, n)
                    sm.launches(what + " backward", bf16_form(want) if form else want, SEEN)
                    bw.append((ig, sg))
                torch.cuda.synchronize()
                same(bw[1], bw[0], what + " backward")


@pytest.mark.parametrize("vec", [True, False], ids=["vec", "scalar"])
def test_attn_bf16(vec):
    run_attn(vec, ATTN_V if vec else ATTN_S)


def run_attn_exact(vec, widths):
    for g in sm.xgraphs().values():
        for h in widths:
            for heads in sm.valid_heads(h):
                rng = np.random.RandomState(h * 7 + heads + g.n)
                x, xw, s, gd = attn_inputs(rng, g, h, heads, vec)
                od, std = (b.view for b in attn_forward(g, g.plan, xw, s, heads, h, vec, g.n, 0, 0))
                what = "%s exact attention H=%d heads=%d %s" % (g.name, h, heads, "vec" if vec else "scalar")
                bw = []
                for form in (0, 1):
                    ig, sg = sm.guarded(g.n, h, vec), stats_buf(g.n, heads)
                    (g.tr.attn_backward_bf16 if form else g.tr.attn_backward)(
                        g.plan, x if form else xw, s, od, std, gd, heads, sm.SLOPE, in_grad=ig.view,
                        score_grad=sg.view)
                    want = sm.attn_backward(g.sched, g.sched_t, vec, h, g.n)
                    sm.launches(what, bf16_form(want) if form else want, SEEN)
                    bw.append((ig, sg))
                torch.cuda.synchronize()
                same(bw[1], bw[0], what)


@pytest.mark.parametrize("vec", [True, False], ids=["vec", "scalar"])
def test_attn_exact_bf16(vec):
    run_attn_exact(vec, ATTN_V if vec else ATTN_S)


# ------------------------------------------------------------------------------------------------- refusals ---
def test_bf16_forms_refuse_bad_layouts():
    """in not 16-byte aligned or ldIn not a multiple of 8: ROC_ERR_INVALID from every bf16 form."""
    g = sm.wgraphs()["tiny"]
    h = 12
    good = bf16_rows(np.random.RandomState(1), g.n, h)
    bad_ld = torch.zeros((g.n, 20), dtype=torch.bfloat16, device=sm.DEV)[:, :h]
    shifted = torch.zeros((g.n * 16 + 4,), dtype=torch.bfloat16, device=sm.DEV)[4:].view(g.n, 16)[:, :h]
    w = torch.ones(max(g.E, 1), device=sm.DEV)
    s = torch.zeros((g.n, 2), device=sm.DEV)
    gd = K.padded(g.n, h)
    od, std = g.plan.attn_forward(widened(good), s)
    calls = [lambda x: g.plan.minmax_forward_bf16(x, _lib.AGGR_MAX),
             lambda x: g.plan.weighted_forward_bf16(x, w),
             lambda x: g.plan.edge_dot_bf16(gd, x),
             lambda x: g.plan.attn_forward_bf16(x, s),
             lambda x: g.plan.attn_backward_bf16(x, s, od, std, gd),
             lambda x: g.tr.attn_backward_bf16(g.plan, x, s, od, std, gd)]
    for call in calls:
        for bad in (bad_ld, shifted):
            with pytest.raises(_lib.RocError):
                call(bad)
        call(good)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------- full size ---
@pytest.mark.parametrize("h", [64, 41])
def test_bf16_forms_rmat22(h):
    """Config 2's graph (R-MAT scale 22) at its two aggregation widths: every bf16 form, one head."""
    row_end, col = datasets.rmat_graph(22, 1 << 25, seed=1, device=sm.DEV)
    torch.cuda.synchronize()
    n = row_end.shape[0]
    plan = K.SgPlan(0, n - 1, 0, row_end, col)
    gen = torch.Generator(device=sm.DEV)
    gen.manual_seed(h)
    ld = (h + 7) // 8 * 8
    x = torch.randn((n, ld), device=sm.DEV, generator=gen).to(torch.bfloat16)[:, :h]
    xw = widened(x)
    e = plan.num_edges()
    w = torch.rand(e, device=sm.DEV, generator=gen)
    gy = torch.randn((n, sm.r4(h)), device=sm.DEV, generator=gen)[:, :h]
    s = torch.randn((n, 2), device=sm.DEV, generator=gen) * 0.5

    def eq(a, b, what):
        torch.cuda.synchronize()
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "R-MAT-22 H=%d %s" % (h, what)

    for aggr in (_lib.AGGR_MAX, _lib.AGGR_MIN):
        (o0, a0), (o1, a1) = plan.minmax_forward(xw, aggr), plan.minmax_forward_bf16(x, aggr)
        eq(o1, o0, "minmax out")
        eq(a1, a0, "minmax arg")
        del o0, a0, o1, a1
    eq(plan.weighted_forward_bf16(x, w), plan.weighted_forward(xw, w), "weighted forward")
    eq(plan.edge_dot_bf16(gy, x), plan.edge_dot(gy, xw), "edge dot")
    (o0, st0), (o1, st1) = plan.attn_forward(xw, s), plan.attn_forward_bf16(x, s)
    eq(o1, o0, "attention out")
    eq(st1, st0, "attention stats")
    del o1, st1
    (i0, sg0), (i1, sg1) = plan.attn_backward(xw, s, o0, st0, gy), plan.attn_backward_bf16(x, s, o0, st0, gy)
    eq(i1, i0, "attention input gradient")
    eq(sg1, sg0, "attention score gradient")
    plan.close()


# --------------------------------------------------------------------------------------------- relu to bf16 ---
def test_relu_y_bf16():
    """fwd stores f32_to_bf16 of roc_activation_fwd's bits; bwd is roc_activation_bwd on the widened y, overwriting and
    accumulating; a value at most 2^-134 rounds to +0 and masks its gradient; any mode but relu is refused."""
    rng = np.random.RandomState(5)
    for rows, h in ((1000, 37), (257, 64), (3, 1)):
        v = rng.standard_normal((rows, h)) * np.exp2(rng.randint(-20, 20, size=(rows, h)))
        flat = v.reshape(-1)
        flat[:8] = [np.nan, -np.nan, 0.0, -0.0, 2.0 ** -134, 2.0 ** -133.5, -(2.0 ** -134), np.inf][:flat.shape[0]]
        x = sm.dev_in(v.astype(np.float32), True)
        y = K.activation_fwd_y_bf16(x)
        want = K.f32_to_bf16(K.activation_fwd(x, _lib.AC_MODE_RELU))
        torch.cuda.synchronize()
        assert torch.equal(y.view(torch.int16), want.view(torch.int16)), "relu fwd H=%d" % h
        if rows * h >= 5:
            assert float(y.reshape(-1)[4]) == 0.0 and float(y.reshape(-1)[5]) > 0.0
        dy = sm.dev_in(rng.standard_normal((rows, h)).astype(np.float32), False)
        yw = widened(y)
        got = K.activation_bwd_y_bf16(y, dy)
        ref = K.activation_bwd(yw, dy, _lib.AC_MODE_RELU)
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), "relu bwd H=%d" % h
        base = torch.randn((rows, h), device=sm.DEV)
        acc, acc_ref = base.clone(), base.clone()
        K.activation_bwd_y_bf16(y, dy, dx=acc)
        K.activation_bwd(yw, dy, _lib.AC_MODE_RELU, dx=acc_ref)
        torch.cuda.synchronize()
        assert torch.equal(acc.view(torch.int32), acc_ref.view(torch.int32)), "relu bwd accumulate H=%d" % h
    x = K.padded(4, 8)
    for f in (lambda: K.activation_fwd_y_bf16(x, _lib.AC_MODE_SIGMOID),
              lambda: K.activation_bwd_y_bf16(K.bf16_padded(4, 8), x, _lib.AC_MODE_SIGMOID)):
        with pytest.raises(_lib.RocError):
            f()


def test_bf16_forms_ran_every_instantiation():
    """After the matrices: every main-kernel instantiation of every bf16 form, on both paths at every rung."""
    if not SEEN:
        pytest.skip("run with the matrices")
    want = {(k, r + BF, v, ln, nch) for k, r, v, ln, nch in sm.every_instantiation(NEW) if k == "main"}
    assert want <= SEEN, sorted(want - SEEN)
