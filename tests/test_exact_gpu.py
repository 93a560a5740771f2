"""The exact backwards of the sum, max / min and attention aggregations over the transpose (include/roc_b200.h,
roc_sg_transpose_sum_backward, roc_sg_transpose_minmax_backward, roc_sg_attn_backward_exact) on the GPU.

Every whole graph of the ScatterGather matrix runs, with the weighted tests' directed multigraph and hub, and a
fan-out graph whose one source feeds 3,000 rows: its transposed row needs the big-row fix-up.  Data are multiples of
1/16 in [-8, 8], so the sums, their norm / relu epilogue and the max / min backward are exact in fp32 and compared bit
for bit (test_weighted_gpu.test_exact_bound covers the longest row here too).  Attention is compared with the fp64
adjoint at the attention tests' bars.  Every call runs twice and must give the same bits, launch exactly what the
row-shape table predicts and leave the sentinels around its output alone; input pad columns hold NaN."""
import ctypes as C

import numpy as np
import pytest
import torch

import exact_oracle as xo
import minmax_oracle as mmo
from roc_b200 import _lib
from roc_b200 import kernels as K
from sg_matrix import (DEV, NORM, RELU, SCALAR, SLOPE, SUM, TMASK, TSUM, Guarded, WGraph, attn_backward, check_bits,
                       close_terms, dev_in, every_instantiation, exact, guarded, launches, no_new_nan, planned,
                       same_bits, scores_dev, symmetric_sorted, valid_heads, xgraphs)

pytestmark = pytest.mark.gpu
SUM_V = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 1024, 1025, 2051]
MM_V = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 700]
ATTN_V = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512]
ATTN_S = [1, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256]
SEEN, RAN = set(), set()


# --------------------------------------------------------------------------------------------------------- calls ---
def sum_call(g, gd, h, vec, epi, what):
    outs = []
    for _ in range(2):
        o = guarded(g.n, h, vec)
        g.tr.sum_backward(gd, epilogue=epi, row_end=g.d_re if epi & NORM else None, out=o.view)
        launches(what, planned(g.sched_t, TSUM if epi & NORM else SUM, vec, h), SEEN)
        outs.append(o)
    same_bits(outs[0], outs[1], what)
    outs[0].check_guards(what)
    return outs[0].host()


def minmax_call(g, gd, arg, h, vec, what):
    outs = []
    for _ in range(2):
        o = guarded(g.n, h, vec)
        g.tr.minmax_backward(gd, arg, out=o.view)
        launches(what, planned(g.sched_t, TMASK, vec, h), SEEN)
        outs.append(o)
    same_bits(outs[0], outs[1], what)
    outs[0].check_guards(what)
    return outs[0].host()


def attn_call(g, xd, sd, od, std, gd, heads, h, vec, what):
    runs = []
    for _ in range(2):
        ig, sg = guarded(g.n, h, vec), Guarded(g.n, 2 * heads, 2 * heads + 4, 2 * heads)
        g.tr.attn_backward(g.plan, xd, sd, od, std, gd, heads, SLOPE, in_grad=ig.view, score_grad=sg.view)
        launches(what, attn_backward(g.sched, g.sched_t, vec, h, g.n), SEEN)
        runs.append((ig, sg))
    for a, b in zip(*runs):
        same_bits(a, b, what)
        a.check_guards(what)
    return runs[0][0].host(), runs[0][1].host()


# -------------------------------------------------------------------------------------------------- the matrix ---
def run_sum(vec, h):
    for g in xgraphs().values():
        rng = np.random.RandomState(h * 7 + g.n)
        gy = exact(rng, g.n, h)
        gd = dev_in(gy, vec)
        for epi in (0, NORM, NORM | RELU):
            what = "%s sum H=%d %s epi=%d" % (g.name, h, "vec" if vec else "scalar", epi)
            check_bits(sum_call(g, gd, h, vec, epi, what), xo.sum_backward_epi(g.row_end, g.col, gy, g.n, epi), what)


def run_minmax(vec, h):
    for g in xgraphs().values():
        rng = np.random.RandomState(h * 11 + g.n)
        x, gy = exact(rng, g.n, h), exact(rng, g.n, h)
        xd, gd = dev_in(x, vec), dev_in(gy, vec)
        for aggr in (_lib.AGGR_MAX, _lib.AGGR_MIN):
            what = "%s %s backward H=%d %s" % (g.name, "max" if aggr == 1 else "min", h, "vec" if vec else "scalar")
            _, warg = mmo.forward(0, g.n - 1, 0, g.row_end, g.col, x, aggr)
            _, arg = g.plan.minmax_forward(xd, aggr)
            assert np.array_equal(arg.cpu().numpy().view(np.uint32), warg), what + ": forward indices"
            want = xo.minmax_backward(g.row_end, g.col, gy, warg, g.n)
            got = minmax_call(g, gd, arg, h, vec, what)
            assert np.array_equal(got, want.astype(np.float32)), "%s: differs from the exact reference" % what


def run_attn(vec, h):
    for g in xgraphs().values():
        for heads in [k for k in valid_heads(h) if k in (1, 2, 8)]:
            rng = np.random.RandomState(h * 13 + heads + g.n)
            x, gy = exact(rng, g.n, h), exact(rng, g.n, h)
            s = rng.randn(g.n, 2 * heads).astype(np.float32)
            xd, gd, sd = dev_in(x, vec), dev_in(gy, vec), scores_dev(s)
            od, std = g.plan.attn_forward(xd, sd, heads, SLOPE)
            what = "%s attention H=%d heads=%d %s" % (g.name, h, heads, "vec" if vec else "scalar")
            ig, sg = attn_call(g, xd, sd, od, std, gd, heads, h, vec, what)
            args = (g.row_end, g.col, x, s, od.cpu().numpy(), std.cpu().numpy(), gy, heads, SLOPE)
            wig, wsg = xo.attn_backward(*args)
            mig, msg = xo.attn_backward(*args, magnitude=True)
            for got, want, mag, part, eps in ((ig, wig, mig, "input gradient", 0.0),
                                              (sg[:, :heads], wsg[:, :heads], msg[:, :heads], "d s_dst", 1e-6),
                                              (sg[:, heads:], wsg[:, heads:], msg[:, heads:], "d s_src", 1e-6)):
                no_new_nan(got, want, what + " " + part)
                close_terms(got, want, mag, what + " " + part, eps)


@pytest.mark.parametrize("h", SUM_V, ids=str)
def test_sum_vector(h):
    run_sum(True, h)
    RAN.add(("sum", True, h))


@pytest.mark.parametrize("h", SCALAR, ids=str)
def test_sum_scalar(h):
    run_sum(False, h)
    RAN.add(("sum", False, h))


@pytest.mark.parametrize("h", MM_V, ids=str)
def test_minmax_vector(h):
    run_minmax(True, h)
    RAN.add(("minmax", True, h))


@pytest.mark.parametrize("h", SCALAR, ids=str)
def test_minmax_scalar(h):
    run_minmax(False, h)
    RAN.add(("minmax", False, h))


@pytest.mark.parametrize("h", ATTN_V, ids=str)
def test_attn_vector(h):
    run_attn(True, h)
    RAN.add(("attn", True, h))


@pytest.mark.parametrize("h", ATTN_S, ids=str)
def test_attn_scalar(h):
    run_attn(False, h)
    RAN.add(("attn", False, h))


# -------------------------------------------------------------------------------------------------- identities ---
@pytest.mark.parametrize("h", [1, 5, 16, 17, 64, 65, 128, 200, 256, 513, 1025])
def test_symmetric_graph_gives_the_gathers_bits(h):
    """On a symmetric graph with strictly increasing sources each exact call returns its Q1 counterpart's bits."""
    re_, col = symmetric_sorted(700, 0.02, 8)
    g = WGraph("symmetric", re_, col, 700)
    assert g.plan.rows_sorted()
    rng = np.random.RandomState(h)
    for vec in (True, False):
        gy, x = rng.randn(g.n, h).astype(np.float32), rng.randn(g.n, h).astype(np.float32)
        gd, xd = dev_in(gy, vec), dev_in(x, vec)
        for epi in (0, NORM, NORM | RELU, RELU):
            a, b = guarded(g.n, h, vec), guarded(g.n, h, vec)
            g.tr.sum_backward(gd, epilogue=epi, row_end=g.d_re, out=a.view)
            g.plan.forward(gd, out=b.view, epilogue=epi)
            assert np.array_equal(a.bits(), b.bits()), "H=%d epi=%d: the exact sum differs from the gather" % (h, epi)
        for aggr in (_lib.AGGR_MAX, _lib.AGGR_MIN):
            _, arg = g.plan.minmax_forward(xd, aggr)
            a, b = guarded(g.n, h, vec), guarded(g.n, h, vec)
            g.tr.minmax_backward(gd, arg, out=a.view)
            g.plan.minmax_backward(gd, arg, out=b.view)
            assert np.array_equal(a.bits(), b.bits()), "H=%d: the exact max / min backward differs" % h
        for heads in [k for k in valid_heads(h) if k in (1, 2, 8)]:
            if h > (512 if vec else 256):
                continue
            sd = scores_dev(rng.randn(g.n, 2 * heads).astype(np.float32))
            od, std = g.plan.attn_forward(xd, sd, heads, SLOPE)
            e = g.tr.attn_backward(g.plan, xd, sd, od, std, gd, heads, SLOPE)
            q = g.plan.attn_backward(xd, sd, od, std, gd, heads, SLOPE)
            for u, v in zip(e, q):
                assert np.array_equal(u.cpu().numpy().view(np.int32), v.cpu().numpy().view(np.int32)), \
                    "H=%d heads=%d: the exact attention backward differs" % (h, heads)


def test_gather_misses_the_adjoint_on_a_directed_graph():
    """Q1's results are not the exact reference on the directed multigraph; the exact calls' are."""
    g = xgraphs()["directed"]
    rng = np.random.RandomState(4)
    h = 24
    gy, x = exact(rng, g.n, h), exact(rng, g.n, h)
    gd, xd = dev_in(gy, True), dev_in(x, True)
    want = xo.sum_backward_epi(g.row_end, g.col, gy, g.n, 0)
    assert not np.array_equal(g.plan.forward(gd).cpu().numpy(), want)
    assert np.array_equal(g.tr.sum_backward(gd).cpu().numpy(), want)
    _, arg = g.plan.minmax_forward(xd, _lib.AGGR_MAX)
    want = xo.minmax_backward(g.row_end, g.col, gy, arg.cpu().numpy().view(np.uint32), g.n).astype(np.float32)
    assert not np.array_equal(g.plan.minmax_backward(gd, arg).cpu().numpy(), want)
    assert np.array_equal(g.tr.minmax_backward(gd, arg).cpu().numpy(), want)
    s = rng.randn(g.n, 2).astype(np.float32)
    sd = scores_dev(s)
    od, std = g.plan.attn_forward(xd, sd, 1, SLOPE)
    wig, _ = xo.attn_backward(g.row_end, g.col, x, s, od.cpu().numpy(), std.cpu().numpy(), gy, 1, SLOPE)
    qig, _ = g.plan.attn_backward(xd, sd, od, std, gd, 1, SLOPE)
    assert not np.allclose(qig.cpu().numpy(), wig, rtol=1e-3, atol=1e-3)


# --------------------------------------------------------------------------------------------- one long object ---
def test_one_transpose_for_a_mixed_sequence():
    """One transpose on a side stream serves sums, max / min and attention backwards at growing and shrinking widths
    and both paths; every result matches a fresh transpose's bit for bit."""
    g = xgraphs()["ragged"]
    rng = np.random.RandomState(12)
    steps = [("sum", True, 8, NORM), ("minmax", False, 33, 0), ("attn", True, 64, 8), ("sum", True, 1100, NORM | RELU),
             ("attn", False, 33, 1), ("minmax", True, 700, 0), ("sum", False, 5, 0), ("attn", True, 512, 2)]
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        tr = K.SgTranspose(g.d_re, g.d_col)
    side.synchronize()

    def run(t, kind, vec, h, arg, gd, xd, sd, od, std):
        if kind == "sum":
            o = guarded(g.n, h, vec)
            t.sum_backward(gd, epilogue=arg, row_end=g.d_re, out=o.view)
            return [o.bits()]
        if kind == "minmax":
            o = guarded(g.n, h, vec)
            t.minmax_backward(gd, mx, out=o.view)
            return [o.bits()]
        ig, sg = guarded(g.n, h, vec), Guarded(g.n, 2 * arg, 2 * arg + 4, 2 * arg)
        t.attn_backward(g.plan, xd, sd, od, std, gd, arg, SLOPE, in_grad=ig.view, score_grad=sg.view)
        return [ig.bits(), sg.bits()]

    for kind, vec, h, arg in steps:
        gd, xd = dev_in(exact(rng, g.n, h), vec), dev_in(exact(rng, g.n, h), vec)
        sd = od = std = mx = None
        if kind == "attn":
            sd = scores_dev(rng.randn(g.n, 2 * arg).astype(np.float32))
            od, std = g.plan.attn_forward(xd, sd, arg, SLOPE)
        if kind == "minmax":
            _, mx = g.plan.minmax_forward(xd, _lib.AGGR_MIN)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            a = run(tr, kind, vec, h, arg, gd, xd, sd, od, std)
        side.synchronize()
        fresh = K.SgTranspose(g.d_re, g.d_col)
        b = run(fresh, kind, vec, h, arg, gd, xd, sd, od, std)
        torch.cuda.synchronize()
        fresh.close()
        for u, v in zip(a, b):
            assert np.array_equal(u, v), "%s H=%d: the long-lived transpose differs from a fresh one" % (kind, h)
    tr.close()


# ----------------------------------------------------------------------------------------------------- refusals ---
def test_refusals():
    g = xgraphs()["tiny"]
    t, p = g.tr.handle, g.plan.handle
    x = torch.zeros(g.n, 16, device=DEV)
    a = torch.zeros(g.n, 16, dtype=torch.int32, device=DEV)
    s = torch.zeros(g.n, 16, device=DEV)
    P = lambda v: C.c_void_p(v.data_ptr())                                  # noqa: E731
    INV, UNS = _lib.ROC_ERR_INVALID, _lib.ROC_ERR_UNSUPPORTED
    L = _lib.lib
    assert L.roc_sg_transpose_sum_backward(None, 8, P(x), 16, P(x), 16, 0, None, None) == INV
    assert L.roc_sg_transpose_sum_backward(t, 8, None, 16, P(x), 16, 0, None, None) == INV
    assert L.roc_sg_transpose_sum_backward(t, 8, P(x), 4, P(x), 16, 0, None, None) == INV
    assert L.roc_sg_transpose_sum_backward(t, 8, P(x), 16, P(x), 4, 0, None, None) == INV
    assert L.roc_sg_transpose_sum_backward(t, 0, P(x), 16, P(x), 16, 0, None, None) == INV
    assert L.roc_sg_transpose_sum_backward(t, 8, P(x), 16, P(x), 16, NORM, None, None) == INV    # NORM, no rowEnd
    assert L.roc_sg_transpose_sum_backward(t, 8, P(x), 16, P(x), 16, RELU, None, None) == 0
    assert L.roc_sg_transpose_minmax_backward(t, 8, P(x), 16, None, 16, P(x), 16, None) == INV
    assert L.roc_sg_transpose_minmax_backward(t, 8, P(x), 16, P(a), 4, P(x), 16, None) == INV
    assert L.roc_sg_transpose_minmax_backward(None, 8, P(x), 16, P(a), 16, P(x), 16, None) == INV

    def attn(plan, tr, heads, h, slope=0.2, ld=16, lds=16):
        return L.roc_sg_attn_backward_exact(plan, tr, heads, h, slope, P(x), ld, P(s), lds, P(x), ld, P(s), lds, P(x),
                                            ld, P(x), ld, P(s), lds, None)
    assert attn(p, t, 1, 8) == 0
    assert attn(None, t, 1, 8) == INV and attn(p, None, 1, 8) == INV
    assert attn(p, t, 1, 8, ld=4) == INV and attn(p, t, 4, 8, lds=6) == INV and attn(p, t, 0, 8) == INV
    assert attn(p, t, 1, 8, slope=-1.0) == INV and attn(p, t, 1, 8, slope=float("inf")) == INV
    assert attn(p, t, 3, 12) == UNS and attn(p, t, 2, 12) == UNS and attn(p, t, 4, 8) == UNS    # heads, F < 4 or odd
    big = torch.zeros(g.n, 520, device=DEV)
    assert L.roc_sg_attn_backward_exact(p, t, 1, 516, 0.2, P(big), 520, P(s), 16, P(big), 520, P(s), 16, P(big), 520,
                                        P(big), 520, P(s), 16, None) == UNS                       # H > 512
    other = xgraphs()["single"]
    assert attn(other.plan.handle, t, 1, 8) == INV                                               # another graph's plan


# ----------------------------------------------------------------------------------------------------- coverage ---
def test_exact_covered():
    wanted = {(k, v, h) for k, ws in (("sum", SUM_V), ("minmax", MM_V), ("attn", ATTN_V)) for v, hs in
              ((True, ws), (False, ATTN_S if k == "attn" else SCALAR)) for h in hs}
    if not wanted <= RAN:
        pytest.skip("%d of the matrix cases did not run in this process" % len(wanted - RAN))
    # TMASK's fix-ups are the sum's, which test_sg_matrix_gpu covers
    missing = {x for x in every_instantiation((TSUM, TMASK)) if x[1] != SUM} - SEEN
    assert not missing, "never launched: %s" % sorted(missing)
