"""Edge-weighted ScatterGather on the GPU: the weighted forward, its transposed backward and the edge-weight gradient
(include/roc_b200.h) at both ends of every rung of the row-shape table and past the widest in column blocks, on every
graph of the ScatterGather matrix (sg_matrix.py) and on directed graphs with duplicate edges and nodes with
no out-edge.

Exact data: features are multiples of 1/16 in [-8, 8], weights multiples of 1/2 in [-4, 4], the gradients of the
edge dot multiples of 1/16 in [-1, 1].  test_exact_bound asserts that every partial sum of every row (the longest has
5 000 edges) and of every dot product then stays below 2^24 units of the products' granularity, so each fp32 result
is exact in any order and is compared bit for bit with the fp64 oracle.  Random fp32 data is compared with fp64 at
1e-4.  Every call runs twice and must give the same bits, launches exactly what the table predicts, leaves the
sentinels around its output alone and never reads an input's NaN pad columns into a result."""
import ctypes as C

import numpy as np
import pytest
import torch

import weighted_oracle as wo
from roc_b200 import _lib
from roc_b200 import kernels as K
from sg_graphs import to_dev
from sg_matrix import (DEV, EDOT, SCALAR, SENT_F, WSUM, WGraph, dev_in, every_instantiation, exact, guarded, launches,
                       planned, same_bits, symmetric_sorted, weighted_backward, wgraphs)

pytestmark = pytest.mark.gpu
VEC_W = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 700, 1024, 1025, 1100, 2051]
SEEN = set()
RAN = set()


# --------------------------------------------------------------------------------------------------------- data ---
def weights(rng, e):
    return (rng.randint(-8, 9, size=max(e, 1)) / 2.0).astype(np.float32)


def small(rng, rows, h):
    return (rng.randint(-16, 17, size=(rows, h)) / 16.0).astype(np.float32)


def wdev(w):
    return torch.from_numpy(w).to(DEV)


def max_row(row_end, col_left=0):
    t = np.asarray(row_end, np.int64) - col_left
    return int(np.diff(np.concatenate([[0], t])).max()) if t.shape[0] else 0


def test_exact_bound():
    """Every exact case's partial sums stay below 2^24 units: the longest row (forward and transposed) times the
    largest product, and the widest dot product plus an accumulated dw."""
    longest = max(max(max_row(g.row_end, g.col_left), max_row(g.re_t) if g.whole else 0) for g in wgraphs().values())
    assert longest == 5000
    assert longest * 8 * 4 * 32 < 2 ** 24                   # |x| <= 8, |w| <= 4, granularity 1/32
    assert (max(VEC_W) * 1 * 8 + 4) * 256 < 2 ** 24        # |gy| <= 1, |x| <= 8, granularity 1/256, |dw0| <= 4


# ------------------------------------------------------------------------------------------------------- calls ---
def bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.int32), np.asarray(b, np.float32).view(np.int32))


def check_exact(got, want, what):
    w32 = want.astype(np.float32)
    assert np.array_equal(w32.astype(np.float64), want), "%s: the reference is not exact in fp32" % what
    bad = got != w32
    assert not bad.any(), "%s: %d/%d differ from the exact reference, first at %s (%r vs %r)" % (
        what, int(bad.sum()), bad.size, np.argwhere(bad)[0], got[bad][0], w32[bad][0])


def fwd(g, xd, wd, h, vec):
    outs = []
    for _ in range(2):
        o = guarded(g.nloc, h, vec)
        g.plan.weighted_forward(xd, wd, out=o.view)
        launches("%s forward H=%d" % (g.name, h), planned(g.sched, WSUM, vec, h), SEEN)
        outs.append(o)
    same_bits(outs[0], outs[1], "%s forward" % g.name)
    outs[0].check_guards("%s forward" % g.name)
    return outs[0].host()


def bwd(g, gd, wd, h, vec):
    outs = []
    for _ in range(2):
        o = guarded(g.n, h, vec)
        g.tr.backward(gd, wd, out=o.view)
        launches("%s backward H=%d" % (g.name, h), weighted_backward(g, vec, h), SEEN)
        outs.append(o)
    same_bits(outs[0], outs[1], "%s backward" % g.name)
    outs[0].check_guards("%s backward" % g.name)
    return outs[0].host()


def edot(g, gd, xd, h, vec, dw0=None):
    """dw into a guarded flat buffer; with dw0, accumulated onto it."""
    res = []
    for _ in range(2):
        buf = torch.full((g.E + 8,), SENT_F, device=DEV)
        if dw0 is not None:
            buf[4:4 + g.E] = torch.from_numpy(dw0[:g.E]).to(DEV)
        g.plan.edge_dot(gd, xd, dw=buf[4:], accumulate=dw0 is not None)
        launches("%s edge dot H=%d" % (g.name, h), planned(g.sched, EDOT, vec, h), SEEN)
        b = buf.cpu().numpy()
        assert bits_equal(b[:4], [SENT_F] * 4) and bits_equal(b[4 + g.E:], [SENT_F] * 4), "%s edge dot: guards" % g.name
        res.append(b[4:4 + g.E])
    assert bits_equal(res[0], res[1]), "%s edge dot: repeated call differs" % g.name
    return res[0]


def run_exact(vec, h):
    for g in wgraphs().values():
        rng = np.random.RandomState(h * 5 + g.nloc)
        what = "%s H=%d %s" % (g.name, h, "vec" if vec else "scalar")
        x, w = exact(rng, g.n, h), weights(rng, g.E)
        xd, wd = dev_in(x, vec), wdev(w)
        check_exact(fwd(g, xd, wd, h, vec), wo.forward(g.row_end, g.col, x, w[:g.E], g.col_left), what + " forward")
        gy = small(rng, g.nloc, h)
        gd = dev_in(gy, vec)
        want = wo.edge_dot(g.row_end, g.col, gy, x, g.col_left)
        check_exact(edot(g, gd, xd, h, vec), want, what + " edge dot")
        dw0 = weights(rng, g.E)
        check_exact(edot(g, gd, xd, h, vec, dw0), want + dw0[:g.E], what + " edge dot accumulated")
        if g.whole:
            gb = exact(rng, g.n, h)
            check_exact(bwd(g, dev_in(gb, vec), wd, h, vec), wo.input_grad(g.row_end, g.col, gb, w[:g.E], g.n),
                        what + " backward")


def run_random(vec, h):
    for g in wgraphs().values():
        rng = np.random.RandomState(h * 3 + g.nloc + 1)
        what = "%s H=%d %s random" % (g.name, h, "vec" if vec else "scalar")
        x, w, gy = (rng.randn(g.n, h).astype(np.float32), rng.randn(max(g.E, 1)).astype(np.float32),
                    rng.randn(g.n, h).astype(np.float32))
        xd, wd, gd = dev_in(x, vec), wdev(w), dev_in(gy[:g.nloc], vec)
        ax, aw, ag = np.abs(x), np.abs(w[:g.E]), np.abs(gy)
        close(fwd(g, xd, wd, h, vec), wo.forward(g.row_end, g.col, x, w[:g.E], g.col_left),
              wo.forward(g.row_end, g.col, ax, aw, g.col_left), what + " forward")
        close(edot(g, gd, xd, h, vec), wo.edge_dot(g.row_end, g.col, gy[:g.nloc], x, g.col_left),
              wo.edge_dot(g.row_end, g.col, ag[:g.nloc], ax, g.col_left), what + " edge dot")
        if g.whole:
            close(bwd(g, dev_in(gy, vec), wd, h, vec), wo.input_grad(g.row_end, g.col, gy, w[:g.E], g.n),
                  wo.input_grad(g.row_end, g.col, ag, aw, g.n), what + " backward")


def close(got, want, mag, what):
    """|got - want| <= 1e-4 * (the sum of the terms' magnitudes) + 1e-30."""
    assert not np.isnan(got).any(), "%s: NaN" % what
    err = np.abs(got.astype(np.float64) - want)
    bad = err > 1e-4 * mag + 1e-30
    assert not bad.any(), "%s: %d elements off, worst %g at %s" % (what, int(bad.sum()), err.max(), np.argwhere(bad)[0])


@pytest.mark.parametrize("h", VEC_W, ids=str)
def test_vector(h):
    run_exact(True, h)
    run_random(True, h)
    RAN.add(("vec", h))


@pytest.mark.parametrize("h", SCALAR, ids=str)
def test_scalar(h):
    run_exact(False, h)
    run_random(False, h)
    RAN.add(("scalar", h))


# --------------------------------------------------------------------------------------------------- identities ---
@pytest.mark.parametrize("h", [1, 4, 5, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 576, 1024, 1025, 2051])
def test_all_ones_is_the_sum(h):
    """With every weight 1.0 the weighted forward is roc_sg_forward_planned's sum bit for bit (signed zeros too) at
    every rung and in column blocks, whose trailing block lands on a narrower rung (513, 576, 1025, 2051)."""
    for vec in (True, False):
        for g in wgraphs().values():
            rng = np.random.RandomState(h)
            x = rng.randn(g.n, h).astype(np.float32)
            x[::3, ::2] = -0.0
            xd = dev_in(x, vec)
            ones = torch.ones(max(g.E, 1), device=DEV)
            a, b = guarded(g.nloc, h, vec), guarded(g.nloc, h, vec)
            g.plan.weighted_forward(xd, ones, out=a.view)
            g.plan.forward(xd, out=b.view)
            assert np.array_equal(a.bits(), b.bits()), "%s H=%d: the all-ones weighted sum differs from the sum" % (
                g.name, h)


@pytest.mark.parametrize("h", [5, 64, 200, 602])
def test_symmetric_transpose_is_the_graph(h):
    """On a symmetric graph with strictly increasing sources the transposed CSR is the CSR, and the all-ones
    transposed backward is roc_sg_backward's bits."""
    re_, col = symmetric_sorted(700, 0.02, 8)
    g = WGraph("symmetric", re_, col, 700)
    info = g.tr.info()
    assert np.array_equal(info["row_end"].cpu().numpy().astype(np.uint64), re_)
    assert np.array_equal(info["col"].cpu().numpy().view(np.uint32), col)
    gy = torch.randn(700, h, device=DEV)
    got = g.tr.backward(gy, torch.ones(col.shape[0], device=DEV))
    want = K.sg_backward(0, 699, 0, g.d_re, g.d_col, gy.contiguous())
    assert np.array_equal(got.cpu().numpy().view(np.int32), want.cpu().numpy().view(np.int32))


def test_directed_backward_is_the_adjoint():
    """On a directed graph the transposed backward is the true adjoint, where the sum's gather (quirk Q1) is not."""
    g = wgraphs()["directed"]
    rng = np.random.RandomState(4)
    gy = exact(rng, g.n, 24)
    gd = dev_in(gy, True)
    ones = torch.ones(g.E, device=DEV)
    want = wo.input_grad(g.row_end, g.col, gy, np.ones(g.E), g.n)
    check_exact(g.tr.backward(gd, ones).cpu().numpy(), want, "directed adjoint")
    q1 = g.plan.forward(gd).cpu().numpy()
    assert not np.array_equal(q1, want.astype(np.float32))


# ---------------------------------------------------------------------------------------------------- transpose ---
def test_transpose_matches_the_oracle():
    for g in wgraphs().values():
        if not g.whole:
            continue
        info = g.tr.info()
        assert np.array_equal(info["row_end"].cpu().numpy().astype(np.uint64), g.re_t), g.name
        assert np.array_equal(info["col"].cpu().numpy().view(np.uint32), g.col_t), g.name
        assert np.array_equal(info["perm"].cpu().numpy().view(np.uint32), g.perm), g.name


def test_transpose_refuses_a_slice_and_bad_ids():
    g = wgraphs()["slice"]
    h = C.c_void_p()
    # the slice's rows rebased to its own edges: its ids are global, beyond its row count
    re_local = torch.from_numpy((g.row_end - np.uint64(g.col_left)).astype(np.int64)).to(DEV)
    rc = _lib.lib.roc_sg_transpose_create(g.nloc, C.c_void_p(re_local.data_ptr()), C.c_void_p(g.d_col.data_ptr()),
                                          None, C.byref(h))
    assert rc == _lib.ROC_ERR_UNSUPPORTED and not h.value
    re_, col = to_dev(np.array([2, 3], np.uint64), np.array([0, 1, 2], np.uint32))     # id 2 with N = 2
    rc = _lib.lib.roc_sg_transpose_create(2, C.c_void_p(re_.data_ptr()), C.c_void_p(col.data_ptr()), None, C.byref(h))
    assert rc == _lib.ROC_ERR_UNSUPPORTED
    assert _lib.lib.roc_sg_transpose_create(0, C.c_void_p(re_.data_ptr()), None, None, C.byref(h)) == \
        _lib.ROC_ERR_INVALID
    t = wgraphs()["tiny"].tr
    x = torch.zeros(t.n, 8, device=DEV)
    assert _lib.lib.roc_sg_weighted_backward_planned(t.handle, 8, C.c_void_p(x.data_ptr()), 4, None,
                                                     C.c_void_p(x.data_ptr()), 8, None) == _lib.ROC_ERR_INVALID


# --------------------------------------------------------------------------------------------- one long object ---
def test_one_transpose_for_every_call():
    """One transpose on a side stream through growing and shrinking widths, both paths and changing weights (its
    permuted-weight buffer is grown in stream order) matches a fresh one bit for bit."""
    g = wgraphs()["ragged"]
    rng = np.random.RandomState(9)
    steps = [(True, 8), (False, 33), (True, 700), (True, 64), (False, 300), (True, 1)]
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        tr = K.SgTranspose(g.d_re, g.d_col)
    for vec, h in steps:
        gd = dev_in(rng.randn(g.n, h).astype(np.float32), vec)
        wd = wdev(rng.randn(g.E).astype(np.float32))
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            o1 = guarded(g.n, h, vec)
            tr.backward(gd, wd, out=o1.view)
        side.synchronize()
        fresh = K.SgTranspose(g.d_re, g.d_col)
        o2 = guarded(g.n, h, vec)
        fresh.backward(gd, wd, out=o2.view)
        torch.cuda.synchronize()
        fresh.close()
        assert np.array_equal(o1.bits(), o2.bits()), "H=%d: the long-lived transpose differs from a fresh one" % h
    tr.close()


# ----------------------------------------------------------------------------------------------------- coverage ---
def test_weighted_covered():
    wanted = {("vec", h) for h in VEC_W} | {("scalar", h) for h in SCALAR}
    if not wanted <= RAN:
        pytest.skip("%d of the matrix cases did not run in this process" % len(wanted - RAN))
    want = every_instantiation((WSUM, EDOT)) | {("permute", -1, 1, 1, 1)}
    missing = want - SEEN
    assert not missing, "never launched: %s" % sorted(missing)
    assert SEEN <= want, "launched outside the table: %s" % sorted(SEEN - want)
