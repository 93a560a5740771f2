"""The teleport sum (roc_sg_forward_teleport_planned) and scaled_add (roc_scaled_add_fwd / _bwd) on the GPU.

The teleport's bit contract: its bytes equal the unfused chain roc_sg_forward_planned (NORM or NONE) ->
roc_scaled_add_fwd -> (NORM_OUT) roc_indegree_norm, on every row-shape rung of both row forms (sg_matrix.RUNGS,
SCALAR), with padded and odd pitches, on the sg_matrix graphs (heavy and big rows, rows of degree 0, a slice with
global ids), for all four epilogues.  scaled_add is checked against fp64 and against roc_add_fwd at (1, 1)."""
import numpy as np
import pytest
import torch

import sg_matrix as M
from roc_b200 import _lib
from roc_b200 import kernels as K

pytestmark = pytest.mark.gpu
TELE = _lib.SG_RED_TELE
NORM, NORM_OUT = _lib.SG_EPI_NORM, _lib.SG_EPI_NORM_OUT
EPIS = (0, NORM, NORM_OUT, NORM | NORM_OUT)
ALPHA, BETA = float(np.float32(1.0 - 0.1)), float(np.float32(0.1))
# TELE's row of the reduction table, restated here: SUM's column blocks, no ring form, its own fix-ups
TELE_RED = M.Red(256, 256, False, "own", False)
VEC_WIDTHS = sorted({w for qc, _, _ in M.RUNGS for w in (4 * qc - 3, 4 * qc)} | {1025, 2048 + 6})
GRAPHS = ("single", "tiny", "aligned", "straddle", "carry32", "ragged", "slice")


def want_launches(s, vec, h):
    """TELE's launches: per column block of SUM's width, the main kernel and its own fix-ups."""
    vw = 4 if vec else 1
    block = vw * (TELE_RED.q4 if vec else TELE_RED.q1)
    out = []
    for c0 in range(0, h, block):
        lanes, nch = M.shape(M.cdiv(min(h - c0, block), vw))
        out.append(("main", TELE, vw, lanes, nch, M.cdiv(s.chunks, 256 // lanes)))
        out += M.fixups(s, TELE, vw, lanes, nch)
    return out


def rng_rows(rng, rows, h):
    """normal values with some +-0 (the norm skips zero numerators)"""
    a = rng.standard_normal((rows, h)).astype(np.float32)
    a[rng.random_sample((rows, h)) < 0.05] = 0.0
    a[rng.random_sample((rows, h)) < 0.05] = -0.0
    return a


def t_dev(t, vec, odd):
    """t on the device: padded like `in`, or (odd) at a pitch that is not a multiple of 4 and off 16-byte alignment"""
    if not odd:
        return M.dev_in(t, vec)
    h = t.shape[1]
    buf = torch.full((t.shape[0] * (h + 3) + 1,), float("nan"), device=M.DEV)
    v = buf[1:1 + t.shape[0] * (h + 3)].view(t.shape[0], h + 3)[:, :h]
    v.copy_(torch.from_numpy(t))
    return v


def chain(g, x, t, epi, vec, h):
    """the unfused three-kernel chain, each output laid out like the teleport's"""
    s = M.guarded(g.nloc, h, vec)
    g.plan.forward(x, out=s.view, epilogue=epi & NORM)
    y = M.guarded(g.nloc, h, vec)
    K.scaled_add_fwd(s.view, t, ALPHA, BETA, out=y.view)
    if not epi & NORM_OUT:
        return y
    z = M.guarded(g.nloc, h, vec)
    K.indegree_norm(g.row_left, g.row_right, g.col_left, g.d_re, y.view, out=z.view)
    return z


def valid_bits(gd, h):
    return gd.bits()[1:gd.rows + 1, :h]


@pytest.mark.parametrize("name", GRAPHS)
@pytest.mark.parametrize("vec", [True, False], ids=["vec", "scalar"])
def test_teleport_is_the_unfused_chain(name, vec):
    g = M.graphs()[name]
    rng = np.random.RandomState(len(name) * 7 + vec)
    widths = VEC_WIDTHS if vec else M.SCALAR
    for h in widths:
        x = M.dev_in(rng_rows(rng, g.n, h), vec)
        t_host = rng_rows(rng, g.nloc, h)
        for odd in (False, True):
            t = t_dev(t_host, vec, odd)
            for epi in EPIS:
                what = "%s %s H=%d epi=%d odd t=%s" % (name, "vec" if vec else "scalar", h, epi, odd)
                out = M.guarded(g.nloc, h, vec)
                g.plan.teleport_forward(x, t, ALPHA, BETA, epilogue=epi, out=out.view)
                M.launches(what, want_launches(g.sched, vec, h), set())
                out.check_guards(what)
                ref = chain(g, x, t, epi, vec, h)
                assert np.array_equal(valid_bits(out, h), valid_bits(ref, h)), what
                again = M.guarded(g.nloc, h, vec)
                g.plan.teleport_forward(x, t, ALPHA, BETA, epilogue=epi, out=again.view)
                M.same_bits(out, again, what)


def test_teleport_degree_zero_rows_follow_the_chain():
    """ragged's rows of degree 0: NORM gives 0 / 0 = NaN, which the teleport keeps, as the chain does"""
    g = M.graphs()["ragged"]
    assert (g.deg == 0).any()
    rng = np.random.RandomState(3)
    for vec in (True, False):
        h = 41
        x, t = M.dev_in(rng_rows(rng, g.n, h), vec), M.dev_in(rng_rows(rng, g.nloc, h), vec)
        for epi in EPIS:
            out = M.guarded(g.nloc, h, vec)
            g.plan.teleport_forward(x, t, ALPHA, BETA, epilogue=epi, out=out.view)
            got, want = valid_bits(out, h), valid_bits(chain(g, x, t, epi, vec, h), h)
            assert np.array_equal(got, want), (vec, epi)
            z = out.host()[g.deg == 0]
            if epi & NORM:                 # 0 / sqrt(0)
                assert np.isnan(z).all(), (vec, epi)
            elif epi & NORM_OUT:           # (beta t) / sqrt(0)
                assert not np.isfinite(z).any(), (vec, epi)
            else:
                assert np.isfinite(z).all(), (vec, epi)


def test_teleport_at_one_and_zero_is_the_sum():
    """alpha = 1, beta = 0 adds +0 to the sum: the sum's bits (t finite)"""
    g = M.graphs()["carry32"]
    rng = np.random.RandomState(5)
    for vec in (True, False):
        for h in (41, 64, 300):
            x, t = M.dev_in(rng_rows(rng, g.n, h), vec), M.dev_in(rng_rows(rng, g.nloc, h), vec)
            out, ref = M.guarded(g.nloc, h, vec), M.guarded(g.nloc, h, vec)
            g.plan.teleport_forward(x, t, 1.0, 0.0, epilogue=NORM, out=out.view)
            g.plan.forward(x, out=ref.view, epilogue=NORM)
            got, want = out.host(), ref.host()
            assert np.array_equal(got + 0.0, want + 0.0, equal_nan=True), (vec, h)


def test_teleport_refusals():
    g = M.graphs()["tiny"]
    h = 8
    x = M.dev_in(np.ones((g.n, h), np.float32), True)
    t = M.dev_in(np.ones((g.nloc, h), np.float32), True)
    out = M.guarded(g.nloc, h, True).view
    P = K._ptr

    def call(H=h, xin=x, tt=t, o=out, alpha=ALPHA, beta=BETA, epi=NORM, ldIn=None, ldT=None, ldOut=None):
        return _lib.lib.roc_sg_forward_teleport_planned(
            g.plan.handle, H, P(xin), ldIn if ldIn is not None else K._ld(x), alpha, P(tt),
            ldT if ldT is not None else K._ld(t), beta, P(o), ldOut if ldOut is not None else K._ld(out), epi,
            K._stream())

    assert call() == _lib.ROC_OK
    for bad in (dict(H=0), dict(xin=None), dict(tt=None), dict(o=None), dict(o=t), dict(ldIn=h - 1),
                dict(ldT=h - 1), dict(ldOut=h - 1), dict(alpha=float("inf")), dict(beta=float("nan")),
                dict(epi=_lib.SG_EPI_RELU), dict(epi=NORM | _lib.SG_EPI_RELU), dict(epi=8)):
        assert call(**bad) == _lib.ROC_ERR_INVALID, bad
    assert K.sg_launches() == []


# ------------------------------------------------------------------------------------------------- scaled_add ---
HALF = 0.5 + 1e-6      # half an ulp, with room for the fp64 reference's own rounding


def _padded(a, vec):
    return M.dev_in(a, vec)


def _ulps(got, want):
    """|got - want| in units of the last place of want (fp32), per element"""
    want32 = want.astype(np.float32)
    spacing = np.spacing(np.abs(want32)).astype(np.float64)
    return np.abs(got.astype(np.float64) - want) / np.maximum(spacing, np.finfo(np.float32).tiny)


@pytest.mark.parametrize("h", [1, 3, 4, 41, 64, 257])
@pytest.mark.parametrize("vec", [True, False], ids=["vec", "scalar"])
def test_scaled_add_matches_fp64(h, vec):
    rng = np.random.RandomState(h)
    rows = 3001
    a, b = rng_rows(rng, rows, h), rng_rows(rng, rows, h)
    for alpha, beta in ((ALPHA, BETA), (-1.75, 3.0e-3), (1.0, 1.0), (0.0, 2.0)):
        da, db = _padded(a, vec), _padded(b, vec)
        y = K.scaled_add_fwd(da, db, alpha, beta, out=M.guarded(rows, h, vec).view).cpu().numpy()
        # the contract's own expression: beta * b rounded to fp32, then one fma
        want = alpha * a.astype(np.float64) + (np.float32(beta) * b).astype(np.float64)
        assert float(_ulps(y, want).max()) <= HALF, (h, alpha, beta)
        # and within one ulp of the terms' magnitude of the exact value (beta * b's rounding is relative to it)
        exact = alpha * a.astype(np.float64) + beta * b.astype(np.float64)
        terms = np.abs(alpha * a.astype(np.float64)) + np.abs(beta * b.astype(np.float64))
        err = np.abs(y.astype(np.float64) - exact)
        ulp = np.maximum(terms * 2.0 ** -23, np.finfo(np.float32).tiny)
        assert float((err / ulp).max()) <= 1.0, (h, alpha, beta)
    # (1, 1) is roc_add_fwd's bits
    da, db = _padded(a, vec), _padded(b, vec)
    y = K.scaled_add_fwd(da, db, 1.0, 1.0)
    ref = K.add_fwd(da, db)
    assert np.array_equal(y.cpu().numpy().view(np.int32), ref.cpu().numpy().view(np.int32))


@pytest.mark.parametrize("h", [1, 41, 64])
@pytest.mark.parametrize("vec", [True, False], ids=["vec", "scalar"])
def test_scaled_add_backward(h, vec):
    rng = np.random.RandomState(100 + h)
    rows = 2049
    g = rng_rows(rng, rows, h)
    base_a, base_b = rng_rows(rng, rows, h), rng_rows(rng, rows, h)
    dg = _padded(g, vec)
    for acc_a in (0, 1):
        for acc_b in (0, 1):
            da, db = _padded(base_a, vec), _padded(base_b, vec)
            K.scaled_add_bwd(dg, ALPHA, da, acc_a, BETA, db, acc_b)
            for d, coef, acc, base in ((da, ALPHA, acc_a, base_a), (db, BETA, acc_b, base_b)):
                got = d.cpu().numpy()
                want = coef * g.astype(np.float64) + (base.astype(np.float64) if acc else 0.0)
                assert float(_ulps(got, want).max()) <= HALF, (h, acc)
    # NULL outputs are skipped
    db = _padded(base_b, vec)
    K.scaled_add_bwd(dg, ALPHA, None, 0, BETA, db, 0)
    assert np.array_equal(db.cpu().numpy(), (np.float32(BETA) * g).astype(np.float32))
    da = _padded(base_a, vec)
    K.scaled_add_bwd(dg, ALPHA, da, 1, BETA, None, 0)
    assert float(_ulps(da.cpu().numpy(), ALPHA * g.astype(np.float64) + base_a).max()) <= HALF
    K.scaled_add_bwd(dg, ALPHA, None, 0, BETA, None, 0)


def test_scaled_add_refusals():
    a = M.dev_in(np.ones((4, 8), np.float32), True)
    y = M.dev_in(np.ones((4, 8), np.float32), True)
    P, ld, st = K._ptr, K._ld, K._stream
    L = _lib.lib

    def fwd(rows=4, H=8, alpha=1.0, beta=1.0, pa=a, pb=a, py=y, ldA=None):
        return L.roc_scaled_add_fwd(rows, H, alpha, P(pa), ldA if ldA is not None else ld(a), beta, P(pb), ld(a),
                                    P(py), ld(y), st())

    assert fwd() == _lib.ROC_OK
    for bad in (dict(rows=-1), dict(H=0), dict(alpha=float("inf")), dict(beta=float("nan")), dict(pa=None),
                dict(pb=None), dict(py=None), dict(ldA=7)):
        assert fwd(**bad) == _lib.ROC_ERR_INVALID, bad

    def bwd(dy=a, da=y, db=None, alpha=1.0, beta=1.0, ldDY=None):
        return L.roc_scaled_add_bwd(4, 8, P(dy), ldDY if ldDY is not None else ld(a), alpha, P(da), ld(y), 0, beta,
                                    P(db), ld(y), 0, st())

    assert bwd() == _lib.ROC_OK
    for bad in (dict(dy=None), dict(alpha=float("-inf")), dict(beta=float("nan")), dict(ldDY=3), dict(db=y)):
        assert bwd(**bad) == _lib.ROC_ERR_INVALID, bad
