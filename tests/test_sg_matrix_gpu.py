"""Every ScatterGather instantiation against an exact or fp64 reference, on graphs built to hit the plan's edge cases.

The row-shape table (sg.cu, with_shape) maps a row of Q T-columns (float4 on the vector path, float on the scalar
path) to L lanes and NCH chunks per lane: Q <= 4 -> (4, 1), <= 8 -> (8, 1), <= 16 -> (16, 1), <= 32 -> (32, 1),
<= 64 -> (32, 2), <= 128 -> (32, 4), <= 256 -> (32, 8).  Each case here is one reduction family on one path at one
width, chosen at both ends of a rung (and past the widest, where the call is cut into column blocks), and loops over
every graph below.  roc_sg_last_call_info reports what each call launched; every case asserts the whole launch list
(kind, reduction, VEC, L, NCH, grid), and test_matrix_covered checks at the end that every main kernel and fix-up
instantiation the table can produce was reached.

Features are multiples of 1/16 with |x| <= 8, so every fp32 partial sum on these graphs is exact in any order: the
sum, its norm / relu epilogue, max / min (values and indices) and the max / min backward are compared bit for bit.
A dropped, doubled or misrouted edge, carry or column is then off by a whole term.  Attention keeps the fp64 oracle
and the error bound of test_attn_gpu.py.  Input pad columns hold NaN; outputs sit in buffers with a guard row above
and below and at least 4 guard columns, filled with a sentinel that must survive (vector path: the pad columns up to
round_up(H, 4) may be written, nothing past them).  Each call is repeated and must give the same bits.

test_one_plan_for_every_call runs one plan, reserved small, on a side stream through growing and shrinking widths,
both paths, every reduction and changing head counts and selfBase; each call must match a fresh plan bit for bit."""
import numpy as np
import pytest
import torch

import attn_oracle as ao
import minmax_oracle as mmo
from conftest import rel_close
from oracle import oracle
from roc_b200 import _lib
from roc_b200 import kernels as K
from sg_graphs import graph, to_dev
from test_attn_gpu import close_terms, valid_heads

pytestmark = pytest.mark.gpu
DEV = "cuda"
CH, BIG = 64, 32                         # edges per chunk; the most carries a row finished by one worker has
SLOPE = 0.2
SUM, MAX, MIN, MASK, ASTAT, ATTN, ADST, ASRC = range(8)
NORM, RELU = _lib.SG_EPI_NORM, _lib.SG_EPI_RELU
SENT_F = -1234.5                         # the sentinel of float outputs
SENT_I = 0x5A5A5A5A                      # and of index outputs
RUNGS = ((4, 4, 1), (8, 8, 1), (16, 16, 1), (32, 32, 1), (64, 32, 2), (128, 32, 4), (256, 32, 8))


def shape(q):
    """(L, NCH) of a row of q T-columns."""
    for qc, lanes, nch in RUNGS:
        if q <= qc:
            return lanes, nch
    raise ValueError(q)


def max_q(vec, red):
    """sg_max_q: the widest row, in T-columns, one launch takes."""
    return 8 if red == ASTAT else 128 if (vec == 4 and red != SUM) else 256


def r4(h):
    return (h + 3) // 4 * 4


def cdiv(a, b):
    return (a + b - 1) // b


# ------------------------------------------------------------------------------------------------------ graphs ---
class Graph:
    """One plan's CSR: row_end holds its rows' END offsets in the edge array (global; the plan's edges start at
    col_left), col their sources, ids < n.  The chunk schedule (chunks, carries, heavy and big rows) is recomputed
    here from the definitions in sg.cu and must match the plan's."""

    def __init__(self, name, row_end, col, n, row_left=0, col_left=0, expect=(), full=None):
        self.name, self.n, self.row_left, self.col_left, self.full = name, n, row_left, col_left, full
        self.row_end = np.asarray(row_end, dtype=np.uint64)
        self.col = np.asarray(col, dtype=np.uint32)
        self.nloc = self.row_end.shape[0]
        self.row_right = row_left + self.nloc - 1
        self.self_base = row_left
        t = self.row_end.astype(np.int64) - col_left
        s = np.concatenate([[0], t[:-1]])
        self.deg = t - s
        carries = np.where(self.deg > CH, (t - 1) // CH - s // CH, 0)
        self.E = int(t[-1])
        assert self.col.shape[0] == self.E
        self.chunks = self.E // CH + 1
        self.carries = int(carries.sum())
        self.heavy = int(((self.deg > CH) & (carries <= BIG)).sum())
        self.big = int((carries > BIG).sum())
        self.id_end = int(self.col.max()) + 1 if self.E else 0
        have = {k for k, v in (("heavy", self.heavy), ("big", self.big), ("carries", self.carries)) if v}
        assert have == set(expect), "%s: the graph has %s, its definition says %s" % (name, sorted(have), sorted(expect))
        self.d_re, self.d_col = to_dev(self.row_end, self.col)
        self.plan = self.new_plan()

    def new_plan(self):
        plan = K.SgPlan(self.row_left, self.row_right, self.col_left, self.d_re, self.d_col)
        assert plan.info() == {"chunks": self.chunks, "carries": self.carries, "heavy_rows": self.heavy + self.big}
        return plan


def from_degrees(deg, seed):
    deg = np.asarray(deg, dtype=np.int64)
    return np.cumsum(deg), np.random.RandomState(seed).randint(0, deg.shape[0], size=int(deg.sum()))


def straddle_degrees():
    """Light rows of degree 1, 2, 3, 31, 32, 33, 62, 63 and 64 starting at every offset within a chunk, each placed by
    a filler row (itself of degree 0..63) in front of it."""
    deg, cur = [], 0
    for o in range(CH):
        for d in (1, 2, 3, 31, 32, 33, 62, 63, 64):
            f = (o - cur) % CH
            deg += [f, d]
            cur += f + d
    return deg


def carry32_degrees():
    """A row with exactly 32 carries (the per-worker fix-up) and one with 33 (the big-row CTA), light rows around."""
    deg = [5, 17]
    s = sum(deg)
    deg.append(CH * (s // CH + 33) - s)          # (t - 1) // 64 - s // 64 = 32, ending on a chunk boundary
    deg += [3, 64, 1, 40]
    s = sum(deg)
    deg.append(CH * (s // CH + 33) + 6 - s)      # 33
    return deg + [2, 0, 7]


def build_graphs():
    gs = {}

    def whole(name, row_end, col, expect):
        gs[name] = Graph(name, row_end, col, len(row_end), expect=expect)

    whole("empty", np.zeros(10, dtype=np.int64), np.zeros(0), ())
    whole("single", *graph("single"), ())
    deg = np.random.RandomState(11).randint(0, 5, size=24)
    deg[0] = deg[-1] = 0
    assert 0 < deg.sum() < CH
    whole("tiny", *from_degrees(deg, 12), ())
    # rows end on chunk boundaries; the 10th chunk ends the edges, so the 11th is empty and owns the last three rows
    whole("aligned", *from_degrees([64, 32, 32, 128, 0, 16, 48, 32, 96, 192, 0, 0, 0], 13), ("heavy", "carries"))
    whole("straddle", *from_degrees(straddle_degrees(), 14), ())
    whole("carry32", *from_degrees(carry32_degrees(), 15), ("heavy", "big", "carries"))
    whole("ragged", *graph("ragged"), ("heavy", "big", "carries"))
    # a slice of rmat with global ids, rowLeft > 0, and its edge offsets moved past 2^32
    re_, col = graph("rmat")
    rm = Graph("rmat", re_, col, re_.shape[0], expect=("heavy", "carries"))
    k, vb, eb = oracle.partition(re_, 4)
    rl, rr, cl, cr = int(vb[1, 0]), int(vb[1, 1]), int(eb[1, 0]), int(eb[1, 1])
    shift = (1 << 32) + 2 * CH + 5
    gs["slice"] = Graph("slice", re_[rl:rr + 1] - np.uint64(cl) + np.uint64(shift), col[cl:cr + 1], rm.n,
                        row_left=rl, col_left=shift, expect=("heavy", "carries"), full=rm)
    assert rl > 0 and gs["slice"].col_left >= 1 << 32
    assert gs["aligned"].E % CH == 0 and (gs["carry32"].heavy, gs["carry32"].big) == (1, 1)
    return gs


_GRAPHS = None


def graphs():
    global _GRAPHS
    if _GRAPHS is None:
        _GRAPHS = build_graphs()
    return _GRAPHS


# ----------------------------------------------------------------------------------------------------- buffers ---
def exact(rng, rows, h):
    """Multiples of 1/16 in [-8, 8]: every partial sum of up to 2^15 of them is exact in fp32."""
    return (rng.randint(-128, 129, size=(rows, h)) / 16.0).astype(np.float32)


def in_ld(h, vec):
    return r4(h) + 4 if vec else (h + 1 if (h + 1) % 4 else h + 2)


def out_ld(h, vec):
    return r4(h) + 4 if vec else (h + 4 if h % 4 else h + 5)


def dev_in(a, vec, ld=None):
    """a on the device with NaN in its pad columns: ld = round_up(H, 4) + 4 (vector path), else ld % 4 != 0."""
    h = a.shape[1]
    t = torch.full((a.shape[0], ld or in_ld(h, vec)), float("nan"), device=DEV)
    t[:, :h] = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)
    return t[:, :h]


class Guarded:
    """A [rows][h] output view of a buffer with one guard row above and below and columns past h, all holding a
    sentinel.  `valid`: the columns a call may write (round_up(H, 4) on the vector path, H on the scalar path)."""

    def __init__(self, rows, h, ld, valid, index=False):
        self.rows, self.valid = rows, valid
        if index:
            self.buf = torch.full((rows + 2, ld), SENT_I, dtype=torch.int32, device=DEV)
        else:
            self.buf = torch.full((rows + 2, ld), SENT_F, device=DEV)
        self.view = self.buf[1:rows + 1, :h]

    def bits(self):
        return self.buf.cpu().view(torch.int32).numpy()

    def host(self):
        return self.view.cpu().numpy()

    def check_guards(self, what):
        b = self.bits()
        sent = np.int32(SENT_I) if self.buf.dtype == torch.int32 else np.float32(SENT_F).view(np.int32)
        keep = np.ones(b.shape, dtype=bool)
        keep[1:self.rows + 1, :self.valid] = False
        bad = keep & (b != sent)
        assert not bad.any(), "%s: %d elements outside the output window changed, first at %s" % (
            what, int(bad.sum()), np.argwhere(bad)[0])


def guarded(rows, h, vec, index=False):
    return Guarded(rows, h, out_ld(h, vec), r4(h) if vec else h, index)


def no_new_nan(got, want, what):
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: NaN where the reference has none (or v.v.)" % what


# ------------------------------------------------------------------------------------------------ launch lists ---
RAN, SEEN = set(), set()


def launches(what, want):
    """The hook's list for the last call against `want` [(kind, red, vec, L, NCH, grid)]; records what ran."""
    got = [(l["kind"], l["red"], l["vec"], l["lanes"], l["nch"], l["grid"]) for l in K.sg_launches()]
    assert got == want, "%s: launched\n  %s\nexpected\n  %s" % (what, got, want)
    SEEN.update(x[:5] for x in got)


def fixups(g, fix, vec, lanes, nch, heads=False):
    out = []
    if g.heavy:
        out.append(("heads_fixup" if heads else "fixup", fix, vec, lanes, nch, cdiv(g.heavy, 256 // lanes)))
    if g.big:
        out.append(("heads_big_fixup" if heads else "big_fixup", fix, vec, lanes, nch, g.big))
    return out


def main_launch(g, red, vec, q):
    lanes, nch = shape(q)
    if vec == 4 and red == SUM and lanes == 32 and nch <= 2:
        return [("ring", SUM, 4, 32, nch, cdiv(g.chunks, 4))]
    return [("main", red, vec, lanes, nch, cdiv(g.chunks, 256 // lanes))]


def expect_planned(g, red, vec, h):
    """Sum, max / min and their backward: per column block the main kernel, then the fix-ups of the rows it cut."""
    vw = 4 if vec else 1
    block = 256 if not vec else 1024 if red == SUM else 512
    want = []
    for c0 in range(0, h, block):
        q = cdiv(min(h - c0, block), vw)
        want += main_launch(g, red, vw, q)
        want += fixups(g, red if red in (MAX, MIN) else SUM, vw, *shape(q))
    return want


def expect_attn_fwd(g, vec, h, heads):
    vw = 4 if vec else 1
    want = main_launch(g, ASTAT, 1, heads)
    if g.heavy + g.big:
        want.append(("stat_fixup", ASTAT, 1, 32, 1, cdiv(g.heavy + g.big, 8)))
    q = cdiv(h, vw)
    return want + main_launch(g, ATTN, vw, q) + fixups(g, SUM, vw, *shape(q))


def expect_attn_bwd(g, vec, h, heads, self_base):
    vw = 4 if vec else 1
    q = cdiv(h, vw)
    lanes, nch = shape(q)
    n = max(g.id_end, self_base + g.nloc)
    want = [("record", -1, vw, lanes, nch, cdiv(n, 256 // lanes))]
    want += main_launch(g, ADST, vw, q) + fixups(g, SUM, 1, 8, 1, heads=True)
    want += main_launch(g, ASRC, vw, q) + fixups(g, SUM, vw, lanes, nch) + fixups(g, SUM, 1, 8, 1, heads=True)
    return want


def every_instantiation():
    """Every (kind, red, VEC, L, NCH) the table can produce."""
    want = set()
    for vec in (4, 1):
        for red in (SUM, MAX, MIN, MASK, ATTN, ADST, ASRC):
            for qc, lanes, nch in RUNGS:
                if qc <= max_q(vec, red):
                    ring = vec == 4 and red == SUM and lanes == 32 and nch <= 2
                    want.add(("ring" if ring else "main", red, vec, lanes, nch))
                    if red in (SUM, MAX, MIN):
                        want |= {(k, red, vec, lanes, nch) for k in ("fixup", "big_fixup")}
                    if red == ATTN:
                        want.add(("record", -1, vec, lanes, nch))
    want |= {("main", ASTAT, 1, 4, 1), ("main", ASTAT, 1, 8, 1), ("stat_fixup", ASTAT, 1, 32, 1),
             ("heads_fixup", SUM, 1, 8, 1), ("heads_big_fixup", SUM, 1, 8, 1)}
    return want


# ---------------------------------------------------------------------------------------------------- the matrix ---
# widths at both ends of every rung, and column blocks whose remainders land on different rungs
SUM_V = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 1024, 1025, 1324, 2051]
SCALAR = [1, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 300]
MM_V = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 700]
ATTN_V = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512]
ATTN_S = [1, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256]
CASES = ([("sum", True, h) for h in SUM_V] + [("sum", False, h) for h in SCALAR] +
         [("minmax", True, h) for h in MM_V] + [("minmax", False, h) for h in SCALAR] +
         [("attn", True, h) for h in ATTN_V] + [("attn", False, h) for h in ATTN_S])


def case_id(c):
    return "%s-%s-%d" % (c[0], "vec" if c[1] else "scalar", c[2])


def repeat_same(first, again, what):
    for a, b in zip(first, again):
        assert np.array_equal(a.bits(), b.bits()), "%s: a repeated call gave different bits" % what


@pytest.mark.parametrize("h", SUM_V, ids=str)
@pytest.mark.parametrize("vec", [True], ids=["vec"])
def test_sum_vector(vec, h):
    run_sum(vec, h)


@pytest.mark.parametrize("h", SCALAR, ids=str)
@pytest.mark.parametrize("vec", [False], ids=["scalar"])
def test_sum_scalar(vec, h):
    run_sum(vec, h)


def run_sum(vec, h):
    for g in graphs().values():
        rng = np.random.RandomState(h * 7 + g.nloc)
        x = exact(rng, g.n, h)
        xd = dev_in(x, vec)
        want = oracle.scatter_gather(g.row_left, g.row_right, g.col_left, g.row_end, g.col, x)
        with np.errstate(divide="ignore", invalid="ignore"):
            normed = want / np.sqrt(g.deg.astype(np.float32))[:, None]          # degree 0: 0 / 0 = NaN (quirk Q5)
        for epi, ref in ((0, want), (NORM, normed), (NORM | RELU, np.maximum(normed, np.float32(0)))):
            what = "%s sum H=%d %s epi=%d" % (g.name, h, "vec" if vec else "scalar", epi)
            outs = []
            for _ in range(2):
                o = guarded(g.nloc, h, vec)
                g.plan.forward(xd, out=o.view, epilogue=epi)
                launches(what, expect_planned(g, SUM, vec, h))
                outs.append(o)
            got = outs[0].host()
            assert ref.dtype == np.float32
            bad = ~((got == ref) | (np.isnan(got) & np.isnan(ref)))
            assert not bad.any(), "%s: %d/%d elements differ from the exact reference, first at %s (%r vs %r)" % (
                what, int(bad.sum()), bad.size, np.argwhere(bad)[0], got[bad][0], ref[bad][0])
            outs[0].check_guards(what)
            repeat_same(outs[:1], outs[1:], what)
    RAN.add(case_id(("sum", vec, h)))


def minmax_call(plan, xd, aggr, rows, h, vec):
    o, a = guarded(rows, h, vec), guarded(rows, h, vec, index=True)
    plan.minmax_forward(xd, aggr, out=o.view, arg=a.view)
    return o, a


@pytest.mark.parametrize("h", MM_V, ids=str)
@pytest.mark.parametrize("vec", [True], ids=["vec"])
def test_minmax_vector(vec, h):
    run_minmax(vec, h)


@pytest.mark.parametrize("h", SCALAR, ids=str)
@pytest.mark.parametrize("vec", [False], ids=["scalar"])
def test_minmax_scalar(vec, h):
    run_minmax(vec, h)


def run_minmax(vec, h):
    """Max and min (values and indices bit-exact, ties resolved to the first edge) and their backward (exact)."""
    for g in graphs().values():
        rng = np.random.RandomState(h * 11 + g.nloc)
        x, gy = exact(rng, g.n, h), exact(rng, g.n, h)
        xd, gd = dev_in(x, vec), dev_in(gy, vec)
        for aggr, red in ((_lib.AGGR_MAX, MAX), (_lib.AGGR_MIN, MIN)):
            what = "%s %s H=%d %s" % (g.name, "max" if red == MAX else "min", h, "vec" if vec else "scalar")
            want, warg = mmo.forward(g.row_left, g.row_right, g.col_left, g.row_end, g.col, x, aggr)
            runs = []
            for _ in range(2):
                runs.append(minmax_call(g.plan, xd, aggr, g.nloc, h, vec))
                launches(what, expect_planned(g, red, vec, h))
            o, a = runs[0]
            assert np.array_equal(o.host().view(np.int32), want.view(np.int32)), "%s: values differ" % what
            assert np.array_equal(a.host().view(np.uint32), warg), "%s: indices differ" % what
            o.check_guards(what)
            a.check_guards(what + " arg")
            repeat_same(runs[0], runs[1], what)
            # the backward gathers the indices of every id: the forward's own for a whole graph, else the whole graph's
            if g.full is None:
                arg_all, warg_all = a.view, warg
            else:
                _, warg_all = mmo.forward(0, g.full.n - 1, 0, g.full.row_end, g.full.col, x, aggr)
                arg_all = minmax_call(g.full.plan, xd, aggr, g.full.n, h, vec)[1].view
            wgrad = mmo.backward(g.row_left, g.row_right, g.col_left, g.row_end, g.col, gy, warg_all,
                                 self_base=g.self_base)
            what = what + " backward"
            grads = []
            for _ in range(2):
                o2 = guarded(g.nloc, h, vec)
                g.plan.minmax_backward(gd, arg_all, self_base=g.self_base, out=o2.view)
                launches(what, expect_planned(g, MASK, vec, h))
                grads.append(o2)
            got = grads[0].host()
            bad = got != wgrad
            assert not bad.any(), "%s: %d/%d elements differ from the exact reference, first at %s" % (
                what, int(bad.sum()), bad.size, np.argwhere(bad)[0])
            grads[0].check_guards(what)
            repeat_same(grads[:1], grads[1:], what)
    RAN.add(case_id(("minmax", vec, h)))


def scores_dev(s):
    """score / stats inputs: [*][2 heads] with NaN in 3 pad columns."""
    return dev_in(s, False, ld=s.shape[1] + 3)


def attn_call(plan, xd, sd, heads, h, vec, rows, self_base):
    o, st = guarded(rows, h, vec), Guarded(rows, 2 * heads, 2 * heads + 4, 2 * heads)
    plan.attn_forward(xd, sd, heads, SLOPE, self_base=self_base, out=o.view, stats=st.view)
    return o, st


def attn_bwd_call(plan, xd, sd, o_all, st_all, gd, heads, h, vec, rows, self_base):
    ig, sg = guarded(rows, h, vec), Guarded(rows, 2 * heads, 2 * heads + 4, 2 * heads)
    plan.attn_backward(xd, sd, o_all, st_all, gd, heads, SLOPE, self_base=self_base, in_grad=ig.view,
                       score_grad=sg.view)
    return ig, sg


def attn_close(got, want, mag, what, eps):
    no_new_nan(got, want, what)
    close_terms(got, want, mag, what, eps)


@pytest.mark.parametrize("h", ATTN_V, ids=str)
@pytest.mark.parametrize("vec", [True], ids=["vec"])
def test_attn_vector(vec, h):
    run_attn(vec, h)


@pytest.mark.parametrize("h", ATTN_S, ids=str)
@pytest.mark.parametrize("vec", [False], ids=["scalar"])
def test_attn_scalar(vec, h):
    run_attn(vec, h)


def run_attn(vec, h):
    """Forward and backward at every valid head count, against the fp64 oracle (test_attn_gpu.check's bounds)."""
    for g in graphs().values():
        for heads in valid_heads(h):
            rng = np.random.RandomState(h * 13 + heads + g.nloc)
            x, gy = exact(rng, g.n, h), exact(rng, g.n, h)
            s = rng.randn(g.n, 2 * heads).astype(np.float32)
            xd, gd, sd = dev_in(x, vec), dev_in(gy, vec), scores_dev(s)
            what = "%s attention H=%d heads=%d %s" % (g.name, h, heads, "vec" if vec else "scalar")
            kw = dict(self_base=g.self_base, col_left=g.col_left)
            fw = []
            for _ in range(2):
                fw.append(attn_call(g.plan, xd, sd, heads, h, vec, g.nloc, g.self_base))
                launches(what + " forward", expect_attn_fwd(g, vec, h, heads))
            out, stats = fw[0]
            want, wstats = ao.forward(g.row_end, g.col, x, s, heads, SLOPE, **kw)
            mag = ao.forward(g.row_end, g.col, np.abs(x), s, heads, SLOPE, **kw)[0]
            attn_close(out.host(), want, mag, what + " forward", 0.0)
            no_new_nan(stats.host(), wstats, what + " stats")
            rel_close(stats.host(), wstats, rtol=1e-4, what=what + " stats")
            for b in (out, stats):
                b.check_guards(what + " forward")
            repeat_same(fw[0], fw[1], what + " forward")
            # the backward reads out / stats of every id: the forward's own for a whole graph, else the whole graph's
            if g.full is None:
                o_all, st_all = out.view, stats.view
            else:
                o_all, st_all = (b.view for b in attn_call(g.full.plan, xd, sd, heads, h, vec, g.full.n, 0))
            bw = []
            for _ in range(2):
                bw.append(attn_bwd_call(g.plan, xd, sd, o_all, st_all, gd, heads, h, vec, g.nloc, g.self_base))
                launches(what + " backward", expect_attn_bwd(g, vec, h, heads, g.self_base))
            ig, sg = bw[0]
            args = (g.row_end, g.col, x, s, o_all.cpu().numpy(), st_all.cpu().numpy())
            wig, wsg = ao.backward(*args, gy, heads, SLOPE, **kw)
            mig = ao.backward(*args, np.abs(gy), heads, SLOPE, **kw)[0]
            msg = ao.score_grad_magnitude(*args, gy, heads, SLOPE, **kw)
            attn_close(ig.host(), wig, mig, what + " input gradient", 0.0)
            sgh = sg.host()
            attn_close(sgh[:, :heads], wsg[:, :heads], msg[:, :heads], what + " d s_dst", 1e-6)
            attn_close(sgh[:, heads:], wsg[:, heads:], msg[:, heads:], what + " d s_src", 1e-6)
            for b in (ig, sg):
                b.check_guards(what + " backward")
            repeat_same(bw[0], bw[1], what + " backward")
    RAN.add(case_id(("attn", vec, h)))


# ----------------------------------------------------------------------------------------------- one long plan ---
def run_step(plan, g, step, inputs):
    """One call of the sequence below on `plan` -> its guarded outputs."""
    kind, vec, h = step[:3]
    x, gy, arg, s, o_all, st_all = (inputs[k] for k in ("x", "gy", "arg", "s", "o", "st"))
    xd, gd = x[(vec, h)], gy[(vec, h)]
    if kind == "sum":
        o = guarded(g.nloc, h, vec)
        plan.forward(xd, out=o.view, epilogue=step[3])
        return [o]
    if kind in ("max", "min"):
        return list(minmax_call(plan, xd, _lib.AGGR_MAX if kind == "max" else _lib.AGGR_MIN, g.nloc, h, vec))
    if kind == "mask":
        o = guarded(g.nloc, h, vec)
        plan.minmax_backward(gd, arg[(vec, h)], self_base=step[3], out=o.view)
        return [o]
    heads, self_base = step[3], step[4]
    sd = s[heads]
    fw = attn_call(plan, xd, sd, heads, h, vec, g.nloc, self_base)
    bw = attn_bwd_call(plan, xd, sd, o_all[(vec, h)], st_all[heads], gd, heads, h, vec, g.nloc, self_base)
    return list(fw) + list(bw)


def run_sequence(g, steps, rows, reserve):
    """Runs `steps` on one plan, on a side stream, after reserving it for width `reserve`, and each step on a fresh
    plan on the default stream; the outputs must agree bit for bit."""
    rng = np.random.RandomState(77)
    inputs = {k: {} for k in ("x", "gy", "arg", "s", "o", "st")}
    for step in steps:
        kind, vec, h = step[:3]
        key = (vec, h)
        if key not in inputs["x"]:
            inputs["x"][key] = dev_in(exact(rng, rows, h), vec)
            inputs["gy"][key] = dev_in(exact(rng, rows, h), vec)
            inputs["o"][key] = dev_in(exact(rng, rows, h), vec)
            a = guarded(rows, h, vec, index=True)
            ids = rng.randint(g.self_base, g.self_base + g.nloc, size=(rows, h))    # often a local row's own id
            a.view.copy_(torch.from_numpy(ids.astype(np.int32)))
            inputs["arg"][key] = a.view
        if kind == "attn" and step[3] not in inputs["s"]:
            heads = step[3]
            inputs["s"][heads] = scores_dev(rng.randn(rows, 2 * heads).astype(np.float32))
            st = np.concatenate([rng.randn(rows, heads), rng.uniform(0.05, 1.0, (rows, heads))], axis=1)
            inputs["st"][heads] = scores_dev(st.astype(np.float32))
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        plan = g.new_plan()
        plan.reserve(reserve)
    for i, step in enumerate(steps):
        with torch.cuda.stream(side):
            got = run_step(plan, g, step, inputs)
        side.synchronize()
        fresh = g.new_plan()
        want = run_step(fresh, g, step, inputs)
        torch.cuda.synchronize()
        fresh.close()
        for k, (a, b) in enumerate(zip(got, want)):
            assert np.array_equal(a.bits(), b.bits()), "%s step %d %s output %d: the long-lived plan differs from a " \
                                                       "fresh one" % (g.name, i, step, k)
    plan.close()


def test_one_plan_for_every_call():
    """Reserve-then-grow (the reserved carries are released on the stream), carries grown by attention and the
    index carries sized from them, shrinking widths, both paths, head counts 1 -> 8 -> 2, and selfBase moved past
    the ids the graph has (the attention record grows)."""
    g = graphs()["slice"]
    rl = g.self_base
    rows = g.n + g.nloc + 8                    # ids up to selfBase + nloc with selfBase = n
    steps = [("sum", True, 8, NORM), ("max", True, 100), ("mask", True, 100, rl), ("attn", False, 37, 1, rl),
             ("sum", False, 257, 0), ("attn", True, 512, 8, rl), ("min", True, 513), ("mask", True, 513, rl + 3),
             ("attn", True, 64, 2, g.n), ("mask", False, 33, rl + 5), ("sum", True, 4, NORM | RELU),
             ("max", False, 5), ("attn", False, 256, 8, rl), ("sum", True, 1025, 0), ("attn", True, 64, 2, rl)]
    run_sequence(g, steps, rows, 8)


def test_zero_carry_plan_through_attention():
    """A plan with no carries: every buffer the carries would need stays empty, through reserve and every pass."""
    g = graphs()["tiny"]
    assert g.carries == 0
    steps = [("attn", True, 8, 1, 0), ("attn", True, 256, 8, 0), ("attn", False, 64, 2, 0), ("sum", True, 700, 0),
             ("max", False, 300), ("attn", False, 1, 1, 3)]
    run_sequence(g, steps, g.n + 8, 64)


# ---------------------------------------------------------------------------------------------------- coverage ---
def test_matrix_covered():
    """Every main-kernel and fix-up instantiation the row-shape table can produce was reached, and the matrix ran
    every case."""
    wanted = {case_id(c) for c in CASES}
    if not wanted <= RAN:
        pytest.skip("%d of the %d matrix cases did not run in this process" % (len(wanted - RAN), len(wanted)))
    missing = every_instantiation() - SEEN
    assert not missing, "never launched: %s" % sorted(missing)
    assert SEEN <= every_instantiation(), "launched outside the table: %s" % sorted(SEEN - every_instantiation())
