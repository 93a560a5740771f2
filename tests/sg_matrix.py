"""The harness of the ScatterGather GPU matrices (test_sg_matrix_gpu.py, test_exact_gpu.py, test_weighted_gpu.py):
the graphs they run on, the launch lists their calls must make, and the buffers and comparisons they share.

The row-shape table (sg.cu, with_shape) maps a row of Q T-columns (float4 on the vector path, float on the scalar
path) to L lanes and NCH chunks per lane: Q <= 4 -> (4, 1), <= 8 -> (8, 1), <= 16 -> (16, 1), <= 32 -> (32, 1),
<= 64 -> (32, 2), <= 128 -> (32, 4), <= 256 -> (32, 8).  REDS restates, independently of sg.cu's SG_REDS, what each
reduction's row there decides about the launches: the widest row one launch takes, the ring form, the fix-ups of the
H-wide partials and of the heads-wide ones.  The rest of a row (gathers in flight, CTAs per SM, carries) does not show
in a launch list, so it is not restated."""
import functools
from typing import NamedTuple

import numpy as np
import torch

import weighted_oracle as wo
from oracle import oracle
from roc_b200 import _lib
from roc_b200 import kernels as K
from sg_graphs import graph, to_dev

DEV = "cuda"
CH, BIG = 64, 32                         # edges per chunk; the most carries a row finished by one worker has
SLOPE = 0.2
SUM, MAX, MIN, MASK, ASTAT, ATTN, ADST, ASRC, WSUM, EDOT, TSUM, TMASK = range(12)
NORM, RELU = _lib.SG_EPI_NORM, _lib.SG_EPI_RELU
SENT_F = -1234.5                         # the sentinel of float outputs
SENT_I = 0x5A5A5A5A                      # and of index outputs
RUNGS = ((4, 4, 1), (8, 8, 1), (16, 16, 1), (32, 32, 1), (64, 32, 2), (128, 32, 4), (256, 32, 8))
# scalar-path widths at both ends of every rung, and one column block past the widest
SCALAR = [1, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 300]


def r4(h):
    return (h + 3) // 4 * 4


def cdiv(a, b):
    return (a + b - 1) // b


def shape(q):
    """(L, NCH) of a row of q T-columns."""
    for qc, lanes, nch in RUNGS:
        if q <= qc:
            return lanes, nch
    raise ValueError(q)


# -------------------------------------------------------------------------------------------- reduction table ---
class Red(NamedTuple):
    q4: int            # the widest row, in T-columns, one launch takes on float4 rows (0: never on float4 rows)
    q1: int            # and on scalar rows
    ring: bool         # float4 rows at L = 32, NCH <= 2 run on the ring kernel
    fix: str           # the fix-up of cut rows: "own" (instantiated for the reduction), "sum", "stats" or None
    heads_fix: bool    # heads-wide partials, finished by the sum's fix-ups at VEC = 1, L = 8


REDS = {
    #            q4   q1   ring   fix      heads_fix
    SUM:   Red(256, 256, True,  "sum",   False),
    MAX:   Red(128, 256, False, "own",   False),
    MIN:   Red(128, 256, False, "own",   False),
    MASK:  Red(128, 256, False, "sum",   False),
    ASTAT: Red(0,   8,   False, "stats", False),      # one score per head
    ATTN:  Red(128, 256, False, "sum",   False),
    ADST:  Red(128, 256, False, None,    True),
    ASRC:  Red(128, 256, False, "sum",   True),
    WSUM:  Red(256, 256, False, "sum",   False),
    EDOT:  Red(128, 256, False, None,    False),      # one output per edge: nothing carried
    TSUM:  Red(256, 256, True,  "own",   False),
    TMASK: Red(128, 256, False, "sum",   False),
}


def max_q(red, vec):
    return REDS[red].q4 if vec == 4 else REDS[red].q1


# ----------------------------------------------------------------------------------------------------- graphs ---
class Sched(NamedTuple):
    chunks: int
    carries: int
    heavy: int         # cut rows of at most BIG carries (one worker each)
    big: int           # cut rows of more (one CTA each)


def schedule(row_end, col_left=0):
    """The chunk schedule of a plan over row_end, from the definitions in sg.cu."""
    t = np.asarray(row_end, dtype=np.int64) - col_left
    s = np.concatenate([[0], t[:-1]])
    deg = t - s
    carries = np.where(deg > CH, (t - 1) // CH - s // CH, 0)
    e = int(t[-1]) if t.shape[0] else 0
    return Sched(e // CH + 1, int(carries.sum()), int(((deg > CH) & (carries <= BIG)).sum()),
                 int((carries > BIG).sum()))


class Graph:
    """One plan's CSR: row_end holds its rows' END offsets in the edge array (global; the plan's edges start at
    col_left), col their sources, ids < n.  The chunk schedule is recomputed here and must match the plan's.
    `expect`: the parts of the schedule ("heavy", "big", "carries") the graph was built to have."""

    def __init__(self, name, row_end, col, n, row_left=0, col_left=0, expect=None, full=None, plan=None):
        self.name, self.n, self.row_left, self.col_left, self.full = name, n, row_left, col_left, full
        self.row_end, self.col = np.asarray(row_end, np.uint64), np.asarray(col, np.uint32)
        self.nloc, self.E = self.row_end.shape[0], self.col.shape[0]
        self.row_right = row_left + self.nloc - 1
        self.self_base = row_left
        self.deg = np.diff(np.concatenate([[0], self.row_end.astype(np.int64) - col_left]))
        assert int(self.deg.sum()) == self.E
        self.sched = schedule(self.row_end, col_left)
        self.id_end = int(self.col.max()) + 1 if self.E else 0
        if expect is not None:
            have = {k for k in ("heavy", "big", "carries") if getattr(self.sched, k)}
            assert have == set(expect), "%s: the graph has %s, its definition says %s" % (
                name, sorted(have), sorted(expect))
        self.d_re, self.d_col = to_dev(self.row_end, self.col)
        self.plan = plan if plan is not None else self.new_plan()

    def new_plan(self):
        plan = K.SgPlan(self.row_left, self.row_right, self.col_left, self.d_re, self.d_col)
        s = self.sched
        assert plan.info() == {"chunks": s.chunks, "carries": s.carries, "heavy_rows": s.heavy + s.big}
        return plan


class WGraph(Graph):
    """A graph with its transpose, and the transpose's schedule, when it is a whole graph."""

    def __init__(self, name, row_end, col, n, row_left=0, col_left=0, plan=None):
        super().__init__(name, row_end, col, n, row_left, col_left, plan=plan)
        self.whole = row_left == 0 and col_left == 0 and self.nloc == n
        self.tr = None
        if self.whole:
            self.tr = K.SgTranspose(self.d_re, self.d_col)
            self.re_t, self.col_t, self.perm = wo.transpose(self.row_end, self.col, n)
            self.sched_t = schedule(self.re_t)


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


@functools.cache
def graphs():
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
    assert gs["aligned"].E % CH == 0 and (gs["carry32"].sched.heavy, gs["carry32"].sched.big) == (1, 1)
    return gs


def directed_dup(n, e, seed):
    rng = np.random.RandomState(seed)
    dst = np.sort(rng.randint(0, n, size=e))
    src = rng.randint(0, n - 3, size=e)                     # the last three nodes have no out-edge
    src[1::3] = src[0::3][:src[1::3].shape[0]]              # duplicate edges
    dst[:200] = 5                                           # one heavy row of duplicates
    dst = np.sort(dst)
    order = np.lexsort((src, dst))
    return np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64), src[order].astype(np.uint32)


def symmetric_sorted(n, p, seed):
    rng = np.random.RandomState(seed)
    a = rng.rand(n, n) < p
    a = a | a.T
    a[:40, :40] = True                                      # heavy rows
    return (np.cumsum(a.sum(axis=1)).astype(np.uint64),
            np.concatenate([np.nonzero(a[i])[0] for i in range(n)]).astype(np.uint32))


@functools.cache
def wgraphs():
    """Every matrix graph (on its own plan), a directed multigraph and a hub whose sources fan out."""
    gs = {g.name: WGraph(g.name, g.row_end, g.col, g.n, g.row_left, g.col_left, plan=g.plan)
          for g in graphs().values()}
    gs["directed"] = WGraph("directed", *directed_dup(3000, 40000, 21), 3000)
    hub = np.zeros(300, dtype=np.int64)
    hub[7] = 4000                                           # long transposed rows too
    re_ = np.cumsum(hub).astype(np.uint64)
    col = np.random.RandomState(3).randint(0, 40, size=4000).astype(np.uint32)
    gs["hub"] = WGraph("hub", re_, col, 300)
    d = gs["directed"]
    assert d.re_t[-1] == d.re_t[-4]                         # empty transposed rows
    dst = np.repeat(np.arange(d.n), d.deg)
    pairs = dst.astype(np.int64) * d.n + d.col
    assert np.unique(pairs).shape[0] < pairs.shape[0]      # duplicate (dst, src) edges
    return gs


@functools.cache
def xgraphs():
    """Every whole graph of wgraphs() plus a fan-out graph whose one source feeds 3,000 rows."""
    gs = {k: g for k, g in wgraphs().items() if g.whole}
    n = 4000
    rng = np.random.RandomState(17)
    deg = rng.randint(0, 4, size=n)
    deg[:3000] += 1                                      # rows 0..2999 each take an edge from the hub 3999
    deg[3000:3100] = 0
    col = []
    for r in range(n):
        k = int(deg[r])
        srcs = list(rng.randint(0, 3000, size=k - 1 if r < 3000 else k)) + ([3999] if r < 3000 else [])
        rng.shuffle(srcs)
        col += srcs
    gs["fanout"] = WGraph("fanout", np.cumsum(deg).astype(np.uint64), np.array(col, np.uint32), n)
    assert gs["fanout"].sched_t.big >= 1                 # a big transposed row
    return gs


# ----------------------------------------------------------------------------------------------- launch lists ---
def launches(what, want, seen):
    """The hook's list for the last call against `want` [(kind, red, vec, L, NCH, grid)]; adds what ran to `seen`."""
    got = [(l["kind"], l["red"], l["vec"], l["lanes"], l["nch"], l["grid"]) for l in K.sg_launches()]
    assert got == want, "%s: launched\n  %s\nexpected\n  %s" % (what, got, want)
    seen.update(x[:5] for x in got)


def fixups(s, fix, vec, lanes, nch, heads=False):
    out = []
    if s.heavy:
        out.append(("heads_fixup" if heads else "fixup", fix, vec, lanes, nch, cdiv(s.heavy, 256 // lanes)))
    if s.big:
        out.append(("heads_big_fixup" if heads else "big_fixup", fix, vec, lanes, nch, s.big))
    return out


def launch(s, red, vec, q):
    """One launch of reduction `red` over rows of q T-columns of `vec` floats on a plan of schedule s: the main kernel,
    then the fix-ups of the rows it cut."""
    r = REDS[red]
    lanes, nch = shape(q)
    if vec == 4 and r.ring and lanes == 32 and nch <= 2:
        want = [("ring", red, 4, 32, nch, cdiv(s.chunks, 4))]
    else:
        want = [("main", red, vec, lanes, nch, cdiv(s.chunks, 256 // lanes))]
    if r.fix == "stats":
        if s.heavy + s.big:
            want.append(("stat_fixup", red, 1, 32, 1, cdiv(s.heavy + s.big, 8)))
    elif r.fix:
        want += fixups(s, red if r.fix == "own" else SUM, vec, lanes, nch)
    if r.heads_fix:
        want += fixups(s, SUM, 1, 8, 1, heads=True)
    return want


def planned(s, red, vec, h):
    """A call that runs one reduction over H = h columns (the sums, max / min and their backwards, plain and over a
    transpose, the weighted sum and the edge dot): one launch per column block of the widest row it takes."""
    vw = 4 if vec else 1
    block = vw * max_q(red, vw)
    return [x for c0 in range(0, h, block) for x in launch(s, red, vw, cdiv(min(h - c0, block), vw))]


def attn_forward(s, vec, h, heads):
    vw = 4 if vec else 1
    return launch(s, ASTAT, 1, heads) + launch(s, ATTN, vw, cdiv(h, vw))


def attn_backward(s1, s2, vec, h, n):
    """The node records of ids [0, n), B1 over a plan of schedule s1 and B2 over one of s2 (the same plan for the
    gather backward, the transposed one for the exact backward)."""
    vw = 4 if vec else 1
    q = cdiv(h, vw)
    lanes, nch = shape(q)
    return [("record", -1, vw, lanes, nch, cdiv(n, 256 // lanes))] + launch(s1, ADST, vw, q) + launch(s2, ASRC, vw, q)


def weighted_backward(g, vec, h):
    """The weights' permutation into transposed edge order, then the weighted sum over the transpose."""
    pre = [("permute", -1, 1, 1, 1, cdiv(g.E, 256))] if g.E else []
    return pre + planned(g.sched_t, WSUM, vec, h)


def every_instantiation(reductions):
    """Every (kind, red, VEC, L, NCH) the calls of `reductions` can launch: each reduction at every rung up to its
    widest row on both paths, on a schedule with heavy and big rows.  The attention backward's node records run in
    ADST's shapes."""
    every = Sched(chunks=1, carries=1, heavy=1, big=1)
    want = set()
    for red in reductions:
        for vec in (4, 1):
            for qc, lanes, nch in RUNGS:
                if qc <= max_q(red, vec):
                    want |= {x[:5] for x in launch(every, red, vec, qc)}
                    if red == ADST:
                        want.add(("record", -1, vec, lanes, nch))
    return want


# ---------------------------------------------------------------------------------------------------- buffers ---
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


def scores_dev(s):
    """score / stats inputs: [*][2 heads] with NaN in 3 pad columns."""
    return dev_in(s, False, ld=s.shape[1] + 3)


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


# ------------------------------------------------------------------------------------------------ comparisons ---
def same_bits(a, b, what):
    """Two calls' Guarded outputs hold the same bits, guards included."""
    assert np.array_equal(a.bits(), b.bits()), "%s: a repeated call gave different bits" % what


def check_bits(got, want, what):
    """got equals the exact fp32 reference, NaN where it has NaN."""
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    assert not bad.any(), "%s: %d/%d elements differ from the exact reference, first at %s (%r vs %r)" % (
        what, int(bad.sum()), bad.size, np.argwhere(bad)[0], got[bad][0], want[bad][0])


def no_new_nan(got, want, what):
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: NaN where the reference has none (or v.v.)" % what


def close_terms(got, want, mag, what, eps):
    """The parity bar, plus `eps` of the magnitude of the summed terms (`mag`: the same sums over |terms|).  A sum
    whose terms cancel is only good to its rounding relative to them, not to the result."""
    err = np.abs(np.asarray(got, dtype=np.float64) - want)
    bound = 1e-4 * np.abs(want) + 1e-5 * np.abs(want).max() + eps * mag + 1e-30
    bad = err > bound
    assert not bad.any(), "%s: %d/%d elements off; worst err %.3e at %s" % (
        what, int(bad.sum()), bad.size, float(err.max()), np.unravel_index((err - bound).argmax(), err.shape))


def valid_heads(h):
    """The head counts the attention kernels take at width h."""
    return [k for k in (1, 2, 4, 8) if k == 1 or (h % k == 0 and (h // k) >= 4 and (h // k) & (h // k - 1) == 0)]
