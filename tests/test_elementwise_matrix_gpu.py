"""The per-step elementwise kernels (elementwise.cu) and the row copies (halo.cu) against fp64 and exact references, at
every launch variant.

Dispatch, restated from the launchers and checked for coverage by test_dispatch_table_covered at the end:
  softmax cross-entropy  k_softmax_xent_narrow<LR = 8 / 16 / 32> for C <= 32 / 64 / 128, the warp-per-row
                         k_softmax_xent above; one-hot or index labels; with or without the fused in-degree norm.
  k_map<OP, VEC, ACC>    VEC = 4 when H, every ld and every base allow float4 (vec_ok), else 1.
  k_dropout<VEC, 2>      VEC = 4 when both ld are multiples of 4 and both bases 16-byte aligned.
  k_norm<VEC>            VEC = 4 under the same rule (whatever H is: the float4 pad columns ride along).
  k_push_rows<VEC, LR>   VEC = 4 when both ld and every base are 16-byte aligned; LR = 16 for <= 16 T-columns per row.
Each grid is capped at 16 CTAs per SM.  Most cases run with roc_set_sm_reserve leaving 8 SMs, so a few thousand rows
take many grid-stride passes; test_full_chip_passes runs one case per kernel on the whole chip at >= 3 full passes
plus a ragged tail, sized from the device's SM count.

Inputs sit in NaN-filled buffers (pad columns and a guard row above and below); outputs in sentinel-filled ones.  The
softmax, dropout, k_map, add backward, fill and copy kernels may write nothing outside their [rows][H] window.  The
float4 paths of k_norm and the three row copies store whole float4s: columns [H, round_up(H, 4)) of each output row
receive the source row's pad columns (for the norm: after the relu mask, divided by the row's divisor); nothing from
round_up(H, 4) on is written (include/roc_b200.h).  Every call runs twice and must give the same bits, except the
softmax loss, a float summed by atomics.

References (u = 2^-24):
  softmax   torch fp64 from the fp32 logits.  Logits are k/8 with |k| <= 800, so z - m is exact in fp32; rows include
            exact ties for the maximum (first index wins), spreads past 104 (p underflows to denormals and 0), missing
            and out-of-range labels, every mask value, and degrees 0, 1, 2^20 + 1 and a hub.
            |g - g64| <= 2u((C + 4) p64 + |g64|): expf within 2 ulp, the fp32 sum within (C - 1) u S in any order, one
            rounded divide; the fused norm adds u |g| after dividing by sqrtf(deg).  A floor of 4 * 2^-149 covers
            expf's 2 ulp where p is denormal.  The six counts are exact; the loss is within (C + 4 + n_train) 2^-23
            of the fp64 sum, relative.  Rows of degree 0 (divisor 0) and the whole fused result equal, bit for bit,
            the unfused kernel followed by roc_indegree_norm; three ragged row blocks called as the host calls them
            equal one call bit for bit.
  dropout   bit-exact against oracle.dropout_mask / dropout_apply, and roc_dropout_mask against the same bits.
  norm      bit-exact against numpy fp32 x / sqrt(float32(deg)) (NaN compared as NaN).
  maps      relu, add, copy and add backward bit-exact against fp32 torch (NaN, +-0 and +-inf included; relu
            forward returns the canonical NaN for a NaN input, so there NaN only has to stay NaN); sigmoid
            within 6u relative of fp64 (expf 2 ulp, the add and the divide) with a 2^-126 floor; its backward within
            3u |r| + u |out| of fp64 (three products, one add).
  scale     within 2u |(b - a) w| + u |r| of fp64.
  Adam      per element, the first-order sum of one u per fp32 operation of optimizer.cc's formula.
  copies    bit-exact against torch indexing; rows no entry names stay sentinel.

Each bound also carries 2^-50 |reference| for the fp64 reference's own roundings.

Worst |error| / bound, measured on one H100 80GB HBM3 (700 W): softmax gradient 0.48, softmax loss 0.014, sigmoid
0.58, sigmoid backward 0.998, scale 0.85, Adam 0.998.  A ratio near 1 is a single rounding of a result just above a
power of two, where half an ulp reaches the u |result| the bound allows for it.  The file runs in about 30 s."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle
from roc_b200 import _lib
from roc_b200 import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
LIB = _lib.lib
U = 2.0 ** -24
SENT = -1234.5
REF = 2.0 ** -50                        # the fp64 reference's own rounding, relative
FEW_SMS = 8
FEW_CTAS = FEW_SMS * 16                 # every elementwise grid under few_sms()
TRAIN, VAL, TEST, NONE = _lib.MASK_TRAIN, _lib.MASK_VAL, _lib.MASK_TEST, _lib.MASK_NONE

SEEN = set()        # launch variants reached, by the dispatch rules above
RAN = set()         # matrix cases that ran in this process
WORST = {}          # family -> worst |error| / bound


def nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def few_sms():
    """sm_count() = 8 for this thread's launches, so every elementwise grid has 128 CTAs (the reserve is thread-local
    and the ctypes calls run on this thread)."""
    prev = LIB.roc_set_sm_reserve(nsm() - FEW_SMS)
    try:
        yield
    finally:
        LIB.roc_set_sm_reserve(prev)


def r4(h):
    return (h + 3) // 4 * 4


def ld_of(h, layout):
    """vec: 16-byte rows with >= 4 pad columns; odd: an ld that is no multiple of 4; dense: ld = h"""
    if layout == "vec":
        return r4(h) + 4
    if layout == "odd":
        return h + 1 if (h + 1) % 4 else h + 2
    return h


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def nan_equal(a, b):
    """a and b have the same bits, or are both NaN"""
    return bool(((bits(a) == bits(b)) | (torch.isnan(a) & torch.isnan(b))).all())


class Frame:
    """A [rows][h] window at row 1, column col0 of a [rows + 2][ld] fp32 buffer filled with `fill`."""

    def __init__(self, rows, h, fill, ld, col0=0, init=None):
        self.base = torch.full((rows + 2, ld), fill, device=DEV, dtype=torch.float32)
        self.rows, self.h, self.col0 = rows, h, col0
        self.v = self.base[1:rows + 1, col0:col0 + h]
        if init is not None:
            self.v.copy_(init)
        self.init = self.base.clone()

    @property
    def ld(self):
        return self.base.stride(0)

    def wide(self, cols, t=None):
        """the first `cols` columns of the window's rows, of `t` (default: the live buffer)"""
        return (self.base if t is None else t)[1:self.rows + 1, self.col0:self.col0 + cols]

    def assert_outside_unchanged(self, cols=None, what=""):
        """nothing outside rows [0, rows) x columns [0, cols) of the window was written (cols defaults to h)"""
        changed = bits(self.base) != bits(self.init)
        changed[1:self.rows + 1, self.col0:self.col0 + (self.h if cols is None else cols)] = False
        if bool(changed.any()):
            r, c = (int(i) for i in torch.nonzero(changed)[0])
            raise AssertionError("%s: wrote outside its window, buffer row %d column %d (window %d x %d at column %d)"
                                 % (what, r, c, self.rows, self.h, self.col0))


def inp(t, layout):
    t = torch.as_tensor(t).to(DEV)
    return Frame(t.shape[0], t.shape[1], float("nan"), ld_of(t.shape[1], layout), init=t)


def outp(rows, h, layout, init=None):
    return Frame(rows, h, SENT, ld_of(h, layout), init=init)


def guarded(t, fill):
    """a 1-D device copy of t between 4 guard elements on each side, and the buffer"""
    t = torch.as_tensor(t).to(DEV)
    b = torch.full((t.numel() + 8,), fill, dtype=t.dtype, device=DEV)
    b[4:-4] = t
    return b[4:-4], b


def worst(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    return ratio


def ok(rc, what):
    assert rc == 0, "%s returned %d" % (what, rc)


# ------------------------------------------------------------------------------- softmax cross-entropy ---
SM_C = (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 300, 602)
COL_LEFT = (1 << 32) + 12345             # a partition slice's first edge, past 2^32


def sm_inst(c):
    """LR of the narrow kernel, or 0 for the warp-per-row kernel (launch_softmax)"""
    return 8 if c <= 32 else 16 if c <= 64 else 32 if c <= 128 else 0


def sm_pass_rows(c, ctas):
    return ctas * (256 // (sm_inst(c) or 32))


def sm_data(n, c, seed):
    """fp32 logits k / 8 (|k| <= 800), int32 labels (some missing: -1 or C), int32 masks, int64 in-degrees"""
    rs = np.random.RandomState(seed)
    lr = sm_inst(c) or 32
    k = rs.randint(-800, 801, size=(n, c))
    kind = rs.randint(0, 6, size=n)
    k[kind == 1] = rs.randint(-40, 41, size=((kind == 1).sum(), c))
    lab = rs.randint(0, c, size=n).astype(np.int32)
    half = rs.rand(n) < 0.5           # rows whose label is the first maximum, so a wrong argmax changes the counts
    # exact ties for the maximum: at the first and last lane of a group and in the next value slot (kind 2), and with
    # the first tied column in a later lane than the second (kind 3: lane LR - 1 of slot 0 against lane 0 of slot 1)
    for kd, cols in ((2, (0, lr - 1, lr, 2 * lr - 1, 3 * lr, c - 1)), (3, (lr - 1, lr, 2 * lr + 5, c - 2))):
        cols = np.array(sorted({x for x in cols if 0 <= x < c}), dtype=np.int64)
        rows = np.nonzero(kind == kd)[0]
        k[rows] = rs.randint(-800, 700, size=(rows.size, c))
        if cols.size:
            k[np.ix_(rows, cols)] = rs.randint(700, 801, size=(rows.size, 1))
            lab[rows] = np.where(half[rows], cols[0], cols[rs.randint(0, cols.size, size=rows.size)])
    # spread past 104 below the maximum: p runs from normal through denormal to 0
    rows = np.nonzero(kind == 4)[0]
    top = rs.randint(0, c, size=rows.size)
    k[rows] = 800 - rs.randint(688, 837, size=(rows.size, c))
    k[rows, top] = 800
    lab[rows] = np.where(half[rows], top, lab[rows])
    rows = np.nonzero(kind == 5)[0]
    k[rows, c - 1] = 800
    z = (k / 8.0).astype(np.float32)
    lab[rs.rand(n) < 0.04] = -1
    lab[rs.rand(n) < 0.03] = c
    mask = rs.randint(0, 4, size=n).astype(np.int32)
    deg = rs.randint(1, 41, size=n).astype(np.int64)
    deg[3::53] = 0
    deg[7::97] = 1
    deg[11::211] = 70000
    deg[13::401] = 2 ** 20 + 1
    return z, lab, mask, deg


def onehot(lab, c):
    oh = np.zeros((lab.shape[0], c), dtype=np.float32)
    valid = (lab >= 0) & (lab < c)
    oh[np.nonzero(valid)[0], lab[valid]] = 1.0
    return oh


def sm_ref(z, lab, mask):
    """fp64 softmax, gradient, argmax (first index of the largest logit = of the largest p: logits differ by >= 1/8)
    and metrics with the kernels' label and mask rules"""
    n, c = z.shape
    z64 = z.double()
    zmax = z64.max(1, keepdim=True).values
    e = torch.exp(z64 - zmax)
    p = e / e.sum(1, keepdim=True)
    lab = lab.long()
    valid = (lab >= 0) & (lab < c)
    lab_c = lab.clamp(0, c - 1)
    onehot_t = torch.zeros_like(p)
    onehot_t.scatter_(1, lab_c[:, None], valid[:, None].double())
    train = mask == TRAIN
    g = torch.where(train[:, None], p - onehot_t, torch.zeros((), dtype=p.dtype, device=DEV))
    cols = torch.arange(c, device=DEV)
    best = torch.where(z64 == zmax, cols, c).min(1).values
    ptrue = torch.where(valid, p.gather(1, lab_c[:, None])[:, 0], torch.zeros((), dtype=p.dtype, device=DEV))
    hit = valid & (best == lab)
    counts = [int(train.sum()), int((mask == TEST).sum()), int((mask == VAL).sum()), int((hit & train).sum()),
              int((hit & (mask == TEST)).sum()), int((hit & (mask == VAL)).sum())]
    return {"p": p, "g": g, "train": train, "counts": counts, "loss": float((1.0 - ptrue)[train].sum()),
            "n_train": counts[0]}


def sm_call(n, c, z, labels, idx, mask, g, row_end, col_left, perf):
    """the C ABI with the host's pointer arithmetic: every argument a view whose data_ptr is the block's first row"""
    pz, pg, pm = z.data_ptr(), g.data_ptr(), mask.data_ptr()
    pp = perf.data_ptr() if perf is not None else None
    if row_end is not None:
        return LIB.roc_softmax_xent_bwd_norm(n, c, pz, z.stride(0), labels.data_ptr() if labels is not None else None,
                                             labels.stride(0) if labels is not None else 0,
                                             idx.data_ptr() if idx is not None else None, pm, pg, g.stride(0),
                                             row_end.data_ptr(), col_left, pp, None)
    if labels is not None:
        return LIB.roc_softmax_xent_bwd(n, c, pz, z.stride(0), labels.data_ptr(), labels.stride(0), pm, pg, g.stride(0),
                                        pp, None)
    return LIB.roc_softmax_xent_bwd_idx(n, c, pz, z.stride(0), idx.data_ptr(), pm, pg, g.stride(0), pp, None)


def perf_of(perf):
    p = perf.cpu()
    return float(p[:1].view(torch.float32)[0]), [int(v) for v in p[1:]]


def sm_check(g, ref, div, c, what):
    """g against the fp64 reference and bound (rows of divisor 0 excluded: they are checked bit for bit)"""
    want, bnd = ref["g"], 2 * U * ((c + 4) * ref["p"] + ref["g"].abs())
    rows = torch.ones(want.shape[0], dtype=torch.bool, device=DEV)
    if div is not None:
        rows = div > 0
        d = torch.where(rows, div, torch.ones_like(div))[:, None]
        want = want / d
        bnd = bnd / d + U * want.abs()
    bnd = bnd + REF * want.abs() + 4 * 2.0 ** -149
    g = g.double()
    r = float(((g - want).abs() / bnd)[rows].max()) if bool(rows.any()) else 0.0
    assert worst("softmax gradient", r) <= 1.0, "%s: worst |error| / bound = %.3g" % (what, r)
    assert bool((g[rows & ~ref["train"]] == 0).all()), "%s: a row outside the training mask has a gradient" % what


def sm_check_metrics(loss, counts, ref, c, what):
    assert counts == ref["counts"], "%s: counts %s, want %s" % (what, counts, ref["counts"])
    bound = (c + 4 + ref["n_train"]) * 2.0 ** -23 * ref["loss"]
    err = abs(loss - ref["loss"])
    assert err <= bound, "%s: loss %.9g, fp64 %.9g" % (what, loss, ref["loss"])
    if bound > 0:
        worst("softmax loss", err / bound)


def softmax_cases(c, layout, n, data, blocks):
    """every label form x norm x perf at n rows of `data`; row blocks too when `blocks`"""
    z_np, lab_np, mask_np, deg_np = (a[:n] for a in data)
    z = inp(z_np, layout)
    oh = inp(onehot(lab_np, c), layout)
    idx, _ = guarded(lab_np, -7)
    mask, _ = guarded(mask_np, -7)
    row_end = torch.from_numpy(COL_LEFT + np.cumsum(deg_np)).to(DEV)
    div = torch.from_numpy(np.sqrt(deg_np.astype(np.float32)).astype(np.float64)).to(DEV)
    ref = sm_ref(z.v, idx, mask)
    ldg = ld_of(c, layout)
    inst = sm_inst(c)
    for form in ("onehot", "index"):
        labels, lidx = (oh.v, None) if form == "onehot" else (None, idx)
        plain = None
        for norm in (False, True):
            what = "softmax C=%d %s n=%d %s%s" % (c, layout, n, form, " norm" if norm else "")
            re_ = row_end if norm else None
            runs = []
            for _ in range(2):
                g = outp(n, c, layout)
                perf = torch.zeros(7, dtype=torch.int32, device=DEV)
                ok(sm_call(n, c, z.v, labels, lidx, mask, g.v, re_, COL_LEFT, perf), what)
                g.assert_outside_unchanged(what=what)
                runs.append((g, perf_of(perf)))
            (g, (loss, counts)), (g2, (_, counts2)) = runs
            assert same_bits(g.v, g2.v) and counts == counts2, "%s: two runs differ" % what
            sm_check(g.v, ref, div if norm else None, c, what)
            sm_check_metrics(loss, counts, ref, c, what)
            g0 = outp(n, c, layout)
            ok(sm_call(n, c, z.v, labels, lidx, mask, g0.v, re_, COL_LEFT, None), what + " perf=NULL")
            assert same_bits(g0.v, g.v), "%s: perf = NULL changes the gradient" % what
            SEEN.add(("softmax", inst, form, norm))
            if not norm:
                plain = g
                continue
            # the fused norm == the unfused kernel followed by roc_indegree_norm, bit for bit (degree 0: NaN / inf)
            want = outp(n, c, layout)
            ok(LIB.roc_indegree_norm(0, n - 1, COL_LEFT, c, row_end.data_ptr(), plain.v.data_ptr(), plain.ld,
                                     want.v.data_ptr(), want.ld, None, None), "roc_indegree_norm")
            assert same_bits(g.v, want.v), "%s: fused norm differs from softmax + roc_indegree_norm" % what
            if blocks:
                # three ragged row blocks as the host calls them: rowEnd + r0, mask + r0, that block's colLeft
                gb = outp(n, c, layout)
                perf = torch.zeros(7, dtype=torch.int32, device=DEV)
                cuts = [0, n // 3 + 1, 2 * n // 3 + 5, n]
                for r0, r1 in zip(cuts, cuts[1:]):
                    cl = COL_LEFT if r0 == 0 else int(row_end[r0 - 1])
                    ok(sm_call(r1 - r0, c, z.v[r0:r1], labels[r0:r1] if labels is not None else None,
                               lidx[r0:r1] if lidx is not None else None, mask[r0:r1], gb.v[r0:r1], row_end[r0:r1],
                               cl, perf), what + " blocks")
                assert same_bits(gb.v, g.v), "%s: row blocks differ from one call" % what
                assert perf_of(perf)[1] == counts, "%s: row blocks count differently" % what


@pytest.mark.parametrize("layout", ["vec", "dense"])
@pytest.mark.parametrize("c", SM_C)
def test_softmax_xent(c, layout):
    """all four kernels x label form x fused norm x perf / NULL, at 1 row, a row count that leaves a warp's row groups
    ragged, and >= 3 grid passes on 8 SMs ending in a ragged warp"""
    n_multi = 3 * sm_pass_rows(c, FEW_CTAS) + 3
    data = sm_data(n_multi, c, seed=c)
    with few_sms():
        for n in (1, 37, n_multi):
            softmax_cases(c, layout, n, data, blocks=(n == n_multi))
    RAN.add(("softmax", c, layout))


def test_softmax_norm_wrapper_returns_metrics():
    n, c = 500, 41
    z_np, lab_np, mask_np, deg_np = sm_data(n, c, seed=5)
    deg_np[deg_np == 0] = 1
    z = K.padded(n, c, DEV, fill=torch.from_numpy(z_np).to(DEV))
    lab, mask = torch.from_numpy(lab_np).to(DEV), torch.from_numpy(mask_np).to(DEV)
    row_end = torch.from_numpy(np.cumsum(deg_np)).to(DEV)
    g, perf = K.softmax_xent_bwd_norm(z, lab, mask, row_end, 0, compact=True, with_perf=True)
    assert torch.equal(K.softmax_xent_bwd_norm(z, lab, mask, row_end, 0, compact=True), g)
    ref = sm_ref(z, lab, mask)
    sm_check_metrics(perf["trainLoss"], [perf[k] for k in ("trainAll", "testAll", "valAll", "trainCorrect",
                                                            "testCorrect", "valCorrect")], ref, c, "wrapper")


# --------------------------------------------------------------------------------------------- dropout ---
DROP_H = (1, 3, 7, 8, 9, 31, 33, 41, 64, 602)
DROP_RATES = (0.0, 0.1, 0.5, 0.9, 0.999995)     # the last rounds to T16 = 65536: clamped to 65535
DROP_FIRST = (0, 12345, 2 ** 32 - 3)            # the last crosses into the counter's high word
SEED, STEP = (0x5EED << 32) | 0x1234, 7


def unpack_mask(m, h):
    m = m.cpu().numpy().view(np.uint32)
    return ((m[:, :, None] >> np.arange(32, dtype=np.uint32)[None, None, :]) & 1).reshape(m.shape[0], -1), m


def dropout_cases(h, n, x_np, rate, first, layouts):
    keep = oracle.dropout_mask(first, n, h, rate, SEED, STEP)
    want = torch.from_numpy(oracle.dropout_apply(x_np[:n], keep, rate)).to(DEV)
    for layout in layouts:
        x = inp(x_np[:n], layout)
        vec = 4 if layout == "vec" else 1
        for fn in (LIB.roc_dropout_fwd, LIB.roc_dropout_bwd):
            what = "dropout H=%d %s n=%d rate=%g first=%d %s" % (h, layout, n, rate, first, fn.__name__)
            ys = []
            for _ in range(2):
                y = outp(n, h, layout)
                ok(fn(n, h, first, rate, SEED, STEP, x.v.data_ptr(), x.ld, y.v.data_ptr(), y.ld, None), what)
                y.assert_outside_unchanged(what=what)
                ys.append(y)
            assert same_bits(ys[0].v, ys[1].v), "%s: two runs differ" % what
            assert same_bits(ys[0].v, want), "%s: differs from the oracle" % what
        SEEN.add(("dropout", vec))
    m = K.dropout_mask(n, h, first, rate, SEED, STEP, DEV)
    assert torch.equal(m, K.dropout_mask(n, h, first, rate, SEED, STEP, DEV))
    b, words = unpack_mask(m, h)
    assert np.array_equal(b[:, :h], keep), "dropout mask H=%d n=%d rate=%g first=%d: keep bits differ" % (
        h, n, rate, first)
    assert not b[:, h:].any(), "dropout mask H=%d: bits or words past H are not zero" % h


@pytest.mark.parametrize("h", DROP_H)
def test_dropout(h):
    """forward, backward and the packed mask on both paths, at 37 rows and at >= 3 grid passes on 8 SMs (two items
    per thread and pass: the second unrolled item and the tail past the last item both run)"""
    n_multi = 3 * FEW_CTAS * 256 * 2 // ((h + 7) // 8) + 5
    x_np = np.random.RandomState(h).randn(n_multi, h).astype(np.float32)
    with few_sms():
        for rate in DROP_RATES:
            for first in DROP_FIRST:
                for n in (37, n_multi):
                    dropout_cases(h, n, x_np, rate, first, ("vec", "odd"))
    RAN.add(("dropout", h))


# ------------------------------------------------------------------------------------------ in-degree norm ---
NORM_H = (1, 3, 4, 41, 64)


def norm_degrees(n, rs):
    deg = rs.randint(1, 41, size=n).astype(np.int64)
    deg[0::11] = 0                     # row 0 too: its start is colLeft
    deg[1::11] = 1
    deg[2::11] = 2
    deg[3::11] = 3
    deg[4::101] = 2 ** 20 + 1
    deg[5::211] = 70000
    return deg


def specials(a, rs, frac=0.02):
    """a with NaN, +-0 and +-inf sprinkled in"""
    a = a.copy()
    for v in (np.nan, 0.0, -0.0, np.inf, -np.inf):
        a[rs.rand(*a.shape) < frac] = v
    return a


def norm_cases(h, layout, n, rs):
    vec = layout == "vec"
    deg = norm_degrees(n, rs)
    row_end = torch.from_numpy(COL_LEFT + np.cumsum(deg)).to(DEV)
    d32 = np.sqrt(deg.astype(np.float32))
    x_np = specials(rs.randn(n, h).astype(np.float32), rs)
    y_np = specials(rs.randn(n, h).astype(np.float32), rs)
    y = inp(y_np, layout)
    wcols = r4(h) if vec else h
    for relu in (False, True):
        for inplace in (False, True):
            what = "norm H=%d %s n=%d relu=%d inplace=%d" % (h, layout, n, relu, inplace)
            outs = []
            for _ in range(2):
                x = inp(x_np, layout)
                out = x if inplace else outp(n, h, layout)
                ok(LIB.roc_indegree_norm(0, n - 1, COL_LEFT, h, row_end.data_ptr(), x.v.data_ptr(), x.ld,
                                         out.v.data_ptr(), out.ld, y.v.data_ptr() if relu else None, None), what)
                out.assert_outside_unchanged(cols=wcols, what=what)
                if not inplace:
                    x.assert_outside_unchanged(cols=0, what=what + " (input)")
                outs.append((x, out))
            (x, out), (_, out2) = outs
            assert same_bits(out.wide(wcols), out2.wide(wcols)), "%s: two runs differ" % what
            # numpy fp32 over the written columns: the window, and on the float4 path the pad columns up to r4(h)
            xw = x.wide(wcols, x.init).cpu().numpy()
            yw = y.wide(wcols, y.init).cpu().numpy()
            with np.errstate(all="ignore"):
                num = np.where(yw > 0, xw, np.float32(0)) if relu else xw
                want = torch.from_numpy((num / d32[:, None]).astype(np.float32)).to(DEV)
            assert nan_equal(out.wide(wcols), want), "%s: differs from x / sqrt(float32(deg))" % what
    SEEN.add(("norm", 4 if vec else 1))


@pytest.mark.parametrize("layout", ["vec", "odd"])
@pytest.mark.parametrize("h", NORM_H)
def test_indegree_norm(h, layout):
    """k_norm<4> / <1>, with and without the relu mask, out of place and in place, degrees 0 .. 2^20 + 1 under a
    colLeft past 2^32, at >= 3 grid passes on 8 SMs"""
    wq = (h + 3) // 4 if layout == "vec" else h
    with few_sms():
        norm_cases(h, layout, max(64, 3 * FEW_CTAS * 256 // wq + 7), np.random.RandomState(h))
    RAN.add(("norm", h, layout))


# ------------------------------------------------------------------------------------------------ maps ---
MAP_SHAPES = ((4, "vec"), (64, "vec"), (1, "vec"), (41, "vec"), (64, "odd"), (5, "odd"))
RELU, SIGM = _lib.AC_MODE_RELU, _lib.AC_MODE_SIGMOID


def map_vec(h, layout):
    """vec_ok: H, every ld (and base, always aligned here) allow float4"""
    return 4 if h % 4 == 0 and layout == "vec" else 1


def twice(make, call, what, cols=None):
    """run `call(out)` on two fresh outputs from `make()`; both must agree and stay in their windows"""
    outs = []
    for _ in range(2):
        o = make()
        ok(call(o), what)
        o.assert_outside_unchanged(cols=cols, what=what)
        outs.append(o)
    assert same_bits(outs[0].v, outs[1].v), "%s: two runs differ" % what
    return outs[0]


def map_cases(h, layout, n, rs):
    vec = map_vec(h, layout)
    z = torch.zeros((), device=DEV)
    x_np = specials(rs.randn(n, h).astype(np.float32) * 40, rs)
    a_np = specials(rs.randn(n, h).astype(np.float32), rs)
    old_np = rs.randn(n, h).astype(np.float32)
    x, a, old = inp(x_np, layout), inp(a_np, layout), inp(old_np, layout)
    tag = "H=%d %s n=%d" % (h, layout, n)
    # relu forward: NaN stays NaN (relu_nanprop; compiled to a NaN-propagating max, which returns the canonical NaN
    # rather than the input's payload), -0 -> +0
    y = twice(lambda: outp(n, h, layout), lambda o: LIB.roc_activation_fwd(n, h, RELU, x.v.data_ptr(), x.ld,
                                                                               o.v.data_ptr(), o.ld, None), "relu " + tag)
    assert nan_equal(y.v, torch.where(x.v > 0, x.v, torch.where(torch.isnan(x.v), x.v, z))), "relu " + tag
    SEEN.add(("map", "relu_f", vec, False))
    # sigmoid forward against fp64
    s = twice(lambda: outp(n, h, layout), lambda o: LIB.roc_activation_fwd(n, h, SIGM, x.v.data_ptr(), x.ld,
                                                                               o.v.data_ptr(), o.ld, None), "sigm " + tag)
    s64 = 1.0 / (1.0 + torch.exp(-x.v.double()))
    nan = torch.isnan(s64)
    assert bool((torch.isnan(s.v) == nan).all()), "sigmoid NaN " + tag
    r = float(((s.v.double() - s64).abs() / ((6 * U + REF) * s64.abs() + 2.0 ** -126))[~nan].max())
    assert worst("sigmoid", r) <= 1.0, "sigmoid %s: worst |error| / bound %.3g" % (tag, r)
    SEEN.add(("map", "sigm_f", vec, False))
    # backward from the output: relu exact, sigmoid against fp64, each accumulating or not
    ys = inp(torch.sigmoid(torch.from_numpy(rs.randn(n, h).astype(np.float32) * 4)), layout)
    for acc in (False, True):
        mk = (lambda: outp(n, h, layout, init=old.v)) if acc else (lambda: outp(n, h, layout))
        g = twice(mk, lambda o: LIB.roc_activation_bwd(n, h, RELU, x.v.data_ptr(), x.ld, a.v.data_ptr(), a.ld,
                                                       o.v.data_ptr(), o.ld, int(acc), None), "relu bwd " + tag)
        want = torch.where(x.v > 0, a.v, z)
        assert same_bits(g.v, old.v + want if acc else want), "relu backward %s acc=%d" % (tag, acc)
        SEEN.add(("map", "relu_b", vec, acc))
        g = twice(mk, lambda o: LIB.roc_activation_bwd(n, h, SIGM, ys.v.data_ptr(), ys.ld, old.v.data_ptr(), old.ld,
                                                       o.v.data_ptr(), o.ld, int(acc), None), "sigm bwd " + tag)
        y64 = ys.v.double()
        res = old.v.double() * y64 * (1.0 - y64)
        want = res + old.v.double() if acc else res
        bnd = 3 * U * res.abs() + (U + REF) * want.abs() + 2.0 ** -149
        r = float(((g.v.double() - want).abs() / bnd).max())
        assert worst("sigmoid backward", r) <= 1.0, "sigmoid backward %s acc=%d: %.3g" % (tag, acc, r)
        SEEN.add(("map", "sigm_b", vec, acc))
    # add, out of place and in place (y == a, as the host issues it), and copy
    y = twice(lambda: outp(n, h, layout), lambda o: LIB.roc_add_fwd(n, h, x.v.data_ptr(), x.ld, a.v.data_ptr(), a.ld,
                                                                        o.v.data_ptr(), o.ld, None), "add " + tag)
    assert same_bits(y.v, x.v + a.v), "add " + tag
    y2 = twice(lambda: inp(x_np, layout), lambda o: LIB.roc_add_fwd(n, h, o.v.data_ptr(), o.ld, a.v.data_ptr(), a.ld,
                                                                        o.v.data_ptr(), o.ld, None), "add in place " + tag)
    assert same_bits(y2.v, y.v), "add in place " + tag
    SEEN.add(("map", "add_f", vec, False))
    y = twice(lambda: outp(n, h, layout), lambda o: LIB.roc_copy2d(n, h, x.v.data_ptr(), x.ld, o.v.data_ptr(), o.ld,
                                                                       None), "copy " + tag)
    assert same_bits(y.v, x.v), "copy " + tag
    SEEN.add(("map", "copy", vec, False))


@pytest.mark.parametrize("h,layout", MAP_SHAPES)
def test_maps(h, layout):
    """k_map's six ops on the path the shape selects, at >= 3 grid passes on 8 SMs"""
    wq = h // 4 if map_vec(h, layout) == 4 else h
    with few_sms():
        map_cases(h, layout, 3 * FEW_CTAS * 256 // wq + 13, np.random.RandomState(100 + h))
    RAN.add(("map", h, layout))


def add_bwd_cases(h, layout, n, rs):
    dy = inp(specials(rs.randn(n, h).astype(np.float32), rs), layout)
    old_a, old_b = inp(rs.randn(n, h).astype(np.float32), layout), inp(rs.randn(n, h).astype(np.float32), layout)
    combos = [(True, True, aa, ab) for aa in (0, 1) for ab in (0, 1)] + [(False, True, 0, 0), (False, True, 0, 1),
                                                                        (True, False, 0, 0), (True, False, 1, 0),
                                                                        (False, False, 1, 1)]
    for has_a, has_b, acc_a, acc_b in combos:
        what = "add_bwd H=%d %s n=%d dA=%d dB=%d acc=%d%d" % (h, layout, n, has_a, has_b, acc_a, acc_b)
        runs = []
        for _ in range(2):
            da, db = outp(n, h, layout, init=old_a.v), outp(n, h, layout, init=old_b.v)
            ok(LIB.roc_add_bwd(n, h, dy.v.data_ptr(), dy.ld, da.v.data_ptr() if has_a else None, da.ld, acc_a,
                               db.v.data_ptr() if has_b else None, db.ld, acc_b, None), what)
            for t, has, old, acc in ((da, has_a, old_a, acc_a), (db, has_b, old_b, acc_b)):
                t.assert_outside_unchanged(what=what)
                want = (old.v + dy.v if acc else dy.v) if has else old.v
                assert same_bits(t.v, want), what
            runs.append((da, db))
        assert same_bits(runs[0][0].v, runs[1][0].v) and same_bits(runs[0][1].v, runs[1][1].v), what


@pytest.mark.parametrize("layout", ["vec", "odd"])
def test_add_bwd_and_fill(layout):
    """roc_add_bwd with either gradient absent and every accumulate flag; roc_fill writes only its window"""
    with few_sms():
        for h in (1, 41, 64):
            n = 3 * FEW_CTAS * 256 // h + 13
            add_bwd_cases(h, layout, n, np.random.RandomState(h))
            twice(lambda: outp(n, h, layout), lambda o: LIB.roc_fill(n, h, -2.75, o.v.data_ptr(), o.ld, None),
                  "fill H=%d %s" % (h, layout))
            f = outp(n, h, layout)
            ok(LIB.roc_fill(n, h, -2.75, f.v.data_ptr(), f.ld, None), "fill")
            assert bool((f.v == -2.75).all()), "fill H=%d %s" % (h, layout)


# --------------------------------------------------------------------------------------------- scale, Adam ---
def scale_case(count, rs):
    w_np = rs.rand(count).astype(np.float32)
    w_np[::17] = 0.0
    a, b = np.float32(-0.0734), np.float32(0.0734)
    outs = []
    for _ in range(2):
        w, buf = guarded(w_np, SENT)
        ok(LIB.roc_scale(count, float(a), float(b), w.data_ptr(), None), "roc_scale")
        assert bool((buf[:4] == SENT).all() and (buf[-4:] == SENT).all()), "roc_scale wrote outside its range"
        outs.append(w)
    assert same_bits(outs[0], outs[1]), "roc_scale: two runs differ"
    w64 = torch.from_numpy(w_np).to(DEV).double()
    want = (float(b) - float(a)) * w64 + float(a)
    bnd = 2 * U * ((float(b) - float(a)) * w64).abs() + (U + REF) * want.abs() + 2.0 ** -149
    r = float(((outs[0].double() - want).abs() / bnd).max())
    assert worst("scale", r) <= 1.0, "roc_scale: worst |error| / bound %.3g" % r


def adam_case(count, wd, rs):
    alpha, b1, b2, eps = np.float32(0.003), np.float32(0.9), np.float32(0.999), np.float32(1e-8)
    w_np, g_np = rs.randn(count).astype(np.float32), rs.randn(count).astype(np.float32)
    m_np = (rs.randn(count) * 0.1).astype(np.float32)
    v_np = np.abs(rs.randn(count) * 0.1).astype(np.float32)
    zero = np.arange(count) % 13 == 0                 # v = 0 and g + wd w = 0: sqrt(vt) = 0, the eps path
    w_np[zero], g_np[zero], v_np[zero] = 0.0, 0.0, 0.0
    g = torch.from_numpy(g_np).to(DEV)
    outs = []
    for _ in range(2):
        (w, wb), (m, mb), (v, vb) = guarded(w_np, SENT), guarded(m_np, SENT), guarded(v_np, SENT)
        ok(LIB.roc_adam_update(count, float(alpha), float(b1), float(b2), float(wd), float(eps), g.data_ptr(),
                               m.data_ptr(), v.data_ptr(), w.data_ptr(), None), "roc_adam_update")
        for bb in (wb, mb, vb):
            assert bool((bb[:4] == SENT).all() and (bb[-4:] == SENT).all()), "roc_adam_update wrote outside its range"
        outs.append((w, m, v))
    for a_, b_ in zip(*outs):
        assert same_bits(a_, b_), "roc_adam_update: two runs differ"
    # fp64 from the fp32 inputs; 1 - beta is exact in fp32 (Sterbenz).  Each fp32 operation rounds once: u |result|
    d = lambda t: torch.from_numpy(t).to(DEV).double()
    W, G, M, V = d(w_np), d(g_np), d(m_np), d(v_np)
    a, b1, b2, wd, eps = float(alpha), float(b1), float(b2), float(np.float32(wd)), float(eps)
    c1, c2 = 1.0 - b1, 1.0 - b2
    gt = G + wd * W
    e_g = U * ((wd * W).abs() + gt.abs())
    mt = b1 * M + c1 * gt
    e_m = U * ((b1 * M).abs() + (c1 * gt).abs() + mt.abs()) + c1 * e_g
    vt = b2 * V + c2 * gt * gt
    e_v = U * ((b2 * V).abs() + 2 * c2 * gt * gt + vt.abs()) + 2 * c2 * gt.abs() * e_g
    s = vt.sqrt()
    e_s = torch.where(vt > 0, e_v / (2 * s.clamp_min(1e-300)), torch.zeros_like(s)) + U * s
    den = s + eps
    e_den = e_s + U * den
    q = a * mt / den
    e_q = (a * e_m + U * (a * mt).abs() + q.abs() * e_den) / den + U * q.abs()
    wn = W - q
    e_w = e_q + U * wn.abs()
    w, m, v = outs[0]
    for name, got, want, e in (("w", w, wn, e_w), ("m", m, mt, e_m), ("v", v, vt, e_v)):
        r = float(((got.double() - want).abs() / (e + REF * want.abs() + 2.0 ** -149)).max())
        assert worst("Adam", r) <= 1.0, "roc_adam_update %s (wd=%g): worst |error| / bound %.3g" % (name, wd, r)


def test_scale_and_adam():
    """roc_scale and roc_adam_update against fp64 at >= 3 grid passes on 8 SMs, Adam with and without weight decay"""
    count = 3 * FEW_CTAS * 256 + 77
    rs = np.random.RandomState(9)
    with few_sms():
        scale_case(count, rs)
        for wd in (0.0, 0.05):
            adam_case(count, wd, rs)


# ------------------------------------------------------------------------------------------- row copies ---
ROW_H = (5, 16, 41, 64, 65, 200)
NSRC = 2000


def copy_vec(layout):
    return 4 if layout == "vec" else 1


def pack_cases(h, layout, n, rs):
    vec = copy_vec(layout)
    wcols = r4(h) if vec == 4 else h
    src = inp(rs.randn(NSRC, h).astype(np.float32), layout)
    rows = torch.from_numpy(rs.randint(0, NSRC, size=n).astype(np.int32)).to(DEV)      # with duplicates
    what = "pack_rows H=%d %s n=%d" % (h, layout, n)
    dst = twice(lambda: outp(n, h, layout), lambda o: LIB.roc_pack_rows(n, h, rows.data_ptr(), src.v.data_ptr(),
                                                                            src.ld, o.v.data_ptr(), o.ld, None),
                what, cols=wcols)
    assert same_bits(dst.wide(wcols), src.wide(wcols)[rows.long()]), what
    SEEN.add(("pack", vec))
    # a subset of a send list, written to its places
    nsel = n * 2 // 3
    sel = torch.from_numpy(rs.permutation(n)[:nsel].astype(np.int32)).to(DEV)
    what = "pack_rows_at H=%d %s n=%d" % (h, layout, n)
    dst = twice(lambda: outp(n, h, layout), lambda o: LIB.roc_pack_rows_at(nsel, h, sel.data_ptr(), rows.data_ptr(),
                                                                               src.v.data_ptr(), src.ld,
                                                                               o.v.data_ptr(), o.ld, None),
                what, cols=wcols)
    want = dst.init.clone()
    dst.wide(wcols, want)[sel.long()] = src.wide(wcols)[rows.long()[sel.long()]]
    assert same_bits(dst.base, want), what
    SEEN.add(("pack_at", vec))


@pytest.mark.parametrize("layout", ["vec", "odd"])
@pytest.mark.parametrize("h", ROW_H)
def test_pack_rows(h, layout):
    """roc_pack_rows and roc_pack_rows_at at >= 3 grid passes on 8 SMs"""
    wq = (h + 3) // 4 if layout == "vec" else h
    with few_sms():
        pack_cases(h, layout, 3 * FEW_CTAS * 256 // wq + 11, np.random.RandomState(h))
    RAN.add(("pack", h, layout))


def push_lr(wq):
    return 16 if wq <= 16 else 32


def push_case(h, path, peers, sm_limit, n, rs):
    """roc_push_rows into `peers` local slabs: entry j stores src row srcRows[j] to row dstRow[j] of slab peer[j];
    the destinations are a random injection into the slabs.  The scalar path is forced by one slab base 4 bytes off
    16-byte alignment."""
    vec = 4 if path == "vec" else 1
    wcols = r4(h) if vec == 4 else h
    src = inp(rs.randn(NSRC, h).astype(np.float32), "vec")
    slab_rows = n // peers + 50
    slot = rs.permutation(peers * slab_rows)[:n]
    peer_np, dst_np = (slot // slab_rows).astype(np.uint8), (slot % slab_rows).astype(np.int32)
    src_rows = torch.from_numpy(rs.randint(0, NSRC, size=n).astype(np.int32)).to(DEV)
    peer, dst_row = torch.from_numpy(peer_np).to(DEV), torch.from_numpy(dst_np).to(DEV)
    ld = r4(h) + 8
    what = "push_rows H=%d %s peers=%d smLimit=%d n=%d" % (h, path, peers, sm_limit, n)
    runs = []
    for _ in range(2):
        slabs = [Frame(slab_rows, h, SENT, ld, col0=(1 if (vec == 1 and p == peers - 1) else 0))
                 for p in range(peers)]
        bases = (C.c_void_p * peers)(*[s.v.data_ptr() for s in slabs])
        ok(LIB.roc_push_rows(n, h, src_rows.data_ptr(), peer.data_ptr(), dst_row.data_ptr(), src.v.data_ptr(), src.ld,
                             C.cast(bases, C.c_void_p), peers, ld, sm_limit, None), what)
        runs.append(slabs)
    for p, (s, s2) in enumerate(zip(*runs)):
        assert same_bits(s.base, s2.base), "%s: two runs differ" % what
        sel = torch.from_numpy(np.nonzero(peer_np == p)[0]).to(DEV)
        want = s.init.clone()
        s.wide(wcols, want)[dst_row.long()[sel]] = src.wide(wcols)[src_rows.long()[sel]]
        assert same_bits(s.base, want), "%s: slab %d differs from torch indexing" % (what, p)
    SEEN.add(("push", vec, push_lr((h + 3) // 4 if vec == 4 else h)))


@pytest.mark.parametrize("peers", [1, 2, 16])
@pytest.mark.parametrize("path", ["vec", "scalar"])
@pytest.mark.parametrize("h", ROW_H)
def test_push_rows(h, path, peers):
    """both paths and both LR at 1, 2 and ROC_MAX_PEERS local slabs; smLimit = 1 runs 8 CTAs through many turns of
    the U = 8 loop and a ragged tail, smLimit = 0 sizes the grid for the whole chip"""
    rs = np.random.RandomState(h * 100 + peers)
    for sm_limit in (1, 0):
        push_case(h, path, peers, sm_limit, 3001, rs)
    RAN.add(("push", h, path, peers))


# ---------------------------------------------------------------------------------- the whole chip ---
def test_full_chip_passes():
    """One case per kernel with no SM reserve, at >= 3 full grid passes plus a ragged tail on this device"""
    ctas = nsm() * 16
    threads = ctas * 256
    for c in (32, 64, 128, 602):
        n = 3 * sm_pass_rows(c, ctas) + 5 * (256 // (sm_inst(c) or 32)) + 3
        data = sm_data(n, c, seed=1000 + c)
        z = inp(data[0], "vec")
        lab, mask = torch.from_numpy(data[1]).to(DEV), torch.from_numpy(data[2]).to(DEV)
        deg = np.maximum(data[3], 1)
        row_end = torch.from_numpy(COL_LEFT + np.cumsum(deg)).to(DEV)
        div = torch.from_numpy(np.sqrt(deg.astype(np.float32)).astype(np.float64)).to(DEV)
        g = outp(n, c, "vec")
        perf = torch.zeros(7, dtype=torch.int32, device=DEV)
        ok(sm_call(n, c, z.v, None, lab, mask, g.v, row_end, COL_LEFT, perf), "softmax C=%d" % c)
        g.assert_outside_unchanged(what="softmax full chip")
        ref = sm_ref(z.v, lab, mask)
        sm_check(g.v, ref, div, c, "softmax full chip C=%d" % c)
        loss, counts = perf_of(perf)
        sm_check_metrics(loss, counts, ref, c, "softmax full chip C=%d" % c)
        del ref, g, z
    h = 64
    n = 3 * threads * 2 // ((h + 7) // 8) + 77
    x_np = np.random.RandomState(3).randn(n, h).astype(np.float32)
    dropout_cases(h, n, x_np, 0.5, 2 ** 32 - 3, ("vec", "odd"))
    rs = np.random.RandomState(4)
    for layout in ("vec", "odd"):
        norm_cases(41, layout, 3 * threads // (11 if layout == "vec" else 41) + 7, rs)
        pack_cases(41, layout, 3 * threads // (11 if layout == "vec" else 41) + 11, rs)
    for h, layout in ((64, "vec"), (41, "vec")):
        map_cases(h, layout, 3 * threads // (h // 4 if h % 4 == 0 else h) + 13, rs)
    add_bwd_cases(41, "vec", 3 * threads // 41 + 13, rs)
    scale_case(3 * threads + 77, rs)
    adam_case(3 * threads + 77, 0.05, rs)
    push_case(64, "vec", 2, 0, 3 * nsm() * 8 * 16 * 8 + 99, rs)


def test_dispatch_table_covered():
    """Every launch variant the dispatch rules can produce was reached: each softmax instantiation x label form x norm,
    both paths of every k_map op (and accumulate), both paths of k_dropout, k_norm and the packs, and both LR x both
    paths of k_push_rows.  Prints the worst error-to-bound ratio per family."""
    wanted_runs = ({("softmax", c, lay) for c in SM_C for lay in ("vec", "dense")} | {("dropout", h) for h in DROP_H} |
                   {("norm", h, lay) for h in NORM_H for lay in ("vec", "odd")} |
                   {("map", h, lay) for h, lay in MAP_SHAPES} | {("pack", h, lay) for h in ROW_H for lay in ("vec", "odd")} |
                   {("push", h, p, q) for h in ROW_H for p in ("vec", "scalar") for q in (1, 2, 16)})
    if not wanted_runs <= RAN:
        pytest.skip("%d of the %d matrix cases did not run in this process" % (len(wanted_runs - RAN), len(wanted_runs)))
    for k in sorted(WORST):
        print("worst |error| / bound  %-18s %.4f" % (k, WORST[k]))
    wanted = {("softmax", lr, f, nm) for lr in (8, 16, 32, 0) for f in ("onehot", "index") for nm in (False, True)}
    wanted |= {("map", op, v, False) for op in ("relu_f", "sigm_f", "add_f", "copy") for v in (4, 1)}
    wanted |= {("map", op, v, acc) for op in ("relu_b", "sigm_b") for v in (4, 1) for acc in (False, True)}
    wanted |= {(k, v) for k in ("dropout", "norm", "pack", "pack_at") for v in (4, 1)}
    wanted |= {("push", v, lr) for v in (4, 1) for lr in (16, 32)}
    missing = wanted - SEEN
    assert not missing, "never launched: %s" % sorted(missing, key=str)
    assert SEEN <= wanted, "outside the table: %s" % sorted(SEEN - wanted, key=str)
