"""The kernels added after the elementwise matrix (test_elementwise_matrix_gpu.py) held to its bar: every launch variant
against an fp64 or exact reference, mostly under roc_set_sm_reserve leaving 8 SMs so that the grid-stride loops run
many passes and end in a ragged tail, inputs in NaN-padded buffers, outputs in sentinel-filled ones, every call twice.

Dispatch, restated from the launchers and checked for coverage by test_late_dispatch_table_covered at the end:
  k_scaled_add<VEC>        VEC = 4 when H, the three ld and the three bases allow float4 (vec_ok), else 1.
  k_scaled_add_bwd<VEC>    VEC = 4 under the same rule over dY and the non-NULL dA / dB.
  k_relu_fwd_y_bf16        one scalar kernel; roc_activation_fwd_y_bf16 with ROC_AC_MODE_RELU.
  k_relu_bwd_y_bf16<ACC>   ACC = the accumulate flag.
  k_f32_to_bf16            grid-strides over rows * ldDst: whole destination rows, columns [H, ldDst) get zero.
  k_bf16_to_f32            grid-strides over rows * H.
  k_dropout<1, 2, u16>     roc_dropout_fwd_bf16, whatever the layout.
  k_map<ELU_F / ELU_B, VEC, ACC>   as every k_map: VEC = 4 when vec_ok; ACC = accumulate (backward only).
  k_sigmoid_xent<VEC, L>   VEC = 4 when ldZ, ldG and both bases allow float4, else 1; with Q = ceil(C / VEC), L is the
                           smallest of 1, 2, 4, 8, 16, 32 that is >= Q (32 above); the grid is ew_grid(rows * L) capped
                           at ML_MAX_BLOCKS; the block that takes the last ticket adds the per-block partials.
  batch norm               TX = min(ceil(H / 4), 64) column groups by TY = 256 / TX row lanes; colBlocks =
                           ceil(ceil(H / 4) / TX) on blockIdx.y.  k_bn_reduce<BWD, RELU> over rowBlocks =
                           ceil(rows / (128 TY)) fixed row blocks; k_bn_normalise<RELU> and k_bn_backward_apply<RELU,
                           ACC> grid-stride over rows with min(ceil(rows / (4 TY)), 8 * sm_count()) CTAs.
  attention scores         forward k_attn_scores_fwd<float, VEC>, VEC = X 16-byte rows; tiles of TR rows (fwd_shape)
                           on min(tiles, sm_count() * perSm) CTAs.  Backward k_attn_scores_bwd<float, VEC> on
                           rowBlocks x colBlocks CTAs (batch norm's layout), a function of (rows, H) alone.

Windows.  Nothing outside [rows][H] of an output is written (guard rows above and below, pad columns), except
k_f32_to_bf16, which writes whole rows of ldDst with zero past H, and the sigmoid metrics (18 values between guards).
Every call runs twice and must give the same bits.

References (u = 2^-24):
  scaled_add     forward within half an ulp of the fp64 value of fmaf(alpha, a, float32(beta b)) (teleport's test);
                 backward bit-exact against fp32 torch without accumulation, within half an ulp of fp64 with it.
  bf16 relu      bit-exact: numpy's round to nearest even of the fp32 relu (NaN -> 0x7FC0); the backward bit-exact
                 against torch fp32 on the widened y, whose mask differs from x > 0 only for 0 < x <= 2^-134.
  conversions    bit-exact, both ways.
  bf16 dropout   bit-exact against oracle.dropout_mask / dropout_apply on the widened rows.
  ELU            |y - y64| <= 2u |y64| + 2^-149 (expm1f: 1 ulp); the backward from the kernel's own fp32 y,
                 |dx - dx64| <= 2u |r| (+ u |dx64| accumulating), r = dy (y > 0 ? 1 : y + 1): one rounded add, one
                 rounded product.
  sigmoid        s = sigmoid(z) from expf (2 ulp <= 4u relative), 1 + e and its rounded reciprocal: 4u s for z >= 0,
                 9u s for z < 0 (one more product, e's own error).  g = s - y is exact for y = 0 and for s >= 1/2
                 (Sterbenz) and rounds once otherwise, so |g - g64| <= (4 or 9) u s64 + u |g64|; the fused norm divides
                 by sqrtf(deg) (taken into the reference) and rounds once more: u |g / d|.  A floor of 4 * 2^-149 covers
                 expf's 2 ulp where e is subnormal (z < -87.3).  The counts are exact.  The loss of an element is
                 relu(+-z) + log1pf(e): log1pf's 1 ulp (2u) and e's 4u carried through log1p (<= 4u log1p(e)), one add;
                 a float4 chunk adds up to 4 of them in fp32 (3u), fp64 after that, so each split's loss is within
                 (10u or 7u + n 2^-53) of the fp64 sum, relative (all terms are >= 0).
  batch norm     test_batchnorm_gpu.py's fp64 bounds (K_Y, K_DX, K_RED); the running statistics within 2u.
  attention      test_gat_heads_gpu.py's fp64 bounds: S gamma_F sum |a x|, dX 3u, dA 2u.
Each bound also carries 2^-50 |reference| for the fp64 reference's own roundings.

SM budgets.  Batch norm, attention scores, scaled_add, the bf16 relu, the conversions and the sigmoid gradient give
the same bits on the whole chip, on an odd SM count and on 8 SMs.  The sigmoid counts are equal too.  The sigmoid
loss is not bit-invariant: each thread sums the rows it visits, and which rows those are depends on gridDim, so only
its fp64 bound is asserted there (include/roc_b200.h says so).

Worst |error| / bound, measured on one H100 80GB HBM3 (700 W): scaled_add 1.00 and its backward 1.00 (a result
exactly half an ulp from a tie), ELU 0.88, ELU backward 0.999, sigmoid gradient 0.71, sigmoid loss 0.003, batch norm
y 0.64, dx 0.60, dgamma / dbeta 0.23, running statistics 0.50, attention S 0.999, dX 0.65, dA 0.064.  The file runs in
about 35 s."""
import contextlib
import math

import numpy as np
import pytest
import torch

import test_elementwise_matrix_gpu as M
from multilabel_oracle import sigmoid_xent as ml_oracle
from oracle import oracle
from roc_b200 import _lib
from roc_b200.model import pack_multilabels
from test_batchnorm_cpu import bn_backward, bn_forward
from test_batchnorm_gpu import K_DX, K_RED, K_Y
from test_batchnorm_gpu import _inputs as bn_inputs
from test_gat_heads_cpu import elu_ref, scores_bwd_ref, scores_ref

pytestmark = pytest.mark.gpu
DEV, LIB, U, REF, SENT = M.DEV, M.LIB, M.U, M.REF, M.SENT
FEW_CTAS = M.FEW_CTAS
SENT16 = -12345                        # a bf16 sentinel (0xCFC7)
NAN16 = 0x7FC0
HALF = 0.5 + 1e-6                      # half an ulp, with room for the fp64 reference's own rounding
COL_LEFT = M.COL_LEFT
inp, outp, twice, ok, ld_of, same_bits, nan_equal, guarded = (M.inp, M.outp, M.twice, M.ok, M.ld_of, M.same_bits,
                                                              M.nan_equal, M.guarded)

# This file's own bookkeeping, kept apart from the matrix's: its coverage test asserts that SEEN holds nothing
# outside its own table.
SEEN = set()        # launch variants reached, by the dispatch rules above
RAN = set()         # matrix cases that ran in this process
WORST = {}          # family -> worst |error| / bound


def worst(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    return ratio


@contextlib.contextmanager
def sms(n):
    """sm_count() = n for this thread's launches"""
    prev = LIB.roc_set_sm_reserve(M.nsm() - n)
    try:
        yield
    finally:
        LIB.roc_set_sm_reserve(prev)


def budgets():
    """the whole chip, an odd SM count, 8 SMs"""
    return (M.nsm(), (M.nsm() // 2) | 1, M.FEW_SMS)


def guard_ok(buf, what):
    assert bool((buf[:4] == SENT).all() and (buf[-4:] == SENT).all()), "%s wrote outside its range" % what


# ----------------------------------------------------------------------------------------------- bf16 frames ---
class BFrame:
    """M.Frame over bf16 bits (int16): a [rows][h] window at row 1 of a [rows + 2][ld] buffer filled with `fill`"""

    def __init__(self, rows, h, fill, ld, init=None):
        self.base = torch.full((rows + 2, ld), fill, device=DEV, dtype=torch.int16)
        self.rows, self.h = rows, h
        self.v = self.base[1:rows + 1, :h]
        if init is not None:
            self.v.copy_(init)
        self.init = self.base.clone()

    @property
    def ld(self):
        return self.base.stride(0)

    def assert_outside_unchanged(self, cols=None, what=""):
        changed = self.base != self.init
        changed[1:self.rows + 1, :(self.h if cols is None else cols)] = False
        if bool(changed.any()):
            r, c = (int(i) for i in torch.nonzero(changed)[0])
            raise AssertionError("%s: wrote outside its window, buffer row %d column %d" % (what, r, c))


def twice16(make, call, what, cols=None):
    """M.twice for bf16 frames"""
    outs = []
    for _ in range(2):
        o = make()
        ok(call(o), what)
        o.assert_outside_unchanged(cols=cols, what=what)
        outs.append(o)
    assert torch.equal(outs[0].base, outs[1].base), "%s: two runs differ" % what
    return outs[0]


def rne(x):
    """numpy fp32 -> bf16 bits (uint16), round to nearest even; NaN -> 0x7FC0"""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), np.uint16(NAN16), r)


def widen(t16):
    """bf16 bits (int16 tensor) -> fp32, exactly"""
    return (t16.to(torch.int32) << 16).view(torch.float32)


def u16(t16):
    return t16.cpu().numpy().view(np.uint16)


# ------------------------------------------------------------------------------------------------ scaled add ---
ALPHA, BETA = float(np.float32(0.9)), float(np.float32(0.1))
SA_SHAPES = ((64, "vec"), (4, "vec"), (64, "dense"), (41, "vec"), (64, "odd"), (5, "dense"), (1, "vec"))
SA_COEFS = ((ALPHA, BETA), (-1.75, 3.0e-3), (1.0, 1.0), (0.0, 2.0), (0.0, BETA))
SA_BWD = [(True, True, aa, ab) for aa in (0, 1) for ab in (0, 1)] + [(False, True, 0, 1), (True, False, 1, 0),
                                                                     (False, True, 0, 0), (True, False, 0, 0)]


def sa_vec(h, layout):
    return 4 if h % 4 == 0 and layout != "odd" else 1


def sa_rows(h, layout, ctas):
    """>= 3 grid passes plus a ragged tail"""
    return 3 * ctas * 256 // (h // 4 if sa_vec(h, layout) == 4 else h) + 13


def spread(n, h, rs):
    """normals scaled by 2^-12 .. 2^12, with +-0"""
    a = (rs.randn(n, h) * np.exp2(rs.randint(-12, 13, size=(n, h)))).astype(np.float32)
    a[rs.rand(n, h) < 0.02] = 0.0
    a[rs.rand(n, h) < 0.02] = -0.0
    return a


def ulps(got, want):
    """|got - want| in units of the last place of want (fp32), per element (test_teleport_gpu.py's _ulps)"""
    want32 = want.astype(np.float32)
    spacing = np.spacing(np.abs(want32)).astype(np.float64)
    return np.abs(got.astype(np.float64) - want) / np.maximum(spacing, np.finfo(np.float32).tiny)


def sa_cases(h, layout, n, rs):
    vec = sa_vec(h, layout)
    a_np, b_np = spread(n, h, rs), spread(n, h, rs)
    a, b = inp(a_np, layout), inp(b_np, layout)
    outs = {}
    for alpha, beta in SA_COEFS:
        what = "scaled_add H=%d %s n=%d (%g, %g)" % (h, layout, n, alpha, beta)
        y = twice(lambda: outp(n, h, layout), lambda o: LIB.roc_scaled_add_fwd(n, h, alpha, a.v.data_ptr(), a.ld, beta,
                                                                                b.v.data_ptr(), b.ld, o.v.data_ptr(),
                                                                                o.ld, None), what)
        want = alpha * a_np.astype(np.float64) + (np.float32(beta) * b_np).astype(np.float64)
        r = float(ulps(y.v.cpu().numpy(), want).max()) / HALF
        assert worst("scaled_add", r) <= 1.0, "%s: %.3g half-ulps" % (what, r)
        if (alpha, beta) == (1.0, 1.0):
            add = outp(n, h, layout)
            ok(LIB.roc_add_fwd(n, h, a.v.data_ptr(), a.ld, b.v.data_ptr(), b.ld, add.v.data_ptr(), add.ld, None), what)
            assert same_bits(y.v, add.v), "%s: differs from roc_add_fwd" % what
        outs["fwd %g %g" % (alpha, beta)] = y.v
    SEEN.add(("scaled_add", vec))
    dy = inp(spread(n, h, rs), layout)
    old_a, old_b = inp(rs.randn(n, h).astype(np.float32), layout), inp(rs.randn(n, h).astype(np.float32), layout)
    for alpha, beta in ((ALPHA, BETA), (-3.0, 0.0)):
        for has_a, has_b, acc_a, acc_b in SA_BWD:
            what = "scaled_add_bwd H=%d %s n=%d (%g, %g) dA=%d dB=%d acc=%d%d" % (h, layout, n, alpha, beta, has_a,
                                                                                 has_b, acc_a, acc_b)
            runs = []
            for _ in range(2):
                da = outp(n, h, layout, init=old_a.v if acc_a else None)
                db = outp(n, h, layout, init=old_b.v if acc_b else None)
                ok(LIB.roc_scaled_add_bwd(n, h, dy.v.data_ptr(), dy.ld, alpha, da.v.data_ptr() if has_a else None,
                                          da.ld, acc_a, beta, db.v.data_ptr() if has_b else None, db.ld, acc_b, None),
                   what)
                for t, has in ((da, has_a), (db, has_b)):
                    t.assert_outside_unchanged(cols=h if has else 0, what=what)
                runs.append((da, db))
            assert all(same_bits(p.v, q.v) for p, q in zip(*runs)), "%s: two runs differ" % what
            for t, has, acc, coef, old in ((runs[0][0], has_a, acc_a, alpha, old_a), (runs[0][1], has_b, acc_b, beta,
                                                                                       old_b)):
                if not has:
                    continue
                if not acc:
                    want = dy.v * torch.tensor(coef, dtype=torch.float32, device=DEV)
                    assert same_bits(t.v, want), "%s: differs from fp32 coef * dY" % what
                else:
                    want = coef * dy.v.double() + old.v.double()
                    r = float(ulps(t.v.cpu().numpy(), want.cpu().numpy()).max()) / HALF
                    assert worst("scaled_add backward", r) <= 1.0, "%s: %.3g half-ulps" % (what, r)
                outs["bwd (%g, %g) %d%d%d%d %g" % (alpha, beta, has_a, has_b, acc_a, acc_b, coef)] = t.v
    SEEN.add(("scaled_add_bwd", vec))
    return outs


@pytest.mark.parametrize("h,layout", SA_SHAPES)
def test_scaled_add(h, layout):
    """k_scaled_add and k_scaled_add_bwd on the path the shape selects, five (alpha, beta) forward, every accumulate
    flag and NULL output backward, at >= 3 grid passes on 8 SMs"""
    with M.few_sms():
        sa_cases(h, layout, sa_rows(h, layout, FEW_CTAS), np.random.RandomState(h))
    RAN.add(("scaled_add", h, layout))


# ------------------------------------------------------------------------------------------- bf16 relu, casts ---
BF_SHAPES = ((1, "vec"), (5, "odd"), (41, "odd"), (64, "dense"), (64, "vec"))
RELU, ELU = _lib.AC_MODE_RELU, _lib.AC_MODE_ELU
BF_SPECIALS = (0.0, -0.0, np.nan, np.inf, -np.inf, 2.0 ** -134, 2.0 ** -133.5, -2.0 ** -134, -2.0 ** -133.5,
               2.0 ** -133, 2.0 ** -126, 3.4e38, -3.4e38)


def bf_x(n, h, rs):
    """fp32 over the whole exponent range, bf16 rounding ties (low half 0x8000) and BF_SPECIALS"""
    with np.errstate(over="ignore"):                    # past fp32's range: +-inf
        x = (rs.randn(n, h) * np.exp2(rs.randint(-150, 129, size=(n, h)))).astype(np.float32)
    ties = ((rs.randint(0, 0xFF7F, size=(n, h)).astype(np.uint32) << 16) | 0x8000).view(np.float32)
    x = np.where(rs.rand(n, h) < 0.1, ties, x)
    for v in BF_SPECIALS:
        x[rs.rand(n, h) < 0.01] = v
    return x


def bf_rows(h, ctas):
    return 3 * ctas * 256 // h + 13


def relu_bf16_cases(h, layout, n, rs):
    tag = "H=%d %s n=%d" % (h, layout, n)
    x_np = bf_x(n, h, rs)
    x = inp(x_np, layout)
    y = twice16(lambda: BFrame(n, h, SENT16, ld_of(h, layout)),
                lambda o: LIB.roc_activation_fwd_y_bf16(n, h, RELU, x.v.data_ptr(), x.ld, o.v.data_ptr(), o.ld, None),
                "relu_fwd_y_bf16 " + tag)
    with np.errstate(invalid="ignore"):
        r = np.where(x_np > 0, x_np, np.where(np.isnan(x_np), x_np, np.float32(0)))
    assert np.array_equal(u16(y.v), rne(r)), "relu_fwd_y_bf16 %s: differs from RNE of the fp32 relu" % tag
    SEEN.add(("relu_fwd_y_bf16",))
    yw = widen(y.v)
    xt = x.v
    small = (xt > 0) & (xt <= 2.0 ** -134)
    assert bool(small.any()) and torch.equal(yw > 0, (xt > 0) & ~small), "relu_fwd_y_bf16 %s: mask" % tag
    dy = inp(M.specials(rs.randn(n, h).astype(np.float32), rs), layout)
    old = inp(rs.randn(n, h).astype(np.float32), layout)
    z = torch.zeros((), device=DEV)
    outs = {"y": y.v}
    for acc in (False, True):
        what = "relu_bwd_y_bf16 %s acc=%d" % (tag, acc)
        dx = twice(lambda: outp(n, h, layout, init=old.v if acc else None),
                   lambda o: LIB.roc_activation_bwd_y_bf16(n, h, RELU, y.v.data_ptr(), y.ld, dy.v.data_ptr(), dy.ld,
                                                           o.v.data_ptr(), o.ld, int(acc), None), what)
        g = torch.where(yw > 0, dy.v, z)
        assert nan_equal(dx.v, old.v + g if acc else g), what
        SEEN.add(("relu_bwd_y_bf16", acc))
        outs["dx %d" % acc] = dx.v
    return outs


def cast_cases(h, layout, n, rs):
    tag = "H=%d %s n=%d" % (h, layout, n)
    x_np = bf_x(n, h, rs)
    x = inp(x_np, layout)
    ldd = ld_of(h, layout)
    d = twice16(lambda: BFrame(n, h, SENT16, ldd),
                lambda o: LIB.roc_f32_to_bf16(n, h, x.v.data_ptr(), x.ld, o.v.data_ptr(), o.ld, None),
                "f32_to_bf16 " + tag, cols=ldd)
    rows = u16(d.base[1:n + 1])
    assert np.array_equal(rows[:, :h], rne(x_np)), "f32_to_bf16 %s: differs from RNE" % tag
    assert not rows[:, h:].any(), "f32_to_bf16 %s: pad columns are not zero" % tag
    SEEN.add(("f32_to_bf16",))
    src_np = rs.randint(-32768, 32768, size=(n, h)).astype(np.int16)       # every bit pattern: NaN, inf, subnormals
    src = BFrame(n, h, NAN16, ldd, init=torch.from_numpy(src_np))
    w = twice(lambda: outp(n, h, layout),
              lambda o: LIB.roc_bf16_to_f32(n, h, src.v.data_ptr(), src.ld, o.v.data_ptr(), o.ld, None),
              "bf16_to_f32 " + tag)
    assert torch.equal(M.bits(w.v), M.bits(widen(src.v))), "bf16_to_f32 %s: not the exact widening" % tag
    SEEN.add(("bf16_to_f32",))
    return {"to_bf16": d.base, "to_f32": w.v}


@pytest.mark.parametrize("h,layout", BF_SHAPES)
def test_relu_bf16_and_casts(h, layout):
    """k_relu_fwd_y_bf16, k_relu_bwd_y_bf16 at both ACC and the two conversions, at >= 3 grid passes on 8 SMs"""
    rs = np.random.RandomState(200 + h)
    with M.few_sms():
        relu_bf16_cases(h, layout, bf_rows(h, FEW_CTAS), rs)
        cast_cases(h, layout, bf_rows(ld_of(h, layout), FEW_CTAS), rs)
    RAN.add(("bf16", h, layout))


# ------------------------------------------------------------------------------------------------ bf16 dropout ---
DROP16_H = (1, 7, 8, 9, 41, 64, 602)
DROP16_RATES = (0.0, 0.3, 0.5)
SEED, STEP = M.SEED, M.STEP


def dropout_bf16_cases(h, n, rs, firsts=(12345, 2 ** 32 - 3)):
    x16 = torch.from_numpy(rs.randn(n, h).astype(np.float32) * 3).bfloat16().view(torch.int16)
    x16[torch.from_numpy(rs.rand(n, h) < 0.02)] = 0
    for layout in ("odd", "dense"):
        x = BFrame(n, h, NAN16, ld_of(h, layout), init=x16)
        xw = widen(x.v).cpu().numpy()
        for rate in DROP16_RATES:
            for first in firsts:
                what = "dropout_fwd_bf16 H=%d %s n=%d rate=%g first=%d" % (h, layout, n, rate, first)
                y = twice(lambda: outp(n, h, "vec"),
                          lambda o: LIB.roc_dropout_fwd_bf16(n, h, first, rate, SEED, STEP, x.v.data_ptr(), x.ld,
                                                             o.v.data_ptr(), o.ld, None), what)
                keep = oracle.dropout_mask(first, n, h, rate, SEED, STEP)
                want = torch.from_numpy(oracle.dropout_apply(xw, keep, rate)).to(DEV)
                assert same_bits(y.v, want), "%s: differs from the oracle" % what
    SEEN.add(("dropout_bf16",))


@pytest.mark.parametrize("h", DROP16_H)
def test_dropout_bf16(h):
    """k_dropout<1, 2, uint16_t> at rates 0, 0.3 and 0.5, odd and dense bf16 pitches, >= 3 grid passes on 8 SMs"""
    with M.few_sms():
        dropout_bf16_cases(h, 3 * FEW_CTAS * 256 * 2 // ((h + 7) // 8) + 5, np.random.RandomState(300 + h))
    RAN.add(("dropout_bf16", h))


# ------------------------------------------------------------------------------------------------------- ELU ---
def elu_cases(h, layout, n, rs):
    vec = M.map_vec(h, layout)
    tag = "H=%d %s n=%d" % (h, layout, n)
    x_np = M.specials(rs.randn(n, h).astype(np.float32) * 4, rs)
    for v in (-104.0, -88.0, -20.5, 1e-40, -1e-40, -3e-39, 3e38):
        x_np[rs.rand(n, h) < 0.005] = v
    x = inp(x_np, layout)
    y = twice(lambda: outp(n, h, layout), lambda o: LIB.roc_activation_fwd(n, h, ELU, x.v.data_ptr(), x.ld,
                                                                               o.v.data_ptr(), o.ld, None), "elu " + tag)
    want = elu_ref(x.v)
    assert torch.equal(torch.isnan(y.v), torch.isnan(want)), "elu NaN " + tag
    inf = torch.isinf(want)
    assert torch.equal(y.v[inf].double(), want[inf]), "elu inf " + tag
    fin = torch.isfinite(want)
    r = float(((y.v.double() - want).abs() / ((2 * U + REF) * want.abs() + 2.0 ** -149))[fin].max())
    assert worst("ELU", r) <= 1.0, "elu %s: %.3g" % (tag, r)
    SEEN.add(("map", "elu_f", vec, False))
    g = inp(rs.randn(n, h).astype(np.float32), layout)
    old = inp(rs.randn(n, h).astype(np.float32), layout)
    y64 = y.v.double()
    res = g.v.double() * torch.where(y64 > 0, torch.ones_like(y64), y64 + 1)
    for acc in (False, True):
        what = "elu bwd %s acc=%d" % (tag, acc)
        dx = twice(lambda: outp(n, h, layout, init=old.v if acc else None),
                   lambda o: LIB.roc_activation_bwd(n, h, ELU, y.v.data_ptr(), y.ld, g.v.data_ptr(), g.ld,
                                                    o.v.data_ptr(), o.ld, int(acc), None), what)
        want = res + old.v.double() if acc else res
        nan = torch.isnan(want)
        assert torch.equal(torch.isnan(dx.v), nan), what
        bnd = 2 * U * res.abs() + (U * acc + REF) * want.abs() + 2.0 ** -149
        r = float(((dx.v.double() - want).abs() / bnd)[~nan].max())
        assert worst("ELU backward", r) <= 1.0, "%s: %.3g" % (what, r)
        SEEN.add(("map", "elu_b", vec, acc))


@pytest.mark.parametrize("h,layout", M.MAP_SHAPES)
def test_elu(h, layout):
    """k_map<OP_ELU_F> and <OP_ELU_B> at both ACC on the path the shape selects, at >= 3 grid passes on 8 SMs"""
    wq = h // 4 if M.map_vec(h, layout) == 4 else h
    with M.few_sms():
        elu_cases(h, layout, 3 * FEW_CTAS * 256 // wq + 13, np.random.RandomState(400 + h))
    RAN.add(("elu", h, layout))


# --------------------------------------------------------------------------------- sigmoid cross-entropy ---
ML_C = (1, 2, 4, 8, 16, 32, 33, 130)


def ml_vec(layout):
    return 4 if layout == "vec" else 1


def ml_lanes(c, vec):
    q = (c + vec - 1) // vec
    return next(l for l in (1, 2, 4, 8, 16, 32) if l >= q or l == 32)


def ml_rows(c, vec, ctas):
    """>= 3 grid passes, the last row group of a warp ragged"""
    rpb = 256 // ml_lanes(c, vec)
    return 3 * ctas * rpb + rpb // 2 + 3


def ml_data(n, c, rs):
    z = (rs.randn(n, c) * 4).astype(np.float32)
    for v in (0.0, -0.0, -100.0, 100.0, -88.5, 17.0, -17.0, 0.5, -0.5):
        z[rs.rand(n, c) < 0.01] = v
    y = rs.rand(n, c) < 0.3
    kind = rs.randint(0, 4, size=n)
    y[kind == 1] = z[kind == 1] > 0          # exact matches
    y[kind == 2] = True
    y[kind == 3] = False
    mask = rs.randint(0, 4, size=n).astype(np.int32)
    mask[rs.rand(n) < 0.02] = 7              # outside 0..3: counts nowhere
    mask[rs.rand(n) < 0.02] = -1
    return z, y, mask, M.norm_degrees(n, rs)


def ml_call(n, c, z, lb, mask, g, row_end, metrics):
    return LIB.roc_sigmoid_xent_bwd(n, c, z.v.data_ptr(), z.ld, lb.data_ptr(), lb.stride(0), mask.data_ptr(),
                                    g.v.data_ptr(), g.ld, row_end.data_ptr() if row_end is not None else None,
                                    COL_LEFT, metrics.data_ptr() if metrics is not None else None, None)


def ml_metrics(m):
    """(loss [3], counts dict) of a roc_multilabel_metrics read back as 18 doubles"""
    m = m.cpu()
    cnt = m[3:18].view(torch.int64).tolist()
    return m[:3].tolist(), {k: cnt[3 * i:3 * i + 3] for i, k in enumerate(("rows", "exact", "tp", "fp", "fn"))}


def ml_cases(c, layout, n, data):
    """gradient with and without the fused norm, with and without metrics; returns the gradients, counts and losses"""
    vec = ml_vec(layout)
    lanes = ml_lanes(c, vec)
    z_np, y_np, mask_np, deg = (a[:n] for a in data)
    z = inp(z_np, layout)
    words = (c + 31) // 32
    lb = torch.full((n, words + 1), -1, dtype=torch.int32, device=DEV)     # a pitch past W, pad words all ones
    lb[:, :words] = torch.from_numpy(pack_multilabels(y_np).view(np.int32)).to(DEV)
    mask, _ = guarded(mask_np, -7)
    row_end = torch.from_numpy(COL_LEFT + np.cumsum(deg)).to(DEV)
    d32 = torch.from_numpy(np.sqrt(deg.astype(np.float32)).astype(np.float64)).to(DEV)
    z64 = z.v.double()
    s64 = torch.sigmoid(z64)
    y64 = torch.from_numpy(y_np).to(DEV).double()
    train = torch.from_numpy(mask_np == _lib.MASK_TRAIN).to(DEV)[:, None]
    g64 = torch.where(train, s64 - y64, torch.zeros((), dtype=torch.float64, device=DEV))
    ebound = torch.where(z64 >= 0, 4 * U, 9 * U) * s64 + U * g64.abs()
    _, want_m = ml_oracle(z_np, y_np, mask_np)
    loss_k = (10 if vec == 4 else 7) * U + n * c * 2.0 ** -53
    outs, plain = {}, None
    for norm in (False, True):
        re_ = row_end if norm else None
        for with_m in (True, False):
            what = "sigmoid_xent C=%d %s n=%d norm=%d metrics=%d" % (c, layout, n, norm, with_m)
            runs = []
            for _ in range(2):
                g = outp(n, c, layout)
                m, mb = guarded(torch.zeros(18, dtype=torch.float64), SENT) if with_m else (None, None)
                ok(ml_call(n, c, z, lb, mask, g, re_, m), what)
                g.assert_outside_unchanged(what=what)
                if with_m:
                    guard_ok(mb, what)
                runs.append((g, ml_metrics(m) if with_m else None))
            (g, met), (g2, met2) = runs
            assert same_bits(g.v, g2.v), "%s: two runs differ" % what
            if with_m:
                # one budget: the loss has the same bits run to run (the header's promise); the counts are exact
                assert met == met2, "%s: two runs differ in the metrics" % what
                loss, counts = met
                for k, v in counts.items():
                    assert v == want_m[k], "%s: %s %s, want %s" % (what, k, v, want_m[k])
                for s in range(3):
                    err, bound = abs(loss[s] - want_m["loss"][s]), loss_k * want_m["loss"][s]
                    assert err <= bound, "%s: split %d loss %.17g, fp64 %.17g" % (what, s, loss[s], want_m["loss"][s])
                    if bound > 0:
                        worst("sigmoid loss", err / bound)
                outs["counts norm=%d" % norm] = counts
                outs["loss norm=%d" % norm] = loss
                gm = g
            else:
                assert same_bits(g.v, gm.v), "%s: metrics = NULL changes the gradient" % what
            SEEN.add(("sigmoid", vec, lanes))
        # the gradient against fp64: rows of degree 0 (divisor 0) are checked bit for bit below
        rows = torch.ones(n, dtype=torch.bool, device=DEV)
        want, bnd = g64, ebound
        if norm:
            rows = d32 > 0
            d = torch.where(rows, d32, torch.ones_like(d32))[:, None]
            want = g64 / d
            bnd = bnd / d + U * want.abs()
        bnd = bnd + REF * want.abs() + 4 * 2.0 ** -149
        what = "sigmoid_xent C=%d %s n=%d norm=%d" % (c, layout, n, norm)
        r = float(((g.v.double() - want).abs() / bnd)[rows].max())
        assert worst("sigmoid gradient", r) <= 1.0, "%s: worst |error| / bound %.3g" % (what, r)
        assert bool((g.v[rows & ~train[:, 0]] == 0).all()), "%s: a row outside the training mask has a gradient" % what
        outs["g norm=%d" % norm] = g.v
        if not norm:
            plain = g
            continue
        # the fused norm == the plain gradient followed by roc_indegree_norm, bit for bit (degree 0: NaN / inf)
        want = outp(n, c, layout)
        ok(LIB.roc_indegree_norm(0, n - 1, COL_LEFT, c, row_end.data_ptr(), plain.v.data_ptr(), plain.ld,
                                 want.v.data_ptr(), want.ld, None, None), "roc_indegree_norm")
        assert same_bits(g.v, want.v), "%s: fused norm differs from the gradient + roc_indegree_norm" % what
    return outs


@pytest.mark.parametrize("layout", ["vec", "odd"])
@pytest.mark.parametrize("c", ML_C)
def test_sigmoid_xent(c, layout):
    """k_sigmoid_xent at every L on both VEC paths, fused norm x metrics / NULL, at >= 3 grid passes on 8 SMs"""
    n = ml_rows(c, ml_vec(layout), FEW_CTAS)
    data = ml_data(n, c, np.random.RandomState(500 + c))
    with M.few_sms():
        ml_cases(c, layout, n, data)
    RAN.add(("sigmoid", c, layout))


# ------------------------------------------------------------------------------------------------ batch norm ---
BN_H = (1, 3, 257, 300, 512, 602, 1024, 1025)


def bn_shape(h):
    """(TY, colBlocks) of bn_shape in batchnorm.cu"""
    tx = min((h + 3) // 4, 64)
    return 256 // tx, ((h + 3) // 4 + tx - 1) // tx


def bn_rows(h, sm):
    """3 passes of the streaming kernels' grid (8 CTAs per SM, TY rows per CTA and step, 4 steps per pass), then a
    ragged pass longer than one step: there the rows r + u * step past the end include the guard row below"""
    ty, _ = bn_shape(h)
    step = sm * 8 * ty
    return 3 * 4 * step + step + 37


def bn_save(h, fill=0.0):
    """a, b (fp32) and mean, invstd (fp64) between guards: (views, buffers)"""
    made = [guarded(torch.full((h,), fill, dtype=dt), SENT) for dt in (torch.float32, torch.float32, torch.float64,
                                                                        torch.float64)]
    return [v for v, _ in made], [b for _, b in made]


def bn_fwd_call(x, gamma, beta, rm, rv, training, relu, y, save, ws):
    a, b, mean, inv = save
    return LIB.roc_batchnorm_fwd(x.rows, x.h, x.v.data_ptr(), x.ld, gamma.data_ptr(), beta.data_ptr(), 1e-5, 0.1,
                                 rm.data_ptr(), rv.data_ptr(), int(training), int(relu), y.v.data_ptr(), y.ld,
                                 a.data_ptr(), b.data_ptr(), mean.data_ptr(), inv.data_ptr(), ws.data_ptr(),
                                 ws.numel(), None)


def ratio(got, want, bound):
    return float(((got.double() - want).abs() / (bound + REF * want.abs() + 1e-300)).max())


def bn_cases(h, n, seed):
    """training (plain, relu), inference (plain, relu) and every backward; returns every output"""
    _, cb = bn_shape(h)
    multi = cb > 1
    x0, g0, gamma, beta, rm0, rv0 = bn_inputs(n, h, seed)
    x, g = inp(x0, "vec"), inp(g0, "vec")
    x64 = x.v.double()
    ws = torch.empty(max(LIB.roc_batchnorm_workspace_bytes(n, h), 16), dtype=torch.uint8, device=DEV)
    ref = bn_forward(x.v, gamma, beta, rm0, rv0, training=True)
    base = torch.from_numpy(np.random.RandomState(seed).randn(n, h).astype(np.float32)).to(DEV)
    outs = {}
    for relu in (False, True):
        what = "batchnorm H=%d n=%d relu=%d" % (h, n, relu)
        runs = []
        for _ in range(2):
            y = outp(n, h, "vec")
            (rm, rmb), (rv, rvb) = guarded(rm0, SENT), guarded(rv0, SENT)
            save, bufs = bn_save(h)
            ok(bn_fwd_call(x, gamma, beta, rm, rv, True, relu, y, save, ws), what)
            y.assert_outside_unchanged(what=what)
            for bb in [rmb, rvb] + bufs:
                guard_ok(bb, what)
            runs.append(dict(y=y.v, rm=rm, rv=rv, a=save[0], b=save[1], mean=save[2], invstd=save[3]))
        for k in runs[0]:
            assert same_bits(runs[0][k], runs[1][k]) if runs[0][k].dtype == torch.float32 else \
                torch.equal(runs[0][k].view(torch.int64), runs[1][k].view(torch.int64)), "%s: two runs differ" % what
        r = runs[0]
        bound = K_Y * U * ((x64 * ref["a"]).abs() + ref["b"].abs())
        q = ratio(r["y"], torch.relu(ref["y"]) if relu else ref["y"], bound)
        assert worst("batchnorm y", q) <= 1.0, "%s: y %.3g" % (what, q)
        assert bool((r["mean"] - ref["mean"]).abs().le(1e-12 * (1 + ref["mean"].abs())).all()), what + ": mean"
        for k, rk in (("rm", "run_mean"), ("rv", "run_var")):
            q = ratio(r[k], ref[rk], 2 * U * ref[rk].abs() + 1e-30)
            assert worst("batchnorm running", q) <= 1.0, "%s: %s %.3g" % (what, rk, q)
        outs.update({"fwd relu=%d %s" % (relu, k): v for k, v in r.items()})
        SEEN.add(("bn_reduce", False, False, multi))
        SEEN.add(("bn_norm", relu, multi))
        # backward: the mask is the forward's own test, fma(x, a, b) > 0 on the saved fp32 a, b
        gm = g.v.double()
        if relu:
            gm = torch.where(x64 * r["a"].double() + r["b"].double() > 0, gm, 0.0)
        bwd = bn_backward(x.v, gm, gamma, ref["mean"], ref["var"])
        dbound = K_DX * U * (bwd["Ag"].abs() + bwd["Bx"].abs() + bwd["C"].abs())
        for acc in (False, True):
            wb = "%s backward acc=%d" % (what, acc)
            runs = []
            for need_dx in (True, True, False):
                dx = outp(n, h, "vec", init=base if acc else None)
                (dgam, dgb), (dbet, dbb) = guarded(torch.zeros(h), SENT), guarded(torch.zeros(h), SENT)
                ok(LIB.roc_batchnorm_bwd(n, h, x.v.data_ptr(), x.ld, g.v.data_ptr(), g.ld, int(relu), gamma.data_ptr(),
                                         r["a"].data_ptr(), r["b"].data_ptr(), r["mean"].data_ptr(),
                                         r["invstd"].data_ptr(), dgam.data_ptr(), dbet.data_ptr(),
                                         dx.v.data_ptr() if need_dx else None, dx.ld, int(acc), ws.data_ptr(),
                                         ws.numel(), None), wb)
                dx.assert_outside_unchanged(cols=h if need_dx else 0, what=wb)
                guard_ok(dgb, wb)
                guard_ok(dbb, wb)
                runs.append((dx.v, dgam, dbet))
            assert same_bits(runs[0][0], runs[1][0]), "%s: two runs differ" % wb
            for i in (1, 2):      # dX = NULL gives the same dgamma, dbeta
                assert same_bits(runs[0][i], runs[1][i]) and same_bits(runs[0][i], runs[2][i]), "%s: dgamma / dbeta" % wb
            dx, dgam, dbet = runs[0]
            want = bwd["dx"] + (base.double() if acc else 0)
            bnd = dbound + (2 * U * (base.double().abs() + bwd["dx"].abs()) if acc else 0)
            q = ratio(dx, want, bnd)
            assert worst("batchnorm dx", q) <= 1.0, "%s: dx %.3g" % (wb, q)
            # the fp64 reference's mean carries its own rounding, 2^-50 |mean|, into every xhat: on a constant column
            # the kernel's mean is exact and its dgamma 0, the reference's a few 1e-11
            ref_mean = REF * ref["mean"].abs() / torch.sqrt(ref["var"] + 1e-5) * gm.abs().sum(0)
            q = max(ratio(dgam, bwd["dgamma"], K_RED * U * bwd["gxhat"].abs().sum(0) + ref_mean),
                    ratio(dbet, bwd["dbeta"], K_RED * U * gm.abs().sum(0)))
            assert worst("batchnorm dgamma, dbeta", q) <= 1.0, "%s: %.3g" % (wb, q)
            outs.update({"bwd relu=%d acc=%d %d" % (relu, acc, i): v for i, v in enumerate(runs[0])})
            SEEN.add(("bn_reduce", True, relu, multi))
            SEEN.add(("bn_apply", relu, acc, multi))
    # inference: the running statistics' affine map; nothing but y is written
    eref = bn_forward(x.v, gamma, beta, rm0, rv0, training=False)
    for relu in (False, True):
        what = "batchnorm inference H=%d n=%d relu=%d" % (h, n, relu)
        y = twice(lambda: outp(n, h, "vec"), lambda o: bn_fwd_call(x, gamma, beta, rm0.clone(), rv0.clone(), False,
                                                                     relu, o, bn_save(h, SENT)[0], ws), what)
        rm, rv = rm0.clone(), rv0.clone()
        save, bufs = bn_save(h, SENT)
        ok(bn_fwd_call(x, gamma, beta, rm, rv, False, relu, outp(n, h, "vec"), save, ws), what)
        assert same_bits(rm, rm0) and same_bits(rv, rv0), "%s: running statistics written" % what
        assert all(bool((bb == SENT).all()) for bb in bufs), "%s: a saved value written" % what
        q = ratio(y.v, torch.relu(eref["y"]) if relu else eref["y"], K_Y * U * ((x64 * eref["a"]).abs() +
                                                                               eref["b"].abs()))
        assert worst("batchnorm y", q) <= 1.0, "%s: y %.3g" % (what, q)
        outs["infer relu=%d" % relu] = y.v
        SEEN.add(("bn_norm", relu, multi))
    return outs


@pytest.mark.parametrize("h", BN_H)
def test_batchnorm(h):
    """every batch-norm kernel, colBlocks 1 .. 5 with a partial last column group, at >= 3 passes of the streaming
    kernels' grid on 8 SMs"""
    with M.few_sms():
        bn_cases(h, bn_rows(h, M.FEW_SMS), seed=600 + h)
    RAN.add(("batchnorm", h))


# ------------------------------------------------------------------------------------------ attention scores ---
# (14, 43), (2, 301): H = 602 on 3 column blocks; (602, 1) and (512, 2): the last column group spans heads;
# (31, 33): H = 1023, a partial last group; (8, 128): H = 1024 on 4 column blocks; (4, 16): one column block
AT_SHAPES = ((14, 43), (2, 301), (602, 1), (8, 128), (512, 2), (31, 33), (4, 16))
K_DX_AT, K_DA_AT = 3, 2        # test_gat_heads_gpu.py's K_DX, K_DA


def at_fwd_shape(h, heads):
    """(TR, perSm) of fwd_shape / scores_fwd in attn_scores.cu"""
    p = h | 1
    tr = min(max((256 // heads + 31) // 32 * 32, 32), 256)
    while tr > 32 and tr * p * 4 > 72 * 1024:
        tr -= 32
    smem = (2 * h + tr * p) * 4
    return tr, min(max(200 * 1024 // smem, 1), 8)


def at_rows(h, heads, sm):
    """>= 3 passes of the forward's grid, the last tile ragged"""
    tr, per_sm = at_fwd_shape(h, heads)
    return 3 * sm * per_sm * tr + tr // 2 + 3


def at_cases(heads, f, layout, n, seed):
    h = heads * f
    vec = layout == "vec"
    multi = bn_shape(h)[1] > 1
    tag = "heads=%d F=%d %s n=%d" % (heads, f, layout, n)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = inp(torch.randn((n, h), generator=gen, device=DEV), layout)
    a = torch.randn((2 * heads, f), generator=gen, device=DEV) / math.sqrt(f)
    ds = inp(torch.randn((n, 2 * heads), generator=gen, device=DEV), "vec")
    base = torch.randn((n, h), generator=gen, device=DEV)
    s = twice(lambda: outp(n, 2 * heads, "vec"),
              lambda o: LIB.roc_attn_scores_fwd(n, h, heads, x.v.data_ptr(), x.ld, a.data_ptr(), o.v.data_ptr(), o.ld,
                                                None), "attn_scores_fwd " + tag)
    want, b = scores_ref(x.v, a, heads)
    q = ratio(s.v, want, f * U / (1 - f * U) * b)
    assert worst("attention S", q) <= 1.0, "attn_scores_fwd %s: %.3g" % (tag, q)
    SEEN.add(("attn_fwd", vec))
    ws = torch.empty(max(LIB.roc_attn_scores_workspace_bytes(n, h, heads), 16), dtype=torch.uint8, device=DEV)
    ref = scores_bwd_ref(x.v, a, ds.v, heads)
    outs = {"S": s.v}
    for acc in (False, True):
        what = "attn_scores_bwd %s acc=%d" % (tag, acc)
        runs = []
        for need_dx in (True, True, False):
            dx = outp(n, h, layout, init=base if acc else None)
            da, dab = guarded(torch.zeros(2 * heads * f), SENT)
            ok(LIB.roc_attn_scores_bwd(n, h, heads, x.v.data_ptr(), x.ld, a.data_ptr(), ds.v.data_ptr(), ds.ld,
                                       dx.v.data_ptr() if need_dx else None, dx.ld, int(acc), da.data_ptr(),
                                       ws.data_ptr(), ws.numel(), None), what)
            dx.assert_outside_unchanged(cols=h if need_dx else 0, what=what)
            guard_ok(dab, what)
            runs.append((dx.v, da))
        assert same_bits(runs[0][0], runs[1][0]), "%s: two runs differ" % what
        assert same_bits(runs[0][1], runs[1][1]) and same_bits(runs[0][1], runs[2][1]), "%s: dA" % what
        dx, da = runs[0]
        bnd = K_DX_AT * U * ref["dx_abs"]
        want = ref["dx"]
        if acc:
            want = want + base.double()
            bnd = bnd + 2 * U * (base.double().abs() + ref["dx"].abs())
        q = ratio(dx, want, bnd)
        assert worst("attention dX", q) <= 1.0, "%s: dX %.3g" % (what, q)
        q = ratio(da.view(2 * heads, f), ref["da"], K_DA_AT * U * ref["da_abs"])
        assert worst("attention dA", q) <= 1.0, "%s: dA %.3g" % (what, q)
        outs["dx %d" % acc], outs["da %d" % acc] = dx, da
        SEEN.add(("attn_bwd", vec, multi))
    return outs


@pytest.mark.parametrize("layout", ["vec", "odd"])
@pytest.mark.parametrize("heads,f", AT_SHAPES)
def test_attn_scores(heads, f, layout):
    """both forward and backward paths (X 16-byte rows or not), at >= 3 passes of the forward's grid on 8 SMs"""
    with M.few_sms():
        at_cases(heads, f, layout, at_rows(heads * f, heads, M.FEW_SMS), seed=700 + heads * 7 + f)
    RAN.add(("attn", heads, f, layout))


# ---------------------------------------------------------------------------------------- the whole chip ---
def test_late_full_chip_passes():
    """One case per kernel with no SM reserve, at >= 3 full grid passes plus a ragged tail on this device"""
    sm, ctas = M.nsm(), M.nsm() * 16
    rs = np.random.RandomState(7)
    sa_cases(64, "vec", sa_rows(64, "vec", ctas), rs)
    sa_cases(41, "odd", sa_rows(41, "odd", ctas), rs)
    relu_bf16_cases(41, "odd", bf_rows(41, ctas), rs)
    cast_cases(41, "odd", bf_rows(ld_of(41, "odd"), ctas), rs)
    dropout_bf16_cases(64, 3 * ctas * 256 * 2 // 8 + 77, rs, firsts=(2 ** 32 - 3,))
    elu_cases(64, "vec", 3 * ctas * 256 // 16 + 13, rs)
    for c, layout in ((33, "vec"), (8, "odd")):
        n = ml_rows(c, ml_vec(layout), ctas)
        ml_cases(c, layout, n, ml_data(n, c, rs))
    bn_cases(300, bn_rows(300, sm), seed=11)
    at_cases(14, 43, "vec", at_rows(602, 14, sm), seed=12)


# ------------------------------------------------------------------------------------------------ SM budgets ---
def same_everywhere(results, what):
    """every budget's outputs have the bits of the first's"""
    first = results[0][1]
    for sm, r in results[1:]:
        for k, v in first.items():
            w = r[k]
            if torch.is_tensor(v):
                same = torch.equal(v.contiguous().view(torch.uint8), w.contiguous().view(torch.uint8))
            else:
                same = v == w
            assert same, "%s: %s differs between %d and %d SMs" % (what, k, results[0][0], sm)


def test_sm_budget_invariance():
    """The same inputs on the whole chip, an odd SM count and 8 SMs give the same bits.  The sigmoid loss is the
    exception: each thread sums the rows it visits, so its bits depend on gridDim; it is held to its fp64 bound at
    every budget (inside ml_cases) and its counts must be equal."""
    cases = [
        ("scaled_add H=64 vec", lambda: sa_cases(64, "vec", sa_rows(64, "vec", FEW_CTAS), np.random.RandomState(1))),
        ("scaled_add H=41 odd", lambda: sa_cases(41, "odd", sa_rows(41, "odd", FEW_CTAS), np.random.RandomState(2))),
        ("bf16 relu H=41 odd", lambda: relu_bf16_cases(41, "odd", bf_rows(41, FEW_CTAS), np.random.RandomState(3))),
        ("casts H=41 odd", lambda: cast_cases(41, "odd", bf_rows(42, FEW_CTAS), np.random.RandomState(4))),
        ("batchnorm H=602", lambda: bn_cases(602, bn_rows(602, M.FEW_SMS), seed=5)),
        ("batchnorm H=3", lambda: bn_cases(3, bn_rows(3, M.FEW_SMS), seed=6)),
        ("attention (14, 43)", lambda: at_cases(14, 43, "vec", at_rows(602, 14, M.FEW_SMS), seed=7)),
        ("attention (8, 128)", lambda: at_cases(8, 128, "odd", at_rows(1024, 8, M.FEW_SMS), seed=8)),
    ]
    for c, layout in ((33, "vec"), (5, "odd"), (1, "vec")):
        n = ml_rows(c, ml_vec(layout), FEW_CTAS)
        data = ml_data(n, c, np.random.RandomState(9 + c))
        cases.append(("sigmoid C=%d %s" % (c, layout), lambda c=c, layout=layout, n=n, data=data:
                      {k: v for k, v in ml_cases(c, layout, n, data).items() if not k.startswith("loss")}))
    for what, run in cases:
        results = []
        for sm in budgets():
            with sms(sm):
                results.append((sm, run()))
        same_everywhere(results, what)


# -------------------------------------------------------------------------------------------------- coverage ---
def test_late_dispatch_table_covered():
    """Every launch variant the dispatch rules above can produce was reached: both paths of scaled_add forward and
    backward, the bf16 relu at both ACC, both conversions, the bf16 dropout, ELU on both paths (and ACC), every
    (VEC, L) of k_sigmoid_xent, every batch-norm kernel instantiation with one and with several column blocks, and
    both attention paths.  Prints the worst error-to-bound ratio per family."""
    wanted_runs = ({("scaled_add", h, lay) for h, lay in SA_SHAPES} | {("bf16", h, lay) for h, lay in BF_SHAPES} |
                   {("dropout_bf16", h) for h in DROP16_H} | {("elu", h, lay) for h, lay in M.MAP_SHAPES} |
                   {("sigmoid", c, lay) for c in ML_C for lay in ("vec", "odd")} | {("batchnorm", h) for h in BN_H} |
                   {("attn", hd, f, lay) for hd, f in AT_SHAPES for lay in ("vec", "odd")})
    if not wanted_runs <= RAN:
        pytest.skip("%d of the %d matrix cases did not run in this process" % (len(wanted_runs - RAN), len(wanted_runs)))
    for k in sorted(WORST):
        print("worst |error| / bound  %-24s %.4f" % (k, WORST[k]))
    wanted = {("scaled_add", v) for v in (4, 1)} | {("scaled_add_bwd", v) for v in (4, 1)}
    wanted |= {("relu_fwd_y_bf16",), ("f32_to_bf16",), ("bf16_to_f32",), ("dropout_bf16",)}
    wanted |= {("relu_bwd_y_bf16", acc) for acc in (False, True)}
    wanted |= {("map", "elu_f", v, False) for v in (4, 1)} | {("map", "elu_b", v, acc) for v in (4, 1)
                                                               for acc in (False, True)}
    wanted |= {("sigmoid", v, l) for v in (4, 1) for l in (1, 2, 4, 8, 16, 32)}
    for multi in (False, True):
        wanted |= {("bn_reduce", False, False, multi)} | {("bn_reduce", True, r, multi) for r in (False, True)}
        wanted |= {("bn_norm", r, multi) for r in (False, True)}
        wanted |= {("bn_apply", r, acc, multi) for r in (False, True) for acc in (False, True)}
        wanted |= {("attn_bwd", v, multi) for v in (True, False)}
    wanted |= {("attn_fwd", v) for v in (True, False)}
    missing = wanted - SEEN
    assert not missing, "never launched: %s" % sorted(missing, key=str)
    assert SEEN <= wanted, "outside the table: %s" % sorted(SEEN - wanted, key=str)
