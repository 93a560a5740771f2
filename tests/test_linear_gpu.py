"""GPU suite: the Linear GEMMs against an fp64 reference, element by element, at every kernel instantiation.

The tensor-core kernels (k_tc_linear<NC, EPI> for forward and dX, k_tc_linear_dw<NC> for dW; 3xTF32 on wgmma) and
the exact-fp32 SIMT kernels (ROC_B200_GEMM=notc) must meet the bound of tests/tf32_bound.py.  That bound is calibrated
on the CPU (test_tf32_bound_cpu.py) so that a correct kernel passes by a wide margin and a kernel that loses any one of
its three MMAs fails by a wide margin.  For forward and dX that holds at every shape here (K = the layer width).  For
dW, K is the row count, and the bound follows the kernel's split-K ranges; it keeps that power for ranges of 416 rows,
the length test_dw_matrix runs at and asserts.  The production and full-size dW cases have ranges of thousands of
rows: they check the result at scale, not the loss of a lo term.  The reference is torch float64 on the GPU, built
from the same fp32 inputs (dropout applied with the same packed mask and the same fp32 scaling), with the epilogues
composed in fp64.

roc_last_gemm_info reports which instantiation ran and how it was launched, so each case asserts the instantiation
and pipeline regime it targets: the persistent forward loop with >= 3 row tiles per CTA, and dW splits that wrap the
TMA ring at least three times or hold no rows at all.  test_matrix_covered checks at the end that every instantiation
and regime was reached.  Pad columns of every input hold NaN and pad columns of every output a sentinel: no NaN may
reach a result and no sentinel may change.

Worst |error| / bound per data family (C_BOUND = 4), measured on one H100 80GB HBM3 (700 W):
  tensor cores  random_sign 0.26, positive 0.21, scaled_rows 0.24, zeros 0.29
  SIMT          random_sign 0.05, positive 0.07, scaled_rows 0.24, zeros 0.23
The tensor cores' accumulation truncates: against a sqrt(K) model of round-to-nearest accumulation, all-positive data
at K = 602 reached 1.9x the bound (tests/tf32_bound.py).  Row blocks reproduce a single call bit for bit: a row's
result does not depend on its position in a 128-row tile.  The whole file runs in about 15 s.
test_config2_full_size_forward_and_dw (4 194 304 rows, X alone 10 GB; peak 14.8 GB of GPU memory) skips when the GPU
has too little free memory; deselect it with -k "not full_size"."""
import math

import numpy as np
import pytest
import torch

import tf32_bound as tb
from roc_b200 import _lib
from roc_b200 import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = -1.2345e38
EPI_RELU, EPI_OMASK, EPI_RELUOF, EPI_NORM, EPI_ACC = 1, 2, 4, 8, 16
INSTANCES = (0, EPI_NORM, EPI_OMASK, EPI_OMASK | EPI_RELUOF | EPI_NORM)   # the rest take the generic kernel (-1)
BIG_ROWS = 3 * 132 * 128 + 77          # >= 3 row tiles per CTA for every N-tile count on a 132-SM H100
DW_SPLIT_ROWS = 416                    # rows per dW split in the matrix: 13 k-blocks, >= 3 turns of a 4-stage ring
DW_EMPTY_ROWS = 8449                   # the last splits hold no rows

SEEN = set()        # (kind, nc, instantiation) of tensor-core launches, and regime tags
RAN = set()         # ids of the matrix cases that ran in this process
WORST = {}          # (path, family) -> worst |error| / bound


def instance(epi):
    return epi if epi in INSTANCES else -1


def fwd_nc(n):
    return 1 if n <= 32 else 2 if n <= 64 else 4


def dw_nc(out_dim):
    c = (out_dim + 31) // 32
    return 1 if c <= 1 else 2 if c <= 2 else 4 if c <= 4 else 8


def gen(seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return g


def buf(rows, h, fill):
    """[rows][h] view of a [rows][ld] tensor, ld a multiple of 4 with at least 4 pad columns, all filled with `fill`"""
    ld = (h + 3) // 4 * 4 + 4
    return torch.full((rows, ld), fill, device=DEV, dtype=torch.float32)[:, :h]


def padded_with_nan(t):
    v = buf(t.shape[0], t.shape[1], float("nan"))
    v.copy_(t)
    return v


def pads(t):
    return t.as_strided((t.shape[0], t.stride(0) - t.shape[1]), (t.stride(0), 1), t.shape[1])


def out_buf(rows, h, init=None):
    v = buf(rows, h, SENTINEL)
    v.copy_(init if init is not None else torch.zeros((rows, h), device=DEV))
    return v


def unpack(mask, h):
    """bool [rows][h] keep-mask of a packed roc_dropout_mask"""
    cols = torch.arange(h, device=DEV)
    return ((mask[:, cols >> 5] >> (cols & 31)) & 1).bool()


def scale_of(rate):
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(rate)))   # mask_args' fp32 1 / (1 - rate)


def apply_mask(x, mask, rate):
    """the dropout the kernels fuse into their operand loads, in fp32 exactly as they do it"""
    if mask is None:
        return x
    return torch.where(unpack(mask, x.shape[1]), x * scale_of(rate), torch.zeros((), device=DEV))


def degrees(rows, g, col_left=1000):
    """row_end (global end offsets, int64 on the device) of a graph with degrees 1..40 and a few hubs"""
    deg = torch.randint(1, 41, (rows,), generator=g, device=DEV)
    deg[::997] = 70000
    return col_left + torch.cumsum(deg, 0), col_left


def row_divisor(row_end, col_left):
    start = torch.cat([torch.tensor([col_left], device=DEV), row_end[:-1]])
    return torch.sqrt((row_end - start).to(torch.float32)).double()   # sqrtf((float)deg), as the epilogue divides


def compose(ref, bnd, relu=False, omask=None, oscale=1.0, relu_of=None, div=None, old=None):
    """the epilogue (relu -> dropout backward -> relu mask -> / sqrt(deg) -> accumulate) in fp64, on the reference and
    its bound; each fp32 rounding of an epilogue step adds 2^-24 of the value it rounds"""
    if relu:
        ref = ref.clamp_min(0.0)
    if omask is not None:
        ref = torch.where(omask, ref * oscale, torch.zeros((), device=DEV, dtype=ref.dtype))
        bnd = torch.where(omask, bnd * oscale, torch.zeros((), device=DEV, dtype=bnd.dtype))
    if relu_of is not None:
        keep = relu_of > 0
        ref = torch.where(keep, ref, torch.zeros((), device=DEV, dtype=ref.dtype))
        bnd = torch.where(keep, bnd, torch.zeros((), device=DEV, dtype=bnd.dtype))
    if div is not None:
        ref = ref / div[:, None]
        bnd = bnd / div[:, None]
    pre = ref
    if old is not None:
        ref = old.double() + ref
    return ref, bnd + 2.0 ** -22 * (pre.abs() + ref.abs())


def check(got, ref, bnd, path, family, what):
    assert not torch.isnan(got).any(), "%s: NaN in the result" % what
    r = tb.worst_ratio(got, ref, bnd)
    WORST[(path, family)] = max(WORST.get((path, family), 0.0), r)
    assert r <= 1.0, "%s: worst |error| / bound = %.3g" % (what, r)


def check_pads(*outs):
    for t in outs:
        assert bool((pads(t) == SENTINEL).all()), "a pad column of an output was written"


def info_of(which, path):
    info = _lib.last_gemm_info(which)
    assert info["path"] == (1 if path == "tc" else 2), info
    return info


# ---------------------------------------------------------------- forward and dX: all 15 instantiations ---
FWD_SPECS = [dict(relu=r, norm=n) for r in (False, True) for n in (False, True)]
DX_SPECS = [dict(omask=o, reluof=ro, norm=n, acc=a) for o, ro, n, a in
            ((0, 0, 0, 0), (0, 0, 1, 0), (1, 0, 0, 0), (1, 1, 1, 0), (0, 0, 0, 1), (0, 1, 1, 0), (1, 0, 0, 1))]
KS = (8, 13, 32, 41, 100, 602)
NS = {1: (32, 13), 2: (41, 64), 4: (200, 602, 100)}


def _matrix():
    cases, i = [], 0
    for nc in (1, 2, 4):
        for kind, specs in (("fwd", FWD_SPECS), ("dx", DX_SPECS)):
            for spec in specs:
                for big in (False, True):
                    c = dict(kind=kind, spec=spec, k=KS[i % len(KS)], n=NS[nc][i % len(NS[nc])],
                             rows=BIG_ROWS if big else (1, 127, 129)[i % 3], family=tb.FAMILIES[i % 4],
                             masked=(i % 2 == 0), seed=i)
                    cases.append(c)
                    i += 1
    return cases


MATRIX = _matrix()


def _id(c):
    s = c["spec"]
    e = "+".join(k for k, v in s.items() if v) or "plain"
    return "%s-%s-r%d-k%d-n%d-%s%s" % (c["kind"], e, c["rows"], c["k"], c["n"], c["family"],
                                      "-mask" if c["masked"] and c["kind"] == "fwd" else "")


def run_fwd(rows, k, n, family, relu, norm, masked, seed, rate=0.5):
    """one forward GEMM; returns (Y, reference, bound, expected EPI bits) after checking layout"""
    g = gen(seed)
    x = padded_with_nan(tb.family_data(family, rows, k, g, "a", DEV))
    w = tb.family_data(family, n, k, g, "b", DEV).contiguous()
    mask = K.dropout_mask(rows, k, seed, rate, (9 << 32) | seed, 3, DEV) if masked else None
    row_end, col_left = degrees(rows, g) if norm else (None, 0)
    y = out_buf(rows, n)
    K.linear_fwd_dropout(x, w, mask, rate if masked else 0.0, activation=int(relu), norm_row_end=row_end,
                         col_left=col_left, out=y)
    ref, bnd = tb.reference(apply_mask(x, mask, rate), w)
    ref, bnd = compose(ref, bnd, relu=relu, div=row_divisor(row_end, col_left) if norm else None)
    epi = (EPI_RELU if relu else 0) | (EPI_NORM if norm else 0)
    return dict(x=x, w=w, mask=mask, row_end=row_end, col_left=col_left, y=y, ref=ref, bnd=bnd, epi=epi, rate=rate)


def run_dx(rows, k, n, family, omask, reluof, norm, acc, seed, rate=0.3, parts=_lib.LINEAR_BWD_ONLY_DX):
    """one dX GEMM (K = the layer's outDim, N = its inDim) with the fused backward epilogue"""
    g = gen(seed)
    dy = padded_with_nan(tb.family_data(family, rows, k, g, "a", DEV))
    w = tb.family_data(family, k, n, g, "b", DEV).contiguous()       # W_mem[o * inDim + i]: [outDim = K][inDim = N]
    x = padded_with_nan(torch.randn((rows, n), generator=g, device=DEV))
    mask = K.dropout_mask(rows, n, seed, rate, (5 << 32) | seed, 7, DEV) if omask else None
    relu_of = padded_with_nan(torch.relu(torch.randn((rows, n), generator=g, device=DEV))) if reluof else None
    row_end, col_left = degrees(rows, g) if norm else (None, 0)
    old = torch.randn((rows, n), generator=g, device=DEV) if acc else None
    dx = out_buf(rows, n, old)
    dw = torch.zeros((k, n), device=DEV)
    K.linear_bwd_fused(x, w, None, dy, dw, dx, mask=mask, rate=rate if omask else 0.0, relu_of=relu_of,
                       norm_row_end=row_end, col_left=col_left, accumulate_dx=acc, parts=parts)
    ref, bnd = tb.reference(dy, w.T)
    ref, bnd = compose(ref, bnd, omask=unpack(mask, n) if omask else None, oscale=scale_of(rate),
                       relu_of=relu_of, div=row_divisor(row_end, col_left) if norm else None, old=old)
    epi = (EPI_OMASK if omask else 0) | (EPI_RELUOF if reluof else 0) | (EPI_NORM if norm else 0) | \
          (EPI_ACC if acc else 0)
    return dict(x=x, w=w, dy=dy, mask=mask, relu_of=relu_of, row_end=row_end, col_left=col_left, old=old, dx=dx,
                dw=dw, ref=ref, bnd=bnd, epi=epi, rate=rate)


def check_fwd_launch(info, path, rows, n, epi, kind):
    if path != "tc":
        return
    nc = fwd_nc(n)
    assert (info["nc"], info["epi"]) == (nc, instance(epi)), info
    assert info["grid_y"] == -(-n // (32 * nc)), info
    SEEN.add((kind, nc, instance(epi)))
    if -(-rows // 128) >= 3 * info["grid_x"]:
        SEEN.add(("multitile", nc, info["grid_y"]))


@pytest.mark.parametrize("path", ["tc", "notc"])
@pytest.mark.parametrize("case", MATRIX, ids=_id)
def test_fwd_dx_matrix(case, path, monkeypatch):
    if path == "notc":
        monkeypatch.setenv("ROC_B200_GEMM", "notc")
    c = case
    what = "%s %s" % (path, _id(c))
    if c["kind"] == "fwd":
        r = run_fwd(c["rows"], c["k"], c["n"], c["family"], masked=c["masked"], seed=c["seed"], **c["spec"])
        info = info_of(_lib.GEMM_FWD, path)
        out, again = r["y"], lambda: K.linear_fwd_dropout(
            r["x"], r["w"], r["mask"], r["rate"] if r["mask"] is not None else 0.0, activation=int(c["spec"]["relu"]),
            norm_row_end=r["row_end"], col_left=r["col_left"], out=out_buf(c["rows"], c["n"]))
    else:
        s = c["spec"]
        r = run_dx(c["rows"], c["k"], c["n"], c["family"], bool(s["omask"]), bool(s["reluof"]), bool(s["norm"]),
                   bool(s["acc"]), seed=c["seed"])
        info = info_of(_lib.GEMM_DX, path)
        out = r["dx"]

        def again():
            dx = out_buf(c["rows"], c["n"], r["old"])
            K.linear_bwd_fused(r["x"], r["w"], None, r["dy"], torch.zeros_like(r["dw"]), dx, mask=r["mask"],
                               rate=r["rate"] if r["mask"] is not None else 0.0, relu_of=r["relu_of"],
                               norm_row_end=r["row_end"], col_left=r["col_left"], accumulate_dx=bool(s["acc"]),
                               parts=_lib.LINEAR_BWD_ONLY_DX)
            return dx
    check_fwd_launch(info, path, c["rows"], c["n"], r["epi"], c["kind"])
    check(out, r["ref"], r["bnd"], path, c["family"], what)
    RAN.add((_id(c), path))
    check_pads(out)
    if c["rows"] == BIG_ROWS:
        assert torch.equal(again(), out), "%s: a repeated call differs" % what


def test_k7_takes_the_simt_path():
    """K < 8 is below what the tensor-core kernels take: the dispatcher must say so and the SIMT result must hold"""
    r = run_fwd(300, 7, 40, "random_sign", relu=False, norm=True, masked=True, seed=70)
    assert _lib.last_gemm_info(_lib.GEMM_FWD)["path"] == 2
    check(r["y"], r["ref"], r["bnd"], "notc", "random_sign", "fwd K=7")
    r = run_dx(300, 7, 40, "positive", omask=True, reluof=True, norm=True, acc=False, seed=71)
    assert _lib.last_gemm_info(_lib.GEMM_DX)["path"] == 2
    check(r["dx"], r["ref"], r["bnd"], "notc", "positive", "dX K=7")


# -------------------------------------------------------------------------------- dW: all 4 instantiations ---
DW_OUT = (16, 41, 64, 128, 200, 256)
DW_IN = (16, 100, 256, 300, 500, 602)     # 128-column M tiles: 1, 1, 2, 3, 4, 5 (partial last tile but at 256)


def dw_ring_rows(inn):
    """rows that give each of a 132-SM H100's dW splits (132 / M-tiles of them) DW_SPLIT_ROWS rows, the last a few
    less.  Longer splits accumulate more partial sums per range, and the bound of tests/tf32_bound.py then no longer
    tells a lost lo term from the truncation of a correct kernel (test_tf32_bound_cpu.py calibrates 416)."""
    return (132 // -(-inn // 128)) * DW_SPLIT_ROWS - 5


DW_MATRIX = [dict(out=o, inn=i, rows=rows, ring=(j == 0), family=tb.FAMILIES[(a + b + j) % 4],
                  masked=(a + b + j) % 2 == 0, seed=1000 + 100 * a + 10 * b + j)
             for a, o in enumerate(DW_OUT) for b, i in enumerate(DW_IN)
             for j, rows in enumerate((dw_ring_rows(i), DW_EMPTY_ROWS))]


def run_dw(rows, inn, out, family, masked, seed, rate=0.5, parts=_lib.LINEAR_BWD_ONLY_DW):
    """dW += dY^T dropout(X) on a non-zero dW (K = rows).  The reference's bound follows the split-K ranges the kernel
    reports (roc_last_gemm_info): each range accumulates on its own, then the partials are added in order."""
    g = gen(seed)
    x = padded_with_nan(tb.family_data(family, rows, inn, g, "a", DEV))
    dy = padded_with_nan(tb.family_data(family, rows, out, g, "b", DEV))
    mask = K.dropout_mask(rows, inn, seed, rate, (3 << 32) | seed, 1, DEV) if masked else None
    w = torch.randn((out, inn), generator=g, device=DEV)
    dw0 = torch.randn((out, inn), generator=g, device=DEV)
    dw = dw0.clone()
    K.linear_bwd_fused(x, w, None, dy, dw, None, mask=mask, rate=rate if masked else 0.0, parts=parts)
    info = _lib.last_gemm_info(_lib.GEMM_DW)
    assert info["v_per_split"] > 0 and info["v_per_split"] % 8 == 0, info
    acc = tb.RefAccumulator(split=info["v_per_split"])
    xd = apply_mask(x, mask, rate)
    for r0 in range(0, rows, 1 << 16):
        acc.add(dy[r0:r0 + (1 << 16)].T, xd[r0:r0 + (1 << 16)].T)
    ref, bnd = acc.result()
    ref, bnd = compose(ref, bnd, old=dw0)
    return dict(x=x, dy=dy, w=w, mask=mask, dw=dw, dw0=dw0, ref=ref, bnd=bnd, rate=rate, info=info)


def _dw_id(c):
    return "dw-r%d-in%d-out%d-%s%s" % (c["rows"], c["inn"], c["out"], c["family"], "-mask" if c["masked"] else "")


@pytest.mark.parametrize("path", ["tc", "notc"])
@pytest.mark.parametrize("case", DW_MATRIX, ids=_dw_id)
def test_dw_matrix(case, path, monkeypatch):
    if path == "notc":
        monkeypatch.setenv("ROC_B200_GEMM", "notc")
    c = case
    what = "%s dW rows %d %d x %d" % (path, c["rows"], c["out"], c["inn"])
    r = run_dw(c["rows"], c["inn"], c["out"], c["family"], c["masked"], c["seed"])
    info = info_of(_lib.GEMM_DW, path)
    check(r["dw"], r["ref"], r["bnd"], path, c["family"], what)
    if path == "tc":
        nc = dw_nc(c["out"])
        assert info["nc"] == nc and info["grid_y"] == -(-c["inn"] // 128) and info["grid_x"] == info["splits"], info
        assert info["v_per_split"] % 32 == 0 and info["splits"] * info["v_per_split"] >= c["rows"], info
        assert info["v_per_split"] <= DW_SPLIT_ROWS, info      # the split length the bound is calibrated for
        SEEN.add(("dw", nc, 0))
        if info["v_per_split"] // 32 >= 3 * info["stages"]:
            SEEN.add(("dw_ring_wrap", nc, 0))
        if (info["splits"] - 1) * info["v_per_split"] >= c["rows"]:
            SEEN.add(("dw_empty_split", nc, 0))
    RAN.add((_dw_id(c), path))
    if c["ring"]:
        dw = r["dw0"].clone()
        K.linear_bwd_fused(r["x"], r["w"], None, r["dy"], dw, None, mask=r["mask"],
                           rate=r["rate"] if r["mask"] is not None else 0.0, parts=_lib.LINEAR_BWD_ONLY_DW)
        assert torch.equal(dw, r["dw"]), "%s: a repeated call differs" % what


# --------------------------------------------------------------------- production shapes (bench.py CONFIGS) ---
# (config, inDim, outDim, forward: [(input mask, norm epilogue)], dX epilogues [(omask, reluof, norm, acc)], dW mask)
# as the host issues them: dropout fuses into a Linear only when the Linear is its one consumer (configs 2 and 4),
# the residual GCN and GraphSAGE read the dropout output twice and sum two dX (=, then +=); a first layer's input is
# a leaf, so it has no dX.
PRODUCTION = [
    (2, 602, 64, [(True, True)], [], True),
    (2, 64, 41, [(True, True)], [(1, 1, 1, 0)], True),
    (3, 100, 256, [(False, False)], [], False),
    (3, 256, 256, [(False, False)], [(0, 0, 0, 0), (0, 0, 0, 1)], False),
    (3, 256, 47, [(False, False)], [(0, 0, 0, 0), (0, 0, 0, 1)], False),
    (4, 602, 128, [(True, True)], [], True),
    (4, 128, 41, [(True, True)], [(1, 1, 1, 0)], True),
    (5, 602, 256, [(False, True), (False, False)], [], False),
    (5, 256, 256, [(False, True), (False, False)], [(0, 0, 0, 0), (0, 0, 0, 1)], False),
    (5, 256, 41, [(False, True), (False, False)], [(0, 0, 0, 0), (0, 0, 0, 1)], False),
]
PROD_ROWS = 300007


@pytest.mark.parametrize("cfg,inn,out,fwds,dxs,dwmask", PRODUCTION,
                         ids=["cfg%d-%dx%d" % (p[0], p[1], p[2]) for p in PRODUCTION])
def test_production_shapes(cfg, inn, out, fwds, dxs, dwmask):
    """At 300 007 rows a dW split holds thousands of rows: the bound checks the result at the shapes and split-K layout
    the host runs, but at that split length it would also admit a lost lo term (test_dw_matrix is the check for that,
    at 416-row splits).  Forward and dX keep their full power: their K is the layer width."""
    fam = "random_sign"
    for j, (masked, norm) in enumerate(fwds):
        r = run_fwd(PROD_ROWS, inn, out, fam, relu=False, norm=norm, masked=masked, seed=cfg * 100 + j)
        check_fwd_launch(info_of(_lib.GEMM_FWD, "tc"), "tc", PROD_ROWS, out, r["epi"], "fwd")
        check(r["y"], r["ref"], r["bnd"], "tc", fam, "cfg%d fwd %d -> %d" % (cfg, inn, out))
        del r
    for j, (om, ro, nm, ac) in enumerate(dxs):
        r = run_dx(PROD_ROWS, out, inn, fam, bool(om), bool(ro), bool(nm), bool(ac), seed=cfg * 100 + 50 + j)
        check_fwd_launch(info_of(_lib.GEMM_DX, "tc"), "tc", PROD_ROWS, inn, r["epi"], "dx")
        check(r["dx"], r["ref"], r["bnd"], "tc", fam, "cfg%d dX %d <- %d" % (cfg, inn, out))
        del r
    r = run_dw(PROD_ROWS, inn, out, fam, dwmask, seed=cfg * 100 + 90)
    info = info_of(_lib.GEMM_DW, "tc")
    assert info["nc"] == dw_nc(out) and info["v_per_split"] // 32 >= 3 * info["stages"], info
    check(r["dw"], r["ref"], r["bnd"], "tc", fam, "cfg%d dW %d x %d" % (cfg, out, inn))


# ------------------------------------------------------------------------------ layout: row blocks, parts ---
def test_row_blocks_equal_one_call():
    """The host runs the GEMMs in row blocks (model.cc PushPipe): X + r0 * ldX, rowEnd + r0, colLeft = rowEnd[r0 - 1],
    mask + r0 * ldMask, and dX with parts = ONLY_DX, dW separately with ONLY_DW.  A row's MMA sequence does not depend
    on where in a 128-row tile it sits, so the blocks must reproduce the single call bit for bit."""
    rows, k, n = 50011, 602, 64
    cuts = (0, 1000, 33333, rows)          # block starts that are not multiples of 128
    f = run_fwd(rows, k, n, "random_sign", relu=False, norm=True, masked=True, seed=5)
    y = out_buf(rows, n)
    for r0, r1 in zip(cuts[:-1], cuts[1:]):
        cl = f["col_left"] if r0 == 0 else int(f["row_end"][r0 - 1])
        K.linear_fwd_dropout(f["x"][r0:r1], f["w"], f["mask"][r0:r1], f["rate"], norm_row_end=f["row_end"][r0:r1],
                             col_left=cl, out=y[r0:r1])
    assert torch.equal(y, f["y"]), "forward in row blocks"
    check_pads(y)
    # dX of the second layer (41 -> 64 back) with the fused dropout / relu / norm backward, then dW
    d = run_dx(rows, 41, n, "random_sign", True, True, True, False, seed=6, parts=0)     # dX and dW in one call
    dx = out_buf(rows, n)
    for r0, r1 in zip(cuts[:-1], cuts[1:]):
        cl = d["col_left"] if r0 == 0 else int(d["row_end"][r0 - 1])
        K.linear_bwd_fused(d["x"][r0:r1], d["w"], None, d["dy"][r0:r1], torch.zeros_like(d["dw"]), dx[r0:r1],
                           mask=d["mask"][r0:r1], rate=d["rate"], relu_of=d["relu_of"][r0:r1],
                           norm_row_end=d["row_end"][r0:r1], col_left=cl, parts=_lib.LINEAR_BWD_ONLY_DX)
    assert torch.equal(dx, d["dx"]), "dX in row blocks"
    check_pads(dx)
    dw = torch.zeros_like(d["dw"])
    K.linear_bwd_fused(d["x"], d["w"], None, d["dy"], dw, None, mask=d["mask"], rate=d["rate"],
                       parts=_lib.LINEAR_BWD_ONLY_DW)
    assert torch.equal(dw, d["dw"]), "dW alone vs dW of the combined call"


# ------------------------------------------------------------------------------------- non-finite inputs ---
def test_non_finite_inputs_poison_whole_rows_and_columns():
    """3xTF32 quirk: hi(inf) = inf and lo = inf - inf = NaN, so a non-finite element of X turns its whole output row
    NaN (fp32 sgemm would give +-inf in some columns), also for a NaN whose payload lies only in the 13 bits the TF32
    truncation drops (0x7F800001: hi = inf, lo = NaN).  A non-finite weight turns its whole output column NaN, even in
    rows whose X is 0 there (0 * NaN).  An element the dropout mask drops is replaced by 0 before the split and has no
    effect."""
    rows, k, n = 1000, 100, 48
    g = gen(77)
    x0 = torch.randn((rows, k), generator=g, device=DEV)
    w0 = torch.randn((n, k), generator=g, device=DEV)
    rate = 0.5
    mask = K.dropout_mask(rows, k, 0, rate, 99, 1, DEV)
    keep = unpack(mask, k)
    kept = [(int(r), int(keep[r].nonzero()[0])) for r in (3, 400)]
    dropped_r = 555
    dropped_c = int((~keep[dropped_r]).nonzero()[0])
    x = x0.clone()
    for (r, c), v in zip(kept, (math.inf, -math.inf)):
        x[r, c] = v
    x[dropped_r, dropped_c] = math.inf
    w = w0.clone()
    w[17, 5] = -math.inf
    xp, x0p = padded_with_nan(x), padded_with_nan(x0)
    y = K.linear_fwd_dropout(xp, w, mask, rate, out=out_buf(rows, n))
    assert _lib.last_gemm_info(_lib.GEMM_FWD)["path"] == 1
    w_ok = w0.clone()
    y0 = K.linear_fwd_dropout(x0p, w_ok, mask, rate, out=out_buf(rows, n))
    bad_rows = [r for r, _ in kept]
    for r in bad_rows:
        assert bool(torch.isnan(y[r]).all()), "row %d not all NaN" % r
    assert bool(torch.isnan(y[:, 17]).all()), "column 17 not all NaN"
    good_r = torch.ones(rows, dtype=torch.bool, device=DEV)
    good_r[bad_rows] = False
    good_c = torch.ones(n, dtype=torch.bool, device=DEV)
    good_c[17] = False
    assert torch.equal(y[good_r][:, good_c], y0[good_r][:, good_c]), "finite elements changed"
    assert bool(torch.isfinite(y[dropped_r, good_c]).all()), "a dropped inf leaked into its row"
    # a NaN with its payload only in the 13 low mantissa bits: hi = inf, lo = NaN.  Its bits are written through an
    # integer view (a round trip through a Python float would quiet it), and the call has no dropout, whose scaling
    # would quiet it too.
    xq = padded_with_nan(x0)
    xq.view(torch.int32)[999, 7] = 0x7F800001
    assert int(xq.view(torch.int32)[999, 7]) == 0x7F800001
    yq = K.linear_fwd(xq, w0, out=out_buf(rows, n))
    assert _lib.last_gemm_info(_lib.GEMM_FWD)["path"] == 1
    y0q = K.linear_fwd(x0p, w0, out=out_buf(rows, n))
    assert bool(torch.isnan(yq[999]).all()), "the low-payload NaN did not turn its row NaN"
    others = torch.arange(rows, device=DEV) != 999
    assert torch.equal(yq[others], y0q[others])


# ---------------------------------------------------------------------------------- config 2 at full size ---
def test_config2_full_size_forward_and_dw():
    """4 194 304 x 602 -> 64 with the fused dropout mask and norm epilogue, then dW: X alone is 10 GB and has more
    than 2^31 elements.  Y is compared on a seeded sample of rows, dW in full (its fp64 reference in row chunks)."""
    rows, k, n, rate = 1 << 22, 602, 64, 0.5
    free, _ = torch.cuda.mem_get_info()
    if free < 24 * (1 << 30):
        pytest.skip("needs 24 GB of free GPU memory, %.1f GB free" % (free / (1 << 30)))
    torch.cuda.reset_peak_memory_stats()
    g = gen(2022)
    x = buf(rows, k, float("nan"))
    for r0 in range(0, rows, 1 << 20):
        x[r0:r0 + (1 << 20)] = torch.randn((min(1 << 20, rows - r0), k), generator=g, device=DEV)
    assert x.shape[0] * x.stride(0) > 2 ** 31
    w = torch.randn((n, k), generator=g, device=DEV) * 0.05
    mask = K.dropout_mask(rows, k, 0, rate, (2 << 32) | 2, 1, DEV)
    row_end, col_left = degrees(rows, g)
    y = out_buf(rows, n)
    K.linear_fwd_dropout(x, w, mask, rate, norm_row_end=row_end, col_left=col_left, out=y)
    info = info_of(_lib.GEMM_FWD, "tc")
    assert info["nc"] == 2 and info["epi"] == EPI_NORM and -(-rows // 128) >= 3 * info["grid_x"], info
    sample = torch.cat([torch.randperm(rows, generator=g, device=DEV)[:20000],
                        torch.tensor([0, rows - 1], device=DEV)])
    ref, bnd = tb.reference(apply_mask(x[sample], mask[sample], rate), w)
    ref, bnd = compose(ref, bnd, div=row_divisor(row_end, col_left)[sample])
    check(y[sample], ref, bnd, "tc", "random_sign", "full-size forward")
    assert bool((pads(y)[sample] == SENTINEL).all()), "a pad column of Y was written"
    dy = padded_with_nan(torch.randn((rows, n), generator=g, device=DEV))
    dw = torch.zeros((n, k), device=DEV)
    K.linear_bwd_fused(x, w, None, dy, dw, None, mask=mask, rate=rate, parts=_lib.LINEAR_BWD_ONLY_DW)
    info = info_of(_lib.GEMM_DW, "tc")
    assert info["nc"] == 2 and info["v_per_split"] // 32 >= 3 * info["stages"], info
    del y
    acc = tb.RefAccumulator(split=info["v_per_split"])
    for r0 in range(0, rows, 1 << 18):
        acc.add(dy[r0:r0 + (1 << 18)].T, apply_mask(x[r0:r0 + (1 << 18)], mask[r0:r0 + (1 << 18)], rate).T)
    ref, bnd = compose(*acc.result())
    check(dw, ref, bnd, "tc", "random_sign", "full-size dW")
    torch.cuda.synchronize()
    print("\nfull-size test: peak GPU memory %.2f GB" % (torch.cuda.max_memory_allocated() / 1e9))


# ------------------------------------------------------------------------------------------------ coverage ---
def test_matrix_covered():
    """Every forward / dX instantiation (3 NC x 5 epilogues), every dW instantiation, and the pipeline regimes the
    matrix targets were reached on the tensor cores.  Prints the worst error-to-bound ratios per family."""
    wanted = {(_id(c), "tc") for c in MATRIX} | {(_dw_id(c), "tc") for c in DW_MATRIX}
    if not wanted <= RAN:
        pytest.skip("%d of the %d tensor-core matrix cases did not run in this process" % (len(wanted - RAN),
                                                                                           len(wanted)))
    for key in sorted(WORST):
        print("worst |error| / bound  %-5s %-12s %.4f" % (key[0], key[1], WORST[key]))
    fwd_dx = {(nc, e) for kind, nc, e in SEEN if kind in ("fwd", "dx")}
    assert fwd_dx == {(nc, e) for nc in (1, 2, 4) for e in INSTANCES + (-1,)}, sorted(fwd_dx)
    for kind in ("dw", "dw_ring_wrap", "dw_empty_split"):
        assert {nc for kd, nc, _ in SEEN if kd == kind} == {1, 2, 4, 8}, (kind, sorted(SEEN))
    multitile = {(nc, ny) for kd, nc, ny in SEEN if kd == "multitile"}
    assert multitile >= {(1, 1), (2, 1), (4, 1), (4, 2), (4, 5)}, sorted(multitile)
