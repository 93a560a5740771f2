"""GPU suite: bf16 input features.  The Linear forward and dW on a bf16 X, the fp32 <-> bf16 conversions and the bf16
dropout forward, each against the fp32 entry point on the widened X.

A bf16 value has 8 significant bits, so it widens to fp32 exactly and its TF32 split is (hi = x, lo = 0).  The
kernels widen each X element as they read it and then run the fp32 arithmetic unchanged, so every result must be
byte-identical to the fp32 kernel's on X.float(): the same path (tensor cores or SIMT), the same instantiation and the
same dW split-K layout.  roc_last_gemm_info shows both calls took the same kernel and that each case reached the
regime it was chosen for.  A subset is also held to fp64 of the widened inputs with the bound of tests/tf32_bound.py,
in case both paths were wrong the same way.

test_config2_full_size (4 194 304 x 602 -> 64, fp32 and bf16 copies of X together about 15 GB) skips when the GPU has
too little free memory."""
import numpy as np
import pytest
import torch

import tf32_bound as tb
from roc_b200 import _lib, bf16
from roc_b200 import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
BIG_ROWS = 3 * 132 * 128 + 77          # >= 3 row tiles per CTA of the persistent forward on a 132-SM H100


def gen(seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return g


def bits(t):
    """the bytes of an fp32 [rows][h] view, as int32"""
    return t.contiguous().view(torch.int32)


def features(rows, k, seed):
    """(bf16 X, fp32 X.float()) in the node-tensor layouts: bf16 rows of round_up(k, 8), fp32 rows of round_up(k, 4)"""
    x32 = torch.randn((rows, k), generator=gen(seed), device=DEV) * 3.0
    xb = K.f32_to_bf16(x32)
    xw = K.bf16_to_f32(xb)
    assert xb.stride(0) == bf16.row_pitch(k)
    return xb, xw


def degrees(rows, g, col_left=1000):
    deg = torch.randint(1, 41, (rows,), generator=g, device=DEV)
    deg[::997] = 70000
    return col_left + torch.cumsum(deg, 0), col_left


def mask_of(rows, k, rate, seed):
    return K.dropout_mask(rows, k, seed, rate, (11 << 32) | seed, 2, DEV) if rate else None


def same_launch(a, b):
    keys = ("path", "nc", "epi", "grid_x", "grid_y", "stages", "splits", "v_per_split", "w_resident", "epi_bufs")
    return {k: a[k] for k in keys} == {k: b[k] for k in keys}


# --------------------------------------------------------------------------------------------------- forward ---
# (rows, inDim, outDim, rate, relu, norm, expected W residency on the tensor cores)
FWD = [
    (1000, 41, 20, 0.0, False, False, 1),          # NC 1, W resident, partial last tile
    (BIG_ROWS, 64, 32, 0.5, False, True, 1),       # NC 1, persistent loop, norm epilogue
    (129, 100, 64, 0.3, True, False, 1),           # NC 2, relu (generic epilogue)
    (BIG_ROWS, 602, 64, 0.5, False, True, 0),      # NC 2, W streamed: config 2's layer 1
    (5000, 602, 64, 0.0, True, True, 0),           # NC 2, streamed, relu + norm
    (777, 64, 100, 0.3, False, False, 1),          # NC 4, resident
    (777, 200, 100, 0.3, False, False, 0),         # NC 4, streamed
    (BIG_ROWS, 602, 128, 0.5, False, True, 0),     # NC 4, streamed: config 4's layer 1
    (300, 602, 256, 0.0, False, False, 0),         # two N tiles of 128
    (1, 13, 41, 0.5, False, False, 1),             # one row, ragged k
]


def _fwd_id(c):
    rows, k, n, rate, relu, norm, _ = c
    return "r%d-k%d-n%d-rate%g%s%s" % (rows, k, n, rate, "-relu" if relu else "", "-norm" if norm else "")


def run_fwd_pair(rows, k, n, rate, relu, norm, seed):
    g = gen(seed)
    xb, xw = features(rows, k, seed)
    w = torch.randn((n, k), generator=g, device=DEV)
    mask = mask_of(rows, k, rate, seed)
    row_end, col_left = degrees(rows, g) if norm else (None, 0)
    y32 = K.linear_fwd_dropout(xw, w, mask, rate, activation=int(relu), norm_row_end=row_end, col_left=col_left)
    i32 = _lib.last_gemm_info(_lib.GEMM_FWD)
    yb = K.linear_fwd_bf16(xb, w, mask, rate, activation=int(relu), norm_row_end=row_end, col_left=col_left)
    ib = _lib.last_gemm_info(_lib.GEMM_FWD)
    return dict(xw=xw, w=w, mask=mask, row_end=row_end, col_left=col_left, y32=y32, yb=yb, i32=i32, ib=ib)


@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("case", FWD, ids=_fwd_id)
def test_forward_matches_fp32_bit_for_bit(case, path, monkeypatch):
    if path == "simt":
        monkeypatch.setenv("ROC_B200_GEMM", "simt")
    rows, k, n, rate, relu, norm, wres = case
    r = run_fwd_pair(rows, k, n, rate, relu, norm, seed=rows + k + n)
    ib = r["ib"]
    assert ib["path"] == (1 if path == "tc" else 2), ib
    assert same_launch(ib, r["i32"]) or path == "tc", (ib, r["i32"])
    if path == "tc":
        assert ib["nc"] == (1 if n <= 32 else 2 if n <= 64 else 4), ib
        assert ib["w_resident"] == wres, ib
        # the bf16 ring is as deep as the fp32 one or deeper (half-size A stages), never past 12
        assert r["i32"]["stages"] <= ib["stages"] <= 12, (ib, r["i32"])
        assert ib["epi"] == (-1 if relu else 8 if norm else 0), ib
        if rows == BIG_ROWS:
            assert -(-rows // 128) >= 3 * ib["grid_x"], ib
    assert torch.equal(bits(r["yb"]), bits(r["y32"])), "bf16 forward differs from fp32 on X.float()"


def test_bf16_ring_is_deeper_where_it_fits():
    """with W resident the bf16 ring holds 8 KB stages: more of them than fp32's 16 KB ones"""
    r = run_fwd_pair(BIG_ROWS, 64, 32, 0.0, False, False, seed=5)
    assert r["ib"]["w_resident"] == r["i32"]["w_resident"] == 1
    assert r["ib"]["stages"] > r["i32"]["stages"], (r["ib"], r["i32"])


def test_unaligned_pitch_takes_simt(monkeypatch):
    """a bf16 X whose rows are not whole 16-byte units is refused by TMA: the SIMT kernel serves it, with the bits of
    the fp32 SIMT kernel on X.float()"""
    xb, xw = features(300, 41, 3)
    xb2 = torch.zeros((300, 44), device=DEV, dtype=torch.bfloat16)[:, :41]
    xb2.copy_(xb)
    w = torch.randn((20, 41), generator=gen(3), device=DEV)
    yb = K.linear_fwd_bf16(xb2, w)
    assert _lib.last_gemm_info(_lib.GEMM_FWD)["path"] == 2
    monkeypatch.setenv("ROC_B200_GEMM", "simt")
    y32 = K.linear_fwd_dropout(xw, w, None, 0.0)
    assert torch.equal(bits(yb), bits(y32))


# ------------------------------------------------------------------------------------------------------- dW ---
# (rows, inDim, outDim, rate, kernel: "ws" / "sync", relu)
DW = [
    (4000, 41, 20, 0.5, "ws", False),      # inDim <= 64: one consumer warpgroup
    (300, 64, 64, 0.0, "ws", True),        # few rows: 5 splits; relu backward of dY
    (54000, 602, 64, 0.5, "ws", False),    # config 2's dW shape: 5 M tiles, 26 splits
    (20000, 100, 128, 0.3, "ws", False),
    (20000, 100, 128, 0.3, "sync", False), # ROC_B200_DW=sync
    (9000, 200, 200, 0.5, "sync", False),  # outDim > 128: the synchronised kernel
    (777, 602, 256, 0.0, "sync", True),
]


def _dw_id(c):
    rows, inn, out, rate, kern, relu = c
    return "r%d-in%d-out%d-rate%g-%s%s" % (rows, inn, out, rate, kern, "-relu" if relu else "")


def run_dw_pair(rows, inn, out, rate, relu, seed):
    g = gen(seed)
    xb, xw = features(rows, inn, seed)
    dy = torch.randn((rows, out), generator=g, device=DEV)
    y = torch.randn((rows, out), generator=g, device=DEV) if relu else None
    w = torch.zeros((out, inn), device=DEV)
    dw0 = torch.randn((out, inn), generator=g, device=DEV)
    mask = mask_of(rows, inn, rate, seed)
    dy32, dw32 = dy.clone(), dw0.clone()
    K.linear_bwd_dropout(xw, w, y, dy32, dw32, mask, rate, activation=int(relu))
    i32 = _lib.last_gemm_info(_lib.GEMM_DW)
    dyb, dwb = dy.clone(), dw0.clone()
    K.linear_dw_bf16(xb, dyb, dwb, mask, rate, y=y, activation=int(relu))
    ib = _lib.last_gemm_info(_lib.GEMM_DW)
    return dict(xw=xw, dy=dy, dy32=dy32, dyb=dyb, dw0=dw0, dw32=dw32, dwb=dwb, mask=mask, i32=i32, ib=ib)


@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("case", DW, ids=_dw_id)
def test_dw_matches_fp32_bit_for_bit(case, path, monkeypatch):
    rows, inn, out, rate, kern, relu = case
    if path == "simt":
        monkeypatch.setenv("ROC_B200_GEMM", "simt")
    if kern == "sync":
        monkeypatch.setenv("ROC_B200_DW", "sync")
    r = run_dw_pair(rows, inn, out, rate, relu, seed=rows + inn + out)
    ib, i32 = r["ib"], r["i32"]
    assert ib["path"] == (1 if path == "tc" else 2), ib
    assert (ib["splits"], ib["v_per_split"]) == (i32["splits"], i32["v_per_split"]), (ib, i32)
    if path == "tc":
        assert ib["epi"] == i32["epi"] == (1 if kern == "ws" else 0), (ib, i32)
        assert ib["nc"] == i32["nc"] and ib["grid_y"] == -(-inn // 128), ib
    if relu:
        assert torch.equal(bits(r["dyb"]), bits(r["dy32"]))
    assert torch.equal(bits(r["dwb"]), bits(r["dw32"])), "bf16 dW differs from fp32 on X.float()"


def test_dw_kernels_agree_with_bf16_x(monkeypatch):
    """the warp-specialised and the synchronised dW kernels give the same bits on a bf16 X too"""
    xb, _ = features(20000, 100, 21)
    dy = torch.randn((20000, 96), generator=gen(21), device=DEV)
    mask = mask_of(20000, 100, 0.5, 21)
    a = K.linear_dw_bf16(xb, dy, torch.zeros((96, 100), device=DEV), mask, 0.5)
    assert _lib.last_gemm_info(_lib.GEMM_DW)["epi"] == 1
    monkeypatch.setenv("ROC_B200_DW", "sync")
    b = K.linear_dw_bf16(xb, dy, torch.zeros((96, 100), device=DEV), mask, 0.5)
    assert _lib.last_gemm_info(_lib.GEMM_DW)["epi"] == 0
    assert torch.equal(bits(a), bits(b))


# ------------------------------------------------------------------------------------------------ fp64 bound ---
@pytest.mark.parametrize("k,n,rate", [(602, 64, 0.5), (100, 128, 0.0), (41, 20, 0.3)])
def test_forward_within_fp64_bound(k, n, rate):
    rows = 20000
    xb, xw = features(rows, k, 40 + k)
    w = torch.randn((n, k), generator=gen(k), device=DEV)
    mask = mask_of(rows, k, rate, 40 + k)
    y = K.linear_fwd_bf16(xb, w, mask, rate)
    assert _lib.last_gemm_info(_lib.GEMM_FWD)["path"] == 1
    xd = xw
    if mask is not None:
        cols = torch.arange(k, device=DEV)
        keep = ((mask[:, cols >> 5] >> (cols & 31)) & 1).bool()
        scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(rate)))
        xd = torch.where(keep, xw * scale, torch.zeros((), device=DEV))
    ref, bnd = tb.reference(xd, w)
    r = tb.worst_ratio(y, ref, bnd)
    assert r <= 1.0, r


def test_dw_within_fp64_bound():
    rows, inn, out = 132 // 1 * 416 - 5, 64, 64       # splits of <= 416 rows, the length the bound is calibrated for
    xb, xw = features(rows, inn, 50)
    dy = torch.randn((rows, out), generator=gen(50), device=DEV)
    dw = K.linear_dw_bf16(xb, dy, torch.zeros((out, inn), device=DEV))
    info = _lib.last_gemm_info(_lib.GEMM_DW)
    assert info["path"] == 1 and info["v_per_split"] <= 416, info
    acc = tb.RefAccumulator(split=info["v_per_split"])
    acc.add(dy.T, xw.T)
    ref, bnd = acc.result()
    r = tb.worst_ratio(dw, ref, bnd)
    assert r <= 1.0, r


# ------------------------------------------------------------------------------------------------- full size ---
def test_config2_full_size():
    """config 2's first layer at full size: 4 194 304 x 602 -> 64, masked, forward and dW byte-identical"""
    rows, k, n = 4194304, 602, 64
    free, _ = torch.cuda.mem_get_info()
    if free < 18 * 2 ** 30:
        pytest.skip("needs about 18 GB of free GPU memory")
    g = gen(77)
    xb = K.bf16_padded(rows, k)
    xw = K.padded(rows, k)
    step = 1 << 18
    for r0 in range(0, rows, step):      # fill chunk by chunk: no full-size temporary
        chunk = torch.randn((min(step, rows - r0), k), generator=g, device=DEV)
        K.f32_to_bf16(chunk, out=xb[r0:r0 + step])
        K.bf16_to_f32(xb[r0:r0 + step], out=xw[r0:r0 + step])
    del chunk
    w = torch.randn((n, k), generator=g, device=DEV)
    mask = mask_of(rows, k, 0.5, 77)
    y32 = K.linear_fwd_dropout(xw, w, mask, 0.5)
    yb = K.linear_fwd_bf16(xb, w, mask, 0.5)
    assert _lib.last_gemm_info(_lib.GEMM_FWD)["path"] == 1
    assert torch.equal(bits(yb), bits(y32))
    del y32, yb
    dy = torch.randn((rows, n), generator=g, device=DEV)
    dw32 = torch.zeros((n, k), device=DEV)
    K.linear_bwd_dropout(xw, w, None, dy, dw32, mask, 0.5)
    dwb = K.linear_dw_bf16(xb, dy, torch.zeros((n, k), device=DEV), mask, 0.5)
    assert _lib.last_gemm_info(_lib.GEMM_DW)["path"] == 1
    assert torch.equal(bits(dwb), bits(dw32))


# ------------------------------------------------------------------------------------------------ conversion ---
def crafted_f32_bits():
    """fp32 bit patterns that exercise every rounding case, plus random ones"""
    pats = [0x00000000, 0x80000000, 0x3F800000, 0xBF800000,
            0x3F808000, 0x3F818000, 0x3F808001, 0x3F807FFF,      # ties to even (down, up), just above / below a tie
            0x00000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x80000001, 0x807FFFFF,   # subnormals, ties among them
            0x00800000, 0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0xFF7FFFFF,              # overflow to inf at the top
            0x7F800000, 0xFF800000,                                                # +-inf
            0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FFFFFFF, 0xFF800001, 0x7FBF8000]  # NaNs, quiet and signalling
    rnd = np.random.RandomState(0).randint(0, 2 ** 32, size=4000, dtype=np.uint64).astype(np.uint32)
    return np.concatenate([np.array(pats, dtype=np.uint32), rnd])


@pytest.mark.parametrize("h", [13, 64])
def test_conversion_rounds_to_nearest_even(h):
    p = crafted_f32_bits()
    p = np.resize(p, (len(p) + h - 1) // h * h).reshape(-1, h)
    x = torch.from_numpy(p.view(np.float32).copy())
    want = x.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    nan = np.isnan(p.view(np.float32))
    assert np.isnan(bf16.widen(want[nan])).all()
    want[nan] = 0x7FC0                       # torch keeps NaN a NaN; roc_f32_to_bf16 writes the quiet NaN 0x7FC0
    assert np.array_equal(bf16.to_bits(p.view(np.float32)), want)      # the host helper agrees with torch
    xd = K.padded(p.shape[0], h, fill=x.to(DEV))
    out = torch.full((p.shape[0], bf16.row_pitch(h)), -1, device=DEV, dtype=torch.int16).view(torch.bfloat16)[:, :h]
    K.f32_to_bf16(xd, out=out)
    whole = out.as_strided((p.shape[0], out.stride(0)), (out.stride(0), 1)).view(torch.int16).cpu().numpy()
    assert np.array_equal(whole[:, :h].view(np.uint16), want)
    assert not whole[:, h:].any(), "a pad column is not zero"
    back = K.bf16_to_f32(out).cpu()
    assert torch.equal(back.view(torch.int32), torch.from_numpy(bf16.widen(want)).view(torch.int32))


@pytest.mark.parametrize("rate", [0.0, 0.3, 0.5])
def test_dropout_fwd_bf16_matches_fp32(rate):
    xb, xw = features(3001, 45, 60)
    yb = K.dropout_fwd_bf16(xb, 17, rate, 1234, 5)
    y32 = K.dropout_fwd(xw, 17, rate, 1234, 5)
    assert torch.equal(bits(yb), bits(y32))
    if rate == 0.0:
        assert torch.equal(bits(yb), bits(xw))
