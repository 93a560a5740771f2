"""The warp-specialised dW kernel (k_tc_linear_dw_ws, outDim <= 128) against the CTA-synchronised one
(k_tc_linear_dw, ROC_B200_DW=sync), bit for bit.

Both kernels promise the same per-element MMA order, so dW must match to the last bit at every shape the new kernel
takes: outDim 16 / 41 / 64 / 100 / 128 (NC = 1, 2, 2, 4, 4), inDim 64 (its 64-column tile with one consumer warpgroup),
100 and 602 (128-column tiles), with and without the fused dropout mask whose words it loads by TMA.  The rows wrap
each split's ring at least three times and end in a partial k-block, or leave the trailing splits empty.  X and dY
carry NaN in the row padding past inDim / outDim, and the mask has every bit past inDim set.  Both kernels keep those
out of dW only because their X and dY tensor maps end at inDim / outDim and TMA zero-fills the rest (a zero stays
zero under any mask bit), so these inputs catch a tensor map, box or tile that reaches past the data; at inDim 100
a thread's two columns straddle inDim.  roc_last_gemm_info's `epi` says which kernel ran (1 warp-specialised,
0 synchronised).  A mask whose base is not 16-byte aligned cannot be loaded by TMA (its row stride is a multiple of 4
words, which the C ABI requires): it must fall back to the synchronised kernel with the same bits."""
import importlib.util
import os

import pytest
import torch

from roc_b200 import _lib
from roc_b200 import kernels as K

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_dw", os.path.join(HERE, "golden", "make_golden_dw.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)


def nan_padded(src):
    """src [rows][cols] copied into a row-padded buffer whose padding (at least 4 floats per row) is NaN"""
    rows, cols = src.shape
    buf = torch.full((rows, (cols + 3) // 4 * 4 + 4), float("nan"), device=src.device)
    buf[:, :cols] = src
    return buf[:, :cols]


def run(rows, inn, out, masked, kernel, mask_layout="dense"):
    """dW = dY^T dropout(X) from zero through `kernel` ("ws" or "sync"); returns (dW, roc_last_gemm_info).
    mask_layout "offset" passes the mask from a base 4 bytes past an aligned one."""
    x = nan_padded(G.hashed(rows, inn, 1))
    dy = nan_padded(G.hashed(rows, out, 2))
    mask = None
    if masked:
        mask = K.dropout_mask(rows, inn, 0, 0.5, 7, 1)
        past = torch.arange(mask.shape[1] * 32, device="cuda").view(-1, 32) >= inn   # bits of columns >= inDim
        bits = (past.to(torch.int64) << torch.arange(32, device="cuda")).sum(1).to(torch.int64)
        bits = torch.where(bits >= 1 << 31, bits - (1 << 32), bits).to(torch.int32)
        mask |= bits[None, :]
        if mask_layout == "offset":
            flat = torch.zeros(rows * mask.shape[1] + 4, dtype=torch.int32, device="cuda")
            view = flat[1:1 + mask.numel()].view(mask.shape)
            view.copy_(mask)
            mask = view
    w = torch.zeros((out, inn), device="cuda")
    dw = torch.zeros((out, inn), device="cuda")
    old = os.environ.pop("ROC_B200_DW", None)
    try:
        if kernel == "sync":
            os.environ["ROC_B200_DW"] = "sync"
        K.linear_bwd_fused(x, w, None, dy, dw, None, mask=mask, rate=0.5 if masked else 0.0,
                           parts=_lib.LINEAR_BWD_ONLY_DW)
        info = _lib.last_gemm_info(_lib.GEMM_DW)
    finally:
        os.environ.pop("ROC_B200_DW", None)
        if old is not None:
            os.environ["ROC_B200_DW"] = old
    torch.cuda.synchronize()
    return dw, info


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


CASES = [(kind, inn, out, masked) for kind in ("ring", "empty") for inn in (64, 100, 602)
         for out in (16, 41, 64, 100, 128) for masked in (False, True)]


@pytest.mark.parametrize("kind,inn,out,masked", CASES)
def test_dw_ws_matches_sync_bitwise(kind, inn, out, masked):
    rows = G.ring_rows(inn, sms()) if kind == "ring" else G.EMPTY_ROWS
    got, info = run(rows, inn, out, masked, "ws")
    want, info_sync = run(rows, inn, out, masked, "sync")
    assert info["path"] == 1 and info["epi"] == 1, info
    assert info_sync["path"] == 1 and info_sync["epi"] == 0, info_sync
    assert info["nc"] == {16: 1, 41: 2, 64: 2, 100: 4, 128: 4}[out], info
    assert info["grid_y"] == -(-inn // 128) and info["stages"] <= 4, info
    for k in ("splits", "v_per_split", "grid_x", "grid_y", "nc"):
        assert info[k] == info_sync[k], (k, info, info_sync)
    assert rows % 32, rows
    if kind == "ring":
        assert info["v_per_split"] // 32 >= 3 * info["stages"], info
    else:
        assert (info["splits"] - 1) * info["v_per_split"] >= rows, info
    assert torch.isfinite(got).all()
    assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (
        "dW differs from ROC_B200_DW=sync by up to %.3e" % (got - want).abs().max().item())


@pytest.mark.parametrize("out", [129, 200])
def test_dw_wide_output_runs_sync_kernel(out):
    _, info = run(G.EMPTY_ROWS, 100, out, True, "ws")
    assert info["path"] == 1 and info["epi"] == 0 and info["nc"] == 8, info


def test_dw_unaligned_mask_falls_back_to_sync_kernel():
    rows, inn, out = G.ring_rows(602, sms()), 602, 64
    got, info = run(rows, inn, out, True, "ws", mask_layout="offset")
    want, _ = run(rows, inn, out, True, "ws")
    assert info["path"] == 1 and info["epi"] == 0 and info["nc"] == 2, info
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
