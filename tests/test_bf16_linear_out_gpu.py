"""GPU suite: the Linear forward storing bf16 (ROC_LINEAR_Y_BF16).  Every stored value must be exactly roc_f32_to_bf16
of what the same call stores without the flag, on every forward instantiation of the wgmma kernel (outDim <= 32, <= 64
through the bf16 staging tile, > 64 and > 128 stored directly; no epilogue, the norm, relu, the norm with relu),
with the fused dropout and with a bf16 X, and on the SIMT kernel (ROC_B200_GEMM=simt, and an inDim the tensor cores
refuse).  The output rows hold a sentinel in their pad columns and in a guard row on each side, which must survive."""
import numpy as np
import pytest
import torch

from roc_b200 import _lib, datasets
from roc_b200 import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = 0x5A5A                                   # a bf16 sentinel (a normal number, 1.53e16)
ROWS = 1000


def guarded_bf16(rows, h):
    ld = (h + 7) // 8 * 8 + 8
    buf = torch.full((rows + 2, ld), SENT, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    return buf, buf[1:rows + 1, :h]


def norm_rows(rows):
    row_end, _ = datasets.uniform_graph(rows, 4 * rows, seed=5)
    return row_end.to(DEV)


def call(kind, x, w, out, y_bf16, relu, norm, mask, rate):
    act = _lib.AC_MODE_RELU if relu else _lib.AC_MODE_NONE
    if kind == "bf16x":
        return K.linear_fwd_bf16(x, w, mask=mask, rate=rate, activation=act, norm_row_end=norm, out=out, y_bf16=y_bf16)
    if kind == "dropout":
        return K.linear_fwd_dropout(x, w, mask, rate, activation=act, norm_row_end=norm, out=out, y_bf16=y_bf16)
    return K.linear_fwd(x, w, activation=act, norm_row_end=norm, out=out, y_bf16=y_bf16)


def check(kind, in_dim, out_dim, relu, norm, path):
    torch.manual_seed(in_dim * 1000 + out_dim)
    xf = torch.randn((ROWS, in_dim), device=DEV)
    x = K.f32_to_bf16(xf) if kind == "bf16x" else K.padded(ROWS, in_dim, fill=xf)
    w = (torch.randn((out_dim, in_dim), device=DEV) / in_dim ** 0.5).contiguous()
    mask, rate = (None, 0.0)
    if kind in ("dropout", "bf16x"):
        rate = 0.5
        mask = K.dropout_mask(ROWS, in_dim, 0, rate, 77, 1)
    re_ = norm_rows(ROWS) if norm else None
    y = call(kind, x, w, None, False, relu, re_, mask, rate)
    buf, yb = guarded_bf16(ROWS, out_dim)
    call(kind, x, w, yb, True, relu, re_, mask, rate)
    assert _lib.lib.roc_last_gemm_path(0) == path
    torch.cuda.synchronize()
    want = K.f32_to_bf16(y).view(torch.int16).cpu().numpy()
    bits = buf.view(torch.int16).cpu().numpy()
    what = "%s %dx%d relu=%d norm=%d" % (kind, in_dim, out_dim, relu, norm)
    assert np.array_equal(bits[1:ROWS + 1, :out_dim], want), what + ": bits differ from f32_to_bf16 of the fp32 store"
    keep = np.ones(bits.shape, dtype=bool)
    keep[1:ROWS + 1, :out_dim] = False
    assert (bits[keep] == SENT).all(), what + ": the padding or a guard row changed"


@pytest.mark.parametrize("kind", ["fp32x", "dropout", "bf16x"])
@pytest.mark.parametrize("out_dim", [7, 24, 41, 64, 100, 128, 200])
@pytest.mark.parametrize("relu,norm", [(False, False), (False, True), (True, False), (True, True)])
def test_y_bf16_tensor_cores(kind, out_dim, relu, norm):
    check(kind, 72, out_dim, relu, norm, 1)


@pytest.mark.parametrize("kind", ["fp32x", "dropout", "bf16x"])
@pytest.mark.parametrize("out_dim", [7, 41, 200])
@pytest.mark.parametrize("norm", [False, True])
def test_y_bf16_simt_forced(kind, out_dim, norm, monkeypatch):
    monkeypatch.setenv("ROC_B200_GEMM", "simt")
    check(kind, 72, out_dim, False, norm, 2)


@pytest.mark.parametrize("out_dim", [9, 64])
def test_y_bf16_simt_shape(out_dim):
    """inDim 6: below the tensor cores' k8 step, so the dispatcher takes the SIMT kernel."""
    check("fp32x", 6, out_dim, True, True, 2)


def test_y_bf16_refuses_ld():
    x = K.padded(16, 32, fill=torch.ones((16, 32), device=DEV))
    w = torch.ones((12, 32), device=DEV)
    out = torch.zeros((16, 12), dtype=torch.bfloat16, device=DEV)     # ld 12: not a multiple of 8
    with pytest.raises(_lib.RocError):
        K.linear_fwd(x, w, out=out, y_bf16=True)
