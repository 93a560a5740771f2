"""bf16 storage of node features, on the host: the rounding roc_f32_to_bf16 does on the device, and the row pitch
the kernels expect.  numpy only, so it runs without a GPU.

A bf16 tensor is held as its raw bits (uint16): the top half of the fp32 word, rounded to nearest even.  Widening back
to fp32 is exact.
"""
import numpy as np


def row_pitch(h):
    """elements per row of a bf16 node tensor of width h: rows of whole 16-byte units, as TMA loads them"""
    return (int(h) + 7) // 8 * 8


def to_bits(a):
    """fp32 -> bf16 bits (uint16 array of a's shape), round to nearest even; NaN -> 0x7FC0, overflow -> +-inf.
    The same bits as roc_f32_to_bf16, and as torch's Tensor.to(torch.bfloat16) except that torch's NaN bits vary."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(np.asarray(a, dtype=np.float32)), np.uint16(0x7FC0), r)


def widen(bits):
    """bf16 bits -> fp32, exactly"""
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def round_f32(a):
    """a rounded to bf16 and widened back: the fp32 values a bf16 tensor of a holds"""
    return widen(to_bits(a))
