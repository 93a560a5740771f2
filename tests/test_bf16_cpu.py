"""CPU suite: the host side of bf16 input features.  The rounding helper of roc_b200.bf16 against torch's CPU
conversion, the row pitch, and the exactness argument the bf16 Linear kernels rest on: a widened bf16 value splits
into a TF32 head equal to itself and a zero remainder."""
import ctypes as C

import numpy as np
import torch

import tf32_bound as tb
from roc_b200 import _lib, bf16


def crafted():
    pats = [0x00000000, 0x80000000, 0x3F808000, 0x3F818000, 0x3F808001, 0x3F807FFF, 0x00000001, 0x00008000,
            0x00018000, 0x807FFFFF, 0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000,
            0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FFFFFFF, 0xFF800001]
    rnd = np.random.RandomState(1).randint(0, 2 ** 32, size=100000, dtype=np.uint64).astype(np.uint32)
    return np.concatenate([np.array(pats, dtype=np.uint32), rnd]).view(np.float32)


def test_rounding_helper_matches_torch():
    x = crafted()
    want = torch.from_numpy(x.copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    got = bf16.to_bits(x)
    nan = np.isnan(x)
    assert np.array_equal(got[~nan], want[~nan])
    # a NaN stays a NaN; which one torch writes depends on its code path, the helper always writes 0x7FC0
    assert np.isnan(bf16.widen(want[nan])).all() and (got[nan] == 0x7FC0).all()


def test_rounding_cases():
    b = bf16.to_bits(np.array([0x3F808000, 0x3F818000, 0x7F7F8000, 0x7F800001, 0x00008000],
                              dtype=np.uint32).view(np.float32))
    assert list(b) == [0x3F80, 0x3F82, 0x7F80, 0x7FC0, 0x0000]   # ties to even, overflow to inf, NaN, subnormal tie


def test_widen_is_exact_and_round_trips():
    allbits = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    w = bf16.widen(allbits)
    assert np.array_equal(w.view(np.uint32) >> 16, allbits.astype(np.uint32))
    finite = ~np.isnan(w)
    assert np.array_equal(bf16.to_bits(w)[finite], allbits[finite])


def test_widened_bf16_has_a_zero_tf32_remainder():
    """the reason the bf16 kernels compute exactly what the fp32 kernels compute on X.float(): 3xTF32's lo part of a
    widened bf16 value is zero, so the split loses nothing and adds nothing"""
    w = bf16.widen(np.arange(1 << 16, dtype=np.uint32).astype(np.uint16))
    w = w[np.isfinite(w)]
    hi, lo = tb.split(w)
    assert np.array_equal(hi.view(np.uint32), w.view(np.uint32))
    assert not lo.any()


def test_row_pitch():
    assert [bf16.row_pitch(h) for h in (1, 8, 9, 41, 602, 64)] == [8, 8, 16, 48, 608, 64]


def test_bf16_entry_points_refuse_bad_arguments_without_touching_memory():
    """argument checks run before any device work (NULL pointers, leading dimensions too small, a rate without a
    mask): each returns ROC_ERR_INVALID"""
    lib = _lib.lib
    p = C.c_void_p(16)
    assert lib.roc_f32_to_bf16(4, 8, None, 8, p, 8, None) == _lib.ROC_ERR_INVALID
    assert lib.roc_f32_to_bf16(4, 8, p, 8, p, 7, None) == _lib.ROC_ERR_INVALID
    assert lib.roc_bf16_to_f32(4, 8, p, 7, p, 8, None) == _lib.ROC_ERR_INVALID
    assert lib.roc_dropout_fwd_bf16(4, 8, 0, 1.0, 1, 0, p, 8, p, 8, None) == _lib.ROC_ERR_INVALID
    assert lib.roc_linear_fwd_bf16(4, 8, 4, p, 8, p, p, 4, 0, 0, None, 0, None, 0, 0.5, None) == _lib.ROC_ERR_INVALID
    assert lib.roc_linear_fwd_bf16(4, 8, 4, p, 7, p, p, 4, 0, 0, None, 0, None, 0, 0.0, None) == _lib.ROC_ERR_INVALID
    assert lib.roc_linear_dw_bf16(4, 8, 4, p, 8, None, 0, p, 4, p, 0, None, 0, None, 0, 0.0,
                                  None) == _lib.ROC_ERR_INVALID
