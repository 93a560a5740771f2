"""CPU suite: calibrates the element-wise error bound of tests/tf32_bound.py, which tests/test_linear_gpu.py holds the
Linear GEMMs to.  A numpy emulation of the kernels' arithmetic (TF32 truncation of hi and of lo, three MMAs per k8
step, each truncated into the fp32 accumulator as the H100 does) shows, on every data family the GPU tests use, that

  * correct 3xTF32 and plain fp32 GEMMs stay under a quarter of the bound, and
  * a kernel that loses any one of the three MMAs (2xTF32 either way, or 1xTF32) overshoots it at least fourfold,

so a pass on the GPU is evidence that no MMA term is missing or stale, not luck.  This holds for the forward / dX
shapes (K = the layer width, up to 602) and for dW split-K with 416 rows per split (K = the row count, thousands of
rows in 26 or 132 ranges), the split length the GPU dW matrix runs at.  Worst error-to-bound ratios of the emulation
(C_BOUND = 4), single range: 3xTF32 0.07 - 0.21 (largest at K = 8, where the split error of one product is not
averaged down), fp32 0.01 - 0.05; 2xTF32 5.0 - 195 (smallest for all-positive data at K = 602), 1xTF32 9.8 - 307.
dW split-K: 3xTF32 <= 0.09, 2xTF32 >= 5.0, 1xTF32 >= 9.9."""
import numpy as np
import pytest
import torch

import tf32_bound as tb

SHAPES = [(256, 602, 64), (129, 41, 33), (64, 13, 16), (96, 8, 40)]


def _data(family, m, k, n, seed):
    gen = torch.Generator(device="cpu")
    gen.manual_seed(seed)
    a = tb.family_data(family, m, k, gen, "a", "cpu")
    b = tb.family_data(family, n, k, gen, "b", "cpu")
    return a, b


def _ratio(a, b, mode):
    got = torch.from_numpy(tb.emulate(a.numpy(), b.numpy(), mode))
    ref, bnd = tb.reference(a, b)
    return tb.worst_ratio(got, ref, bnd)


def test_truncating_accumulation_is_what_a_k_linear_term_is_for():
    """Same-sign data at K = 602: rounding the accumulator toward zero makes an error several times that of
    round-to-nearest (what the H100 showed against a sqrt(K) model), and the bound still holds it with margin."""
    a, b = _data("positive", 256, 602, 64, seed=7)
    ref, bnd = tb.reference(a, b)
    got = torch.from_numpy(tb.emulate(a.numpy(), b.numpy(), "3xtf32"))
    err = (got.double() - ref).abs().max().item()
    assert (got.double() <= ref + 1e-30).float().mean() > 0.99      # truncation: below the exact sum
    assert err > 2 * (torch.from_numpy(tb.emulate(a.numpy(), b.numpy(), "fp32")).double() - ref).abs().max().item()
    assert tb.worst_ratio(got, ref, bnd) <= 0.25


@pytest.mark.parametrize("family", tb.FAMILIES)
@pytest.mark.parametrize("m,k,n", SHAPES)
def test_correct_arithmetic_passes_with_margin(family, m, k, n):
    a, b = _data(family, m, k, n, seed=m + k + n)
    for mode in ("3xtf32", "fp32"):
        r = _ratio(a, b, mode)
        assert r <= 0.25, "%s %s %dx%dx%d: worst error / bound %.3f" % (mode, family, m, k, n, r)


@pytest.mark.parametrize("family", tb.FAMILIES)
@pytest.mark.parametrize("m,k,n", SHAPES)
def test_a_missing_mma_fails_by_a_wide_margin(family, m, k, n):
    a, b = _data(family, m, k, n, seed=m + k + n)
    for mode in ("2xtf32_no_lo_hi", "2xtf32_no_hi_lo", "1xtf32"):
        r = _ratio(a, b, mode)
        assert r >= 4.0, "%s %s %dx%dx%d: worst error / bound only %.3f" % (mode, family, m, k, n, r)


@pytest.mark.parametrize("family", tb.FAMILIES)
@pytest.mark.parametrize("splits", [26, 132])
def test_split_k_dw_keeps_its_power(family, splits):
    """dW sums over the vertices: K is the row count, split into ranges that accumulate on their own and are then added
    in fp32 (k_tc_linear_dw, k_splitk_reduce).  At the layout of the GPU matrix's ring-wrap cases (416 rows per
    split, 26 or 132 splits, the last short) the bound must still hold a correct kernel with margin and reject a lost
    MMA.  A bound that summed |partial sums| over all rows in one sequence would be ~sqrt(splits) times too loose
    for random signs: every lost lo term would pass."""
    split = 416
    rows = splits * split - 5
    gen = torch.Generator(device="cpu")
    gen.manual_seed(splits)
    x = tb.family_data(family, rows, 40, gen, "a", "cpu")
    dy = tb.family_data(family, rows, 24, gen, "b", "cpu")
    a, b = dy.T.contiguous(), x.T.contiguous()             # dW[o][i] = sum_v dY[v][o] X[v][i]
    acc = tb.RefAccumulator(split=split)
    for r0 in range(0, rows, 4096):                        # chunked over K as the GPU tests do
        acc.add(a[:, r0:r0 + 4096], b[:, r0:r0 + 4096])
    ref, bnd = acc.result()
    assert torch.allclose(ref, a.double() @ b.double().T, rtol=1e-12, atol=1e-9)
    for mode in ("3xtf32", "fp32"):
        r = tb.worst_ratio(torch.from_numpy(tb.emulate_split_k(a.numpy(), b.numpy(), split, mode)), ref, bnd)
        assert r <= 0.25, "%s %s: worst error / bound %.3f" % (mode, family, r)
    for mode in ("2xtf32_no_lo_hi", "2xtf32_no_hi_lo", "1xtf32"):
        r = tb.worst_ratio(torch.from_numpy(tb.emulate_split_k(a.numpy(), b.numpy(), split, mode)), ref, bnd)
        assert r >= 4.0, "%s %s: worst error / bound only %.3f" % (mode, family, r)


def test_emulated_split_is_exact_and_truncating():
    """hi + lo reproduces x to within lo's own truncation, and hi keeps the top 10 mantissa bits"""
    x = np.array([1.0, 1.0 + 2.0 ** -10, 1.0 + 2.0 ** -11, -3.14159265, 2.0 ** -60 * 1.2345, 7e37], np.float32)
    hi, lo = tb.split(x)
    assert np.array_equal(hi[:3], np.array([1.0, 1.0 + 2.0 ** -10, 1.0], np.float32))
    assert lo[2] == np.float32(2.0 ** -11)
    rel = np.abs((hi.astype(np.float64) + lo) - x) / np.abs(x)
    assert (rel < 2.0 ** -20).all()
    zero = torch.zeros(2, 2, dtype=torch.float64)   # an element whose products are all 0 must come out exactly 0
    assert tb.worst_ratio(torch.zeros(2, 2), zero, zero) == 0.0
    assert tb.worst_ratio(torch.full((2, 2), 1e-30), zero, zero) == np.inf
