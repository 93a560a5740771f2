"""Bit-exact pin of the tensor-core dW (k_tc_linear_dw at NC = 1, 2, 4, 8, with and without the fused dropout mask,
and the split-K reduce) against the SHA-256 digests in tests/golden/dw_digests.npz.

test_linear_gpu.py bounds dW's error against fp64, which any correct summation order meets.  A change to the kernel
that reorders the MMAs of an accumulator element, or the split-K partial sums, still passes that bound but moves the
last bits of dW, and of every weight after it.  This file sees such a change.  The cases and their inputs are those of
tests/golden/make_golden_dw.py, which wrote the digests."""
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_dw", os.path.join(HERE, "golden", "make_golden_dw.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)
GOLDEN = dict(np.load(os.path.join(HERE, "golden", "dw_digests.npz")))
SMS = int(GOLDEN["sm_count"])
CASES = G.cases(SMS)


@pytest.mark.parametrize("name", sorted(CASES))
def test_dw_digest(name):
    if torch.cuda.get_device_properties(0).multi_processor_count != SMS:
        pytest.skip("the digests were taken with %d SMs; the split-K ranges follow the SM count" % SMS)
    rows, inn, out, masked = CASES[name]
    dw, info = G.run_case(rows, inn, out, masked)
    assert info["path"] == 1, info
    assert info["nc"] == {16: 1, 41: 2, 64: 2, 128: 4, 200: 8}[out], info
    if name.startswith("ring"):
        assert info["v_per_split"] // 32 >= 3 * info["stages"] and rows % 32, info
    if name.startswith("empty"):
        assert (info["splits"] - 1) * info["v_per_split"] >= rows, info
    got = dw.reshape(-1)[G.sample_index(dw.size)]
    want = GOLDEN["sample_" + name]
    assert G.digest(dw) == str(GOLDEN["sha_" + name]), (
        "%s: dW bits differ from the golden; sampled values differ by up to %.3e (max |dW| %.3e)"
        % (name, float(np.abs(got.astype(np.float64) - want).max()), float(np.abs(dw).max())))
