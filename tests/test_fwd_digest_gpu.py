"""Bit-exact pin of the tensor-core forward and dX GEMMs (k_tc_linear at NC = 1, 2, 4 and two N-tiles, every epilogue
instantiation, with and without the fused input dropout mask) against the SHA-256 digests in
tests/golden/fwd_digests.npz.

test_linear_gpu.py bounds Y's and dX's error against fp64, which any correct summation order meets.  A change to the
kernel that reorders the MMAs of an output element still passes that bound but moves the last bits of the output, and
of everything trained after it.  This file sees such a change.  The cases and their inputs are those of
tests/golden/make_golden_fwd.py, which wrote the digests.  Forward and dX do not depend on the SM count."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_fwd", os.path.join(HERE, "golden", "make_golden_fwd.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)
GOLDEN = dict(np.load(os.path.join(HERE, "golden", "fwd_digests.npz")))
CASES = G.cases()

EPI = {"plain": 0, "norm": 8, "relu": -1, "mask-norm": 8, "omask": 2, "omask-reluof-norm": 14, "acc": -1}
# the shared-memory regimes of k_tc_linear (roc_gemm_info w_resident, epi_bufs): each is reached by one case
REGIMES = {"prod-fwd-in602-out64-mask-norm": (0, 0),          # W streams with A (311 KB per CTA)
           "prod-fwd-in64-out41-mask-norm": (1, 0),           # W resident, no epilogue operands
           "prod-dx-in64-out41-omask-reluof-norm": (1, 2),    # W resident, double-buffered epilogue operands
           "dx-in128-out70-omask-reluof-norm": (0, 1)}        # W streams, one epilogue buffer


@pytest.mark.parametrize("name", sorted(CASES))
def test_fwd_digest(name):
    kind, rows, inn, out, epi = CASES[name]
    got, info = G.run_case(kind, rows, inn, out, epi)
    n = out if kind == "fwd" else inn
    assert info["path"] == 1, info
    assert info["nc"] == (1 if n <= 32 else 2 if n <= 64 else 4), info
    assert info["grid_y"] == -(-n // (32 * info["nc"])), info
    assert info["epi"] == EPI[epi], info
    if rows == G.TILE_ROWS:
        assert rows % 128 and -(-rows // 128) >= 3 * info["grid_x"], info
    if name in REGIMES:
        assert (info["w_resident"], info["epi_bufs"]) == REGIMES[name], info
    want = GOLDEN["sample_" + name]
    smp = got.reshape(-1)[G.sample_index(got.size)]
    assert G.digest(got) == str(GOLDEN["sha_" + name]), (
        "%s: output bits differ from the golden; sampled values differ by up to %.3e (max |out| %.3e)"
        % (name, float(np.abs(smp.astype(np.float64) - want).max()), float(np.abs(got).max())))
