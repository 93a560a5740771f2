import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `pytest -m gpu`)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_golden.npz")


def golden_inputs():
    """The seeded inputs tests/golden/make_golden.py fed the reference's kernels, regenerated in the same order
    (numpy's RandomState stream is stable), so ref_golden.npz only has to hold the outputs."""
    rng = np.random.RandomState(20260921)
    g = {}
    for h in (16, 41, 64):
        g["A_sg_in_%d" % h] = rng.rand(1000, h).astype(np.float32) * 2 - 1
    g["B_sg_in_32"] = rng.rand(1024, 32).astype(np.float32) * 2 - 1
    g["lin_X"] = rng.rand(200, 33).astype(np.float32) * 2 - 1
    g["lin_W"] = rng.rand(9, 33).astype(np.float32) * 2 - 1     # W_mem[o*in + i]
    g["lin_dY"] = rng.rand(200, 9).astype(np.float32) * 2 - 1
    g["act_x"] = rng.randn(64, 24).astype(np.float32)
    g["act_dy"] = rng.randn(64, 24).astype(np.float32)
    g["sm_logits"] = rng.randn(500, 7).astype(np.float32) * 2
    g["sm_labels"] = rng.randint(0, 7, size=500).astype(np.int32)
    g["sm_mask"] = rng.randint(0, 4, size=500).astype(np.int32)
    g["adam_w"] = rng.randn(1000).astype(np.float32)
    g["adam_g"] = rng.randn(3, 1000).astype(np.float32)
    g["adam_m"] = rng.randn(1000).astype(np.float32) * 0.1
    g["adam_v"] = np.abs(rng.randn(1000).astype(np.float32) * 0.1)
    return g


@pytest.fixture(scope="session")
def golden():
    """Outputs of the reference's kernels (tests/golden/ref_golden.npz) plus the inputs they were computed from.
    Graph A's outputs at H = 41 and 64 are kept for the rows A_rows_<H> only; A_rows_16 is every row."""
    g = dict(np.load(GOLDEN))
    g.update(golden_inputs())
    g["A_rows_16"] = np.arange(g["A_row_end"].shape[0])
    return g


def rel_close(got, want, rtol=1e-4, atol_scale=1e-5, what=""):
    """The parity bar of BASELINE.json's north_star: 1e-4 relative fp32.  `atol_scale`
    * max|want| absorbs cancellation in sums (an fp32 sum of d terms is only good to
    ~d*eps*sum|x|, so elements that cancel to ~0 cannot meet a pure relative bound —
    the reference's own atomics-ordered sums do not either)."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    scale = np.abs(want).max() if want.size else 0.0
    err = np.abs(got - want)
    bound = rtol * np.abs(want) + atol_scale * scale + 1e-30
    bad = err > bound
    assert not bad.any(), "%s: %d/%d elements off; worst err %.3e at %s (want %.6g got %.6g)" % (
        what, int(bad.sum()), bad.size, float(err.max()), np.unravel_index(err.argmax(), err.shape),
        float(want.flat[err.argmax()]), float(got.flat[err.argmax()]))
