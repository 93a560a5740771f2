"""make_golden_dw.py — SHA-256 digests of the tensor-core dW (k_tc_linear_dw + k_splitk_reduce), bit for bit.

    python tests/golden/make_golden_dw.py [out.npz]        # needs an H100; run on a build whose dW bits are the golden

The fp64 tests of tests/test_linear_gpu.py bound dW's error; they cannot see a change in the order of the MMAs or of
the split-K partial sums, which moves the last bits.  tests/test_dw_digest_gpu.py recomputes every case below and
compares the digest of the dW bytes.  Inputs come from an integer hash of (row, column, salt) evaluated on the GPU, so
they do not depend on a random number generator's implementation; the dropout mask is the library's own.  The split
count follows the SM count, so the file records it and the test skips on a GPU with another one.  A few sampled
values per case are kept for diagnosis."""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from roc_b200 import _lib  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402

RING_SPLIT_ROWS = 416        # 13 k-blocks per split: >= 3 turns of a 4-stage ring
EMPTY_ROWS = 8449            # the last splits hold no rows
PROD_ROWS = 1 << 22          # bench.py config 2


def ring_rows(inn, sms):
    """each split RING_SPLIT_ROWS rows, the last 5 less (a partial last k-block)"""
    return (sms // -(-inn // 128)) * RING_SPLIT_ROWS - 5


def cases(sms):
    """name -> (rows, inDim, outDim, masked).  outDim 16 / 41 / 128 / 200 select NC = 1 / 2 / 4 / 8."""
    c = {}
    for out, inn in ((16, 100), (41, 602), (128, 256), (200, 300)):
        for masked in (False, True):
            m = "-mask" if masked else ""
            c["ring-in%d-out%d%s" % (inn, out, m)] = (ring_rows(inn, sms), inn, out, masked)
            c["empty-in%d-out%d%s" % (inn, out, m)] = (EMPTY_ROWS, inn, out, masked)
    c["prod-in602-out64-mask"] = (PROD_ROWS, 602, 64, True)
    c["prod-in64-out41-mask"] = (PROD_ROWS, 64, 41, True)
    return c


def hashed(rows, cols, salt, dev="cuda", chunk=1 << 18):
    """[rows][cols] (row-padded) of values in [-1, 1) with full 24-bit mantissas, a hash of (row, col, salt)"""
    out = K.padded(rows, cols, dev)
    c = torch.arange(cols, device=dev, dtype=torch.int64)
    for r0 in range(0, rows, chunk):
        r = torch.arange(r0, min(rows, r0 + chunk), device=dev, dtype=torch.int64)
        h = (r[:, None] * 0x9E3779B1 + c[None, :] * 0x85EBCA77 + salt * 0xC2B2AE3D) & 0xFFFFFFFF
        h = h ^ (h >> 15)
        h = (h * 0x2C1B3C6D) & 0xFFFFFFFF
        h = h ^ (h >> 12)
        out[r0:r0 + r.numel()] = ((h & 0xFFFFFF).float() - 8388608.0) / 8388608.0
    return out


def run_case(rows, inn, out, masked, dev="cuda"):
    """dW = dY^T dropout(X) from zero through the tensor-core path; returns (dW on the host, roc_last_gemm_info)"""
    x = hashed(rows, inn, 1, dev)
    dy = hashed(rows, out, 2, dev)
    mask = K.dropout_mask(rows, inn, 0, 0.5, 7, 1, dev) if masked else None
    w = torch.zeros((out, inn), device=dev)
    dw = torch.zeros((out, inn), device=dev)
    K.linear_bwd_fused(x, w, None, dy, dw, None, mask=mask, rate=0.5 if masked else 0.0,
                       parts=_lib.LINEAR_BWD_ONLY_DW)
    info = _lib.last_gemm_info(_lib.GEMM_DW)
    return dw.cpu().numpy(), info


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def sample_index(n):
    return np.random.RandomState(5).choice(n, min(n, 16), replace=False)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "dw_digests.npz")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    G = {"sm_count": np.int64(sms), "device": np.array(torch.cuda.get_device_name(0))}
    for name, (rows, inn, o, masked) in cases(sms).items():
        dw, info = run_case(rows, inn, o, masked)
        assert info["path"] == 1, (name, info)
        G["sha_" + name] = np.array(digest(dw))
        G["sample_" + name] = dw.reshape(-1)[sample_index(dw.size)]
        print(name, info, G["sha_" + name], flush=True)
    np.savez_compressed(out, **G)
    print("wrote", out)


if __name__ == "__main__":
    main()
