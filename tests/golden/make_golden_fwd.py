"""make_golden_fwd.py — SHA-256 digests of the tensor-core forward and dX GEMMs (k_tc_linear), bit for bit.

    python tests/golden/make_golden_fwd.py [out.npz]       # needs an H100; run on a build whose bits are the golden

The fp64 tests of tests/test_linear_gpu.py bound Y's and dX's error; they cannot see a change in the order of the MMAs,
which moves the last bits.  tests/test_fwd_digest_gpu.py recomputes every case below and compares the digest of the
output bytes.  Inputs come from an integer hash of (row, column, salt) evaluated on the GPU (make_golden_dw.hashed), the
dropout mask is the library's own.  Every N-tile width (NC = 1, 2, 4 and two N-tiles of 4) meets every epilogue
instantiation (none, norm, output mask, output mask + relu mask + norm, and the generic kernel through relu and through
an accumulating dX) and the fused input mask, at K values that are not multiples of 32 and at a row count that gives
every CTA of a 132-SM grid at least 3 tiles and ends in a partial tile.  The three launches of bench.py config 2's step
run at full size.  Forward and dX do not depend on the SM count.  A few sampled values per case are kept for diagnosis."""
import hashlib
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from roc_b200 import _lib  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402

_spec = importlib.util.spec_from_file_location("make_golden_dw", os.path.join(HERE, "make_golden_dw.py"))
_dw = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_dw)
hashed, digest, sample_index = _dw.hashed, _dw.digest, _dw.sample_index

TILE_ROWS = 132 * 128 * 3 + 37     # >= 3 tiles per CTA on 132 SMs, and a partial last tile
PROD_ROWS = 1 << 22                # bench.py config 2

# (inDim, outDim) of each N-tile width: fwd N = outDim, dX N = inDim; K = the other one, never a multiple of 32
FWD_SHAPES = ((100, 16), (602, 41), (70, 128), (300, 200))
DX_SHAPES = ((16, 100), (64, 41), (128, 70), (200, 300))
FWD_EPIS = ("plain", "norm", "relu", "mask-norm")
DX_EPIS = ("plain", "omask", "omask-reluof-norm", "acc")


def cases():
    """name -> (kind, rows, inDim, outDim, epilogue)"""
    c = {}
    for inn, out in FWD_SHAPES:
        for e in FWD_EPIS:
            c["fwd-in%d-out%d-%s" % (inn, out, e)] = ("fwd", TILE_ROWS, inn, out, e)
    for inn, out in DX_SHAPES:
        for e in DX_EPIS:
            c["dx-in%d-out%d-%s" % (inn, out, e)] = ("dx", TILE_ROWS, inn, out, e)
    c["prod-fwd-in602-out64-mask-norm"] = ("fwd", PROD_ROWS, 602, 64, "mask-norm")
    c["prod-fwd-in64-out41-mask-norm"] = ("fwd", PROD_ROWS, 64, 41, "mask-norm")
    c["prod-dx-in64-out41-omask-reluof-norm"] = ("dx", PROD_ROWS, 64, 41, "omask-reluof-norm")
    return c


def row_ends(rows, dev="cuda"):
    """END offsets of a CSR whose row r has 1 + hash(r) % 29 entries"""
    r = torch.arange(rows, device=dev, dtype=torch.int64)
    h = (r * 0x9E3779B1 + 0x7F4A7C15) & 0xFFFFFFFF
    h = (h ^ (h >> 13)) * 0x5BD1E995 & 0xFFFFFFFF
    return torch.cumsum(1 + (h ^ (h >> 15)) % 29, 0)


def run_case(kind, rows, inn, out, epi, dev="cuda"):
    """the output of one tensor-core launch on the host, and roc_last_gemm_info of it"""
    w = hashed(out, inn, 3, dev).contiguous() * 0.25
    norm = row_ends(rows, dev) if "norm" in epi else None
    if kind == "fwd":
        x = hashed(rows, inn, 1, dev)
        y = K.padded(rows, out, dev)
        if "mask" in epi:
            mask = K.dropout_mask(rows, inn, 0, 0.5, 7, 1, dev)
            K.linear_fwd_dropout(x, w, mask, 0.5, norm_row_end=norm, out=y)
        else:
            K.linear_fwd(x, w, activation=1 if epi == "relu" else 0, norm_row_end=norm, out=y)
        info = _lib.last_gemm_info(_lib.GEMM_FWD)
        res = y
    else:
        dy = hashed(rows, out, 2, dev)
        dx = hashed(rows, inn, 5, dev) if epi == "acc" else K.padded(rows, inn, dev)
        ro = hashed(rows, inn, 4, dev) if "reluof" in epi else None
        mask = K.dropout_mask(rows, inn, 0, 0.5, 7, 1, dev) if "omask" in epi else None
        dw = torch.zeros((out, inn), device=dev)
        K.linear_bwd_fused(dx, w, None, dy, dw, dx,       # X is not read when only dX is computed
                           mask=mask, rate=0.5 if mask is not None else 0.0, relu_of=ro, norm_row_end=norm,
                           accumulate_dx=epi == "acc", parts=_lib.LINEAR_BWD_ONLY_DX)
        info = _lib.last_gemm_info(_lib.GEMM_DX)
        res = dx
    return res.cpu().numpy(), info


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "fwd_digests.npz")
    G = {"device": np.array(torch.cuda.get_device_name(0))}
    for name, (kind, rows, inn, o, epi) in cases().items():
        a, info = run_case(kind, rows, inn, o, epi)
        assert info["path"] == 1, (name, info)
        G["sha_" + name] = np.array(digest(a))
        G["sample_" + name] = a.reshape(-1)[sample_index(a.size)]
        print(name, info, G["sha_" + name], flush=True)
        del a
    np.savez_compressed(out, **G)
    print("wrote", out)


if __name__ == "__main__":
    main()
