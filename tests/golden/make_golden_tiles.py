"""make_golden_tiles.py — SHA-256 digests of k_tc_linear at the row counts where the CTAs' tile counts differ.

    python tests/golden/make_golden_tiles.py [out.npz]     # needs an H100; run on a build whose bits are the golden

tests/test_fwd_tiles_gpu.py recomputes every case below at the whole chip and at two smaller SM budgets and compares
the digest of the output bytes.  The inputs and the digest are those of make_golden_fwd.py (run_case, digest).  Forward
and dX do not depend on the SM count, so one set of digests serves every budget.

Streamed W (the CTA's W slice does not fit in shared memory), at NC = 1, 2 and 4:
  - 397 and 264 tiles: uneven and even tile counts per CTA on 132, 130 and 8 CTAs;
  - 1 tile and 2 tiles: fewer tiles than CTAs.
W resident: row counts that give 1, 2 and 3 tiles per CTA on 132 SMs (132, 138 and 272 tiles), each ending in a partial
tile, under every fixed epilogue and the generic one, at NC = 1 and 2.  The digests were written by the build before
the Y staging tile and the input-mask words by TMA."""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_fwd", os.path.join(HERE, "make_golden_fwd.py"))
F = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(F)

STREAM_ROWS = {"t397": 396 * 128 + 37, "t264": 264 * 128 - 5, "t1": 100, "t2": 128 + 77}
RES_ROWS = {"r1": 131 * 128 + 37, "r2": 137 * 128 + 37, "r3": 271 * 128 + 37}   # 132, 138, 272 tiles
# (kind, inDim, outDim, epilogues): streamed shapes at NC = 1, 2, 4 (two N-tiles of 4), resident shapes at NC = 1, 2
STREAM_SHAPES = (("fwd", 602, 64, ("mask-norm", "plain")), ("fwd", 700, 16, ("norm",)), ("fwd", 300, 200, ("relu",)),
                 ("dx", 128, 70, ("omask-reluof-norm",)))
RES_SHAPES = (("fwd", 64, 41, ("plain", "norm", "mask-norm", "relu")), ("fwd", 100, 16, ("norm",)),
              ("dx", 64, 41, ("plain", "omask", "omask-reluof-norm", "acc")), ("dx", 16, 100, ("omask",)))


def cases():
    """name -> (kind, rows, inDim, outDim, epilogue, streamed)"""
    c = {}
    for rows_tab, shapes, streamed in ((STREAM_ROWS, STREAM_SHAPES, True), (RES_ROWS, RES_SHAPES, False)):
        for tag, rows in rows_tab.items():
            for kind, inn, out, epis in shapes:
                for e in epis:
                    c["%s-%s-in%d-out%d-%s" % (tag, kind, inn, out, e)] = (kind, rows, inn, out, e, streamed)
    return c


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "fwd_tile_digests.npz")
    G = {"device": np.array(torch.cuda.get_device_name(0))}
    for name, (kind, rows, inn, o, epi, _) in cases().items():
        a, info = F.run_case(kind, rows, inn, o, epi)
        assert info["path"] == 1, (name, info)
        G["sha_" + name] = np.array(F.digest(a))
        G["sample_" + name] = a.reshape(-1)[F.sample_index(a.size)]
        print(name, info, G["sha_" + name], flush=True)
        del a
    np.savez_compressed(out, **G)
    print("wrote", out)


if __name__ == "__main__":
    main()
