"""make_golden_sg.py — ScatterGather golden rows at four widths (16 to 256 floats), minted on the GPU from
the REFERENCE's own aggre_coop_kernel (oracle/_ref, scattergather_kernel.cu:20-76).

    python tests/golden/make_golden_sg.py [out.npz]        # needs a GPU and oracle/_ref/libroc_ref.so

R-MAT scale 14 (hub rows, rows cut at chunk boundaries) with seeded features of width 16 / 64 / 128 / 256.  The
output is stored for a fixed sample of 96 rows (`rows`), which keeps the file small; the test regenerates graph and
features with graph() / features() and compares those rows."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from roc_b200 import datasets  # noqa: E402

WIDTHS = (16, 64, 128, 256)


def graph():
    re_t, col_t = datasets.rmat_graph(14, 150000, seed=8)
    return re_t.numpy().astype(np.uint64), col_t.numpy().astype(np.uint32)


def features(n, h):
    return np.random.RandomState(h).rand(n, h).astype(np.float32) - 0.5


def main():
    import torch
    from oracle import ref
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_golden_sg.npz")
    assert ref.available(), "oracle/_ref/libroc_ref.so missing"
    row_end, col = graph()
    n = row_end.shape[0]
    d_re = torch.from_numpy(row_end.astype(np.int64)).cuda()
    d_col = torch.from_numpy(col.astype(np.int32)).cuda()
    rp, es = ref.edge_structs(d_col, d_re, 0, 0)
    rows = np.sort(np.random.RandomState(9).choice(n, 96, replace=False))
    G = {"rows": rows}
    for h in WIDTHS:
        y = ref.scatter_gather(0, n - 1, 0, rp, es, torch.from_numpy(features(n, h)).cuda())
        torch.cuda.synchronize()
        G["out_%d" % h] = y.cpu().numpy()[rows]
    np.savez_compressed(out, **G)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
