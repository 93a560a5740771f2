"""fp64 numpy oracle of the multi-label sigmoid cross-entropy (roc_sigmoid_xent_bwd, include/roc_b200.h).

sigmoid_xent(z, y, mask, deg=None) returns the gradient and the metrics dict the kernel computes, from the semantics the
header states: per element l = max(z, 0) - z*y + log1p(exp(-|z|)); gradient sigmoid(z) - y on train rows, 0 elsewhere,
divided by sqrt(deg) when the norm is fused; a class is predicted positive iff z > 0; per split (train, val, test) the
loss sum, rows, exact matches and tp / fp / fn.  No code is shared with the product."""
import numpy as np
from scipy.special import expit

SPLITS = 3   # ROC_MASK_TRAIN, VAL, TEST; ROC_MASK_NONE rows count nowhere


def unpack_multilabels(bits, c):
    """uint32 [rows][W] -> uint8 [rows][c]: bit c % 32 of word c // 32 (the inverse of model.pack_multilabels)."""
    b = np.ascontiguousarray(np.asarray(bits, dtype=np.uint32))
    rows = b.shape[0]
    u8 = b.view(np.uint8).reshape(rows, -1)
    return np.unpackbits(u8, axis=1, bitorder="little")[:, :c]


def element_loss(z, y):
    z = np.asarray(z, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    with np.errstate(over="ignore"):
        return np.maximum(z, 0.0) - z * y + np.log1p(np.exp(-np.abs(z)))


def sigmoid_xent(z, y, mask, deg=None):
    """z: [N][C] fp32 logits, y: [N][C] 0/1, mask: [N] ROC_MASK_*, deg: [N] in-degrees for the fused norm (or None).
    Returns (grad fp64 [N][C], metrics dict with loss (fp64), rows, exact, tp, fp, fn (ints), each [train, val, test])."""
    z64 = np.asarray(z, dtype=np.float64)
    y = np.asarray(y).astype(bool)
    mask = np.asarray(mask)
    train = (mask == 0)[:, None]
    g = np.where(train, expit(z64) - y, 0.0)
    if deg is not None:
        with np.errstate(divide="ignore", invalid="ignore"):
            g = g / np.sqrt(np.asarray(deg, dtype=np.float64))[:, None]
    loss = element_loss(z64, y)
    pred = np.asarray(z) > 0
    m = {k: [0] * SPLITS for k in ("rows", "exact", "tp", "fp", "fn")}
    m["loss"] = [0.0] * SPLITS
    for s in range(SPLITS):
        r = mask == s
        m["loss"][s] = float(loss[r].sum())
        m["rows"][s] = int(r.sum())
        m["exact"][s] = int(np.all(pred[r] == y[r], axis=1).sum())
        m["tp"][s] = int((pred[r] & y[r]).sum())
        m["fp"][s] = int((pred[r] & ~y[r]).sum())
        m["fn"][s] = int((~pred[r] & y[r]).sum())
    return g, m


def micro_f1(m):
    out = []
    for tp, fp, fn in zip(m["tp"], m["fp"], m["fn"]):
        den = 2 * tp + fp + fn
        out.append(2.0 * tp / den if den else float("nan"))
    return out
