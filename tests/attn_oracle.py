"""The attention aggregation of include/roc_b200.h (roc_sg_attn_*), forward and backward, in numpy / scipy fp64.

Rows are the plan's local rows r with id i = self_base + r; row_end holds their END offsets (global, less col_left
gives the position in col).  x, s (2*heads score columns: s_dst | s_src) and, in the backward, every per-node input
are indexed by the ids col holds.  The formulas are applied literally, also on graphs that are not symmetric and
to rows of degree 0."""
import numpy as np
import scipy.sparse as sp

EDGE_BLOCK = 1 << 18      # edges per block of the per-edge dot products


def _edges(row_end, col, col_left, self_base):
    re = np.asarray(row_end, dtype=np.int64) - int(col_left)
    deg = np.diff(np.concatenate([[0], re]))
    r = np.repeat(np.arange(re.shape[0]), deg)
    j = np.asarray(col, dtype=np.int64)[:re[-1] if re.shape[0] else 0]
    return re, deg, r, j, r + int(self_base)


def _leaky(z, slope):
    return np.where(z > 0, z, slope * z)


def _per_head_dot(a, ia, b, ib, heads):
    """[E][heads]: sum over each head's columns of a[ia[e]] * b[ib[e]], in blocks of edges."""
    F = a.shape[1] // heads
    out = np.empty((ia.shape[0], heads))
    for e0 in range(0, ia.shape[0], EDGE_BLOCK):
        e1 = min(e0 + EDGE_BLOCK, ia.shape[0])
        out[e0:e1] = (a[ia[e0:e1]] * b[ib[e0:e1]]).reshape(e1 - e0, heads, F).sum(-1)
    return out


def _weighted_gather(r, j, w, rows, y, heads, n_cols):
    """out[r] += w[e, k] * y[j][kF:(k+1)F] for every edge e, per head k (a sparse product per head)."""
    F = y.shape[1] // heads
    out = np.zeros((rows, y.shape[1]))
    for k in range(heads):
        a = sp.csr_matrix((w[:, k], (r, j)), shape=(rows, n_cols))
        out[:, k * F:(k + 1) * F] = a @ y[:, k * F:(k + 1) * F]
    return out


def _row_sum(r, v, rows):
    return np.stack([np.bincount(r, weights=v[:, k], minlength=rows) for k in range(v.shape[1])], axis=1)


def forward(row_end, col, x, s, heads, slope, self_base=0, col_left=0):
    """-> out [nloc][H], stats [nloc][2*heads] (m | 1/Z), fp64."""
    x = np.asarray(x, dtype=np.float64)
    s = np.asarray(s, dtype=np.float64)
    re, deg, r, j, i = _edges(row_end, col, col_left, self_base)
    nloc = re.shape[0]
    y = _leaky(s[i, :heads] + s[j, heads:2 * heads], slope)                 # [E][heads]
    m = np.full((nloc, heads), -np.inf)
    np.maximum.at(m, r, y)
    m[deg == 0] = 0.0
    ex = np.exp(y - m[r])
    Z = _row_sum(r, ex, nloc)
    iz = np.where(deg[:, None] > 0, 1.0 / np.where(Z > 0, Z, 1.0), 0.0)
    alpha = ex * iz[r]
    out = _weighted_gather(r, j, alpha, nloc, x, heads, x.shape[0])
    return out, np.concatenate([m, iz], axis=1)


def backward(row_end, col, x, s, out, stats, gy, heads, slope, self_base=0, col_left=0):
    """-> in_grad [nloc][H], score_grad [nloc][2*heads] (d s_dst | d s_src), fp64.  x, s, out, stats, gy are indexed
    by col's ids."""
    x, s, out, stats, gy = (np.asarray(a, dtype=np.float64) for a in (x, s, out, stats, gy))
    re, deg, r, j, i = _edges(row_end, col, col_left, self_base)
    nloc = re.shape[0]
    F = x.shape[1] // heads
    D = (gy * out).reshape(gy.shape[0], heads, F).sum(-1)                  # [N][heads]
    m, iz = stats[:, :heads], stats[:, heads:2 * heads]

    def alpha(dst, src):
        z = s[dst, :heads] + s[src, heads:2 * heads]
        a = np.where(iz[dst] == 0, 0.0, np.exp(_leaky(z, slope) - m[dst]) * iz[dst])
        return a, np.where(z > 0, 1.0, slope)

    a1, l1 = alpha(i, j)                                                    # a(i<-j)
    dz1 = a1 * (_per_head_dot(gy, i, x, j, heads) - D[i]) * l1
    a2, l2 = alpha(j, i)                                                    # a(j<-i)
    dz2 = a2 * (_per_head_dot(gy, j, x, i, heads) - D[j]) * l2
    in_grad = _weighted_gather(r, j, a2, nloc, gy, heads, gy.shape[0])
    return in_grad, np.concatenate([_row_sum(r, dz1, nloc), _row_sum(r, dz2, nloc)], axis=1)


def score_grad_magnitude(row_end, col, x, s, out, stats, gy, heads, slope, self_base=0, col_left=0):
    """[nloc][2*heads]: backward's score gradients with every term replaced by its magnitude, sum_e a |l| (sum_f
    |G X| + |D|).  An fp32 evaluation of (G.X - D) cancels; its error is relative to this, not to the result."""
    x, s, out, stats, gy = (np.abs(np.asarray(a, dtype=np.float64)) if k not in (1, 3)
                            else np.asarray(a, dtype=np.float64) for k, a in enumerate((x, s, out, stats, gy)))
    re, deg, r, j, i = _edges(row_end, col, col_left, self_base)
    nloc = re.shape[0]
    F = x.shape[1] // heads
    D = (gy * out).reshape(gy.shape[0], heads, F).sum(-1)
    m, iz = stats[:, :heads], stats[:, heads:2 * heads]

    def alpha(dst, src):
        z = s[dst, :heads] + s[src, heads:2 * heads]
        return np.where(iz[dst] == 0, 0.0, np.exp(_leaky(z, slope) - m[dst]) * iz[dst]) * np.where(z > 0, 1.0, slope)

    t1 = alpha(i, j) * (_per_head_dot(gy, i, x, j, heads) + D[i])
    t2 = alpha(j, i) * (_per_head_dot(gy, j, x, i, heads) + D[j])
    return np.concatenate([_row_sum(r, t1, nloc), _row_sum(r, t2, nloc)], axis=1)
