"""numpy fp64 restatement of edge-weighted ScatterGather (include/roc_b200.h, roc_sg_weighted_* and
roc_sg_edge_dot_planned): the forward, its exact input gradient through the transposed CSR, the edge-weight gradient
(SDDMM), the transpose build and GCN's symmetric normalisation of edge weights.

A CSR is row_end (END offsets of the plan's rows in the edge array, the plan's edges starting at col_left) and col
(the sources of those edges).  w, dw: one value per edge of the plan, in its edge order."""
import numpy as np


def rows_of(row_end, col_left=0):
    """The plan row of every edge, and the rows' [start, end) in the plan's edge array."""
    t = np.asarray(row_end, dtype=np.int64) - int(col_left)
    s = np.concatenate([[0], t[:-1]]).astype(np.int64)
    return np.repeat(np.arange(t.shape[0]), t - s), s, t


def forward(row_end, col, x, w, col_left=0):
    """out[r] = sum over row r's edges e of w[e] * x[col[e]]."""
    row, _, t = rows_of(row_end, col_left)
    out = np.zeros((t.shape[0], x.shape[1]))
    np.add.at(out, row, np.asarray(w, dtype=np.float64)[:, None] * np.asarray(x, dtype=np.float64)[col])
    return out


def input_grad(row_end, col, gy, w, n):
    """The true adjoint of forward on a whole graph: in_grad[j] = sum over the edges e with col[e] = j of
    w[e] * gy[row(e)]."""
    row, _, _ = rows_of(row_end)
    g = np.zeros((n, gy.shape[1]))
    np.add.at(g, np.asarray(col, dtype=np.int64), np.asarray(w, dtype=np.float64)[:, None] * np.asarray(gy, np.float64)[row])
    return g


def edge_dot(row_end, col, gy, x, col_left=0):
    """dw[e] = gy[row(e)] . x[col[e]]: gy has the plan's rows, x is indexed like forward's input."""
    row, _, _ = rows_of(row_end, col_left)
    return np.einsum("eh,eh->e", np.asarray(gy, np.float64)[row], np.asarray(x, np.float64)[col])


def transpose(row_end, col, n):
    """(row_end_t [n] END offsets of each node's out-edges, col_t their destinations, perm the original edge of each
    transposed edge), by a stable sort of the sources."""
    col = np.asarray(col, dtype=np.int64)
    row, _, _ = rows_of(row_end)
    perm = np.argsort(col, kind="stable")
    row_end_t = np.cumsum(np.bincount(col, minlength=n)).astype(np.uint64)
    return row_end_t, row[perm].astype(np.uint32), perm.astype(np.uint32)


def gcn_edge_weights(row_end, col, w):
    """w_e / sqrt(d_i d_j) for edge e = (i <- j), d the weighted in-degree; 0 where d_i d_j is 0."""
    row, _, t = rows_of(row_end)
    w = np.asarray(w, dtype=np.float64)
    d = np.zeros(t.shape[0])
    np.add.at(d, row, w)
    dd = d[row] * d[np.asarray(col, dtype=np.int64)]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(dd != 0, w / np.sqrt(np.where(dd != 0, dd, 1.0)), 0.0)
