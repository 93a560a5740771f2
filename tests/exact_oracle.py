"""numpy / scipy fp64 restatement of the exact backwards of include/roc_b200.h (roc_sg_transpose_sum_backward,
roc_sg_transpose_minmax_backward, roc_sg_attn_backward_exact): the true adjoints of the sum, max / min and attention
aggregations on any whole graph, directed, with duplicate edges or nodes without in- or out-edges.

A graph is row_end (END offsets of its N rows) and col (the source of each edge); dst(e) is the row that owns edge e.
Per-node arrays have N rows."""
import numpy as np
import scipy.sparse as sp

import attn_oracle as ao

NORM, RELU = 1, 2


def edges(row_end):
    """(dst of every edge, in-degree of every row)."""
    t = np.asarray(row_end, dtype=np.int64)
    deg = np.diff(np.concatenate([[0], t]))
    return np.repeat(np.arange(t.shape[0]), deg), deg


def adjacency(row_end, col, n):
    """A[i][j] = the number of edges j -> i (duplicates counted), as a sparse matrix."""
    t = np.asarray(row_end, dtype=np.int64)
    indptr = np.concatenate([[0], t])
    return sp.csr_matrix((np.ones(t[-1] if n else 0), np.asarray(col, dtype=np.int64), indptr), shape=(n, n))


def sum_backward(row_end, col, gy, n):
    """in_grad[j] = sum over the edges e with col[e] = j of gy[dst(e)]  (A^T gy), fp64."""
    return np.asarray(adjacency(row_end, col, n).T @ np.asarray(gy, dtype=np.float64))


def sum_backward_epi(row_end, col, gy, n, epi):
    """sum_backward with the epilogue applied in fp32 as the kernels do: the (exactly representable) sum divided by
    sqrtf of each row's in-degree for NORM (0 / 0 = NaN, x / 0 = inf), then relu.  For data whose sums are exact."""
    s = sum_backward(row_end, col, gy, n)
    out = s.astype(np.float32)
    assert np.array_equal(out.astype(np.float64), s), "the sum is not exact in fp32"
    if epi & NORM:
        _, deg = edges(row_end)
        with np.errstate(divide="ignore", invalid="ignore"):
            out = out / np.sqrt(deg.astype(np.float32))[:, None]
    if epi & RELU:
        out = np.maximum(out, np.float32(0))
    return out


def minmax_forward(row_end, col, x, aggr):
    """Max (aggr 1) or min (2) over each row's in-edges: (values, the source of the first edge holding the extreme;
    0 and 0xFFFFFFFF for a row of degree 0), for data without NaN."""
    t = np.asarray(row_end, dtype=np.int64)
    x = np.asarray(x)
    n, h = t.shape[0], x.shape[1]
    out, arg = np.zeros((n, h), x.dtype), np.full((n, h), 0xFFFFFFFF, np.uint32)
    s = 0
    for r in range(n):
        if t[r] > s:
            src = np.asarray(col[s:t[r]], dtype=np.int64)
            v = x[src]
            k = np.argmax(v, axis=0) if aggr == 1 else np.argmin(v, axis=0)   # the first extreme in edge order
            out[r], arg[r] = v[k, np.arange(h)], src[k]
        s = t[r]
    return out, arg


def minmax_backward(row_end, col, gy, arg, n, block=128):
    """in_grad[j][h] = sum over the DISTINCT destinations i of j's out-edges of (arg[i][h] == j ? gy[i][h] : 0),
    fp64."""
    dst, _ = edges(row_end)
    src = np.asarray(col, dtype=np.int64)
    _, first = np.unique(dst * n + src, return_index=True)        # one entry per distinct (i, j)
    i, j = dst[first], src[first]
    order = np.argsort(j, kind="stable")
    i, j = i[order], j[order]
    gy, arg = np.asarray(gy, dtype=np.float64), np.asarray(arg).astype(np.int64)
    out = np.zeros((n, gy.shape[1]))
    if j.shape[0] == 0:
        return out
    starts = np.flatnonzero(np.concatenate([[True], j[1:] != j[:-1]]))
    for c0 in range(0, gy.shape[1], block):
        c1 = min(c0 + block, gy.shape[1])
        v = np.where(arg[i, c0:c1] == j[:, None], gy[i, c0:c1], 0.0)
        out[j[starts], c0:c1] = np.add.reduceat(v, starts, axis=0)
    return out


def attn_backward(row_end, col, x, s, out, stats, gy, heads, slope, magnitude=False):
    """-> in_grad [N][H], score_grad [N][2*heads] (d s_dst | d s_src), fp64: the true adjoint of the attention forward,
    each edge (duplicates too) counted once, with a recomputed from stats and D = G . O per head from out.  With
    magnitude, every term is replaced by its magnitude: the bound an fp32 evaluation's rounding is relative to."""
    x, s, out, stats, gy = (np.asarray(a, dtype=np.float64) for a in (x, s, out, stats, gy))
    if magnitude:
        x, out, gy = np.abs(x), np.abs(out), np.abs(gy)
    i, _ = edges(row_end)
    j = np.asarray(col, dtype=np.int64)
    n, F = gy.shape[0], x.shape[1] // heads
    D = (gy * out).reshape(n, heads, F).sum(-1)
    m, iz = stats[:, :heads], stats[:, heads:2 * heads]
    z = s[i, :heads] + s[j, heads:2 * heads]
    a = np.where(iz[i] == 0, 0.0, np.exp(ao._leaky(z, slope) - m[i]) * iz[i])    # a(i<-j)
    l = np.where(z > 0, 1.0, slope)
    dot = ao._per_head_dot(gy, i, x, j, heads)
    dz = a * ((dot + D[i]) if magnitude else (dot - D[i])) * l
    in_grad = ao._weighted_gather(j, i, a, n, gy, heads, n)
    return in_grad, np.concatenate([ao._row_sum(i, dz, n), ao._row_sum(j, dz, n)], axis=1)
