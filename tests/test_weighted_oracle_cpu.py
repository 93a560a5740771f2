"""CPU: the numpy oracle of edge-weighted ScatterGather (weighted_oracle.py) against torch fp64 autograd of index_add
on directed, weighted graphs with duplicate edges, and its transpose build against the definition."""
import numpy as np
import pytest
import torch

import weighted_oracle as wo
from roc_b200 import datasets


def directed(n, e, seed, dup=True):
    """A directed graph with random in-degrees (some 0), duplicate edges and a node with no out-edge."""
    rng = np.random.RandomState(seed)
    dst = np.sort(rng.randint(0, n, size=e))
    src = rng.randint(0, n - 1, size=e)                     # node n - 1 has no out-edge
    if dup:
        src[1::5] = src[0::5][:src[1::5].shape[0]]          # repeated (dst, src) pairs wherever dst repeats
    row_end = np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64)
    order = np.lexsort((src, dst))
    return row_end, src[order].astype(np.uint32)


GRAPHS = [directed(30, 200, 1), directed(57, 40, 2), directed(200, 3000, 3), directed(9, 0, 4)]


def autograd(row_end, col, x, w, gy):
    """torch fp64: out = index_add over the edges of w[e] x[col[e]] into row(e); the gradients of <out, gy>."""
    row, _, t = wo.rows_of(row_end)
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    wt = torch.tensor(w, dtype=torch.float64, requires_grad=True)
    out = torch.zeros((t.shape[0], x.shape[1]), dtype=torch.float64)
    out = out.index_add(0, torch.from_numpy(row), wt[:, None] * xt[torch.from_numpy(col.astype(np.int64))])
    (out * torch.tensor(gy, dtype=torch.float64)).sum().backward()
    return out.detach().numpy(), xt.grad.numpy(), wt.grad.numpy()


@pytest.mark.parametrize("gi", range(len(GRAPHS)))
def test_oracle_against_autograd(gi):
    row_end, col = GRAPHS[gi]
    n, e = row_end.shape[0], col.shape[0]
    rng = np.random.RandomState(gi)
    x, gy, w = rng.randn(n, 7), rng.randn(n, 7), rng.randn(e)
    out, gx, gw = autograd(row_end, col, x, w, gy)
    np.testing.assert_allclose(wo.forward(row_end, col, x, w), out, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(wo.input_grad(row_end, col, gy, w, n), gx, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(wo.edge_dot(row_end, col, gy, x), gw, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("gi", range(len(GRAPHS)))
def test_transpose_is_the_adjoint(gi):
    """The transposed CSR lists every edge once, each transposed row's destinations increase, and the forward over it
    with the permuted weights is the oracle's input gradient."""
    row_end, col = GRAPHS[gi]
    n, e = row_end.shape[0], col.shape[0]
    re_t, col_t, perm = wo.transpose(row_end, col, n)
    assert re_t.shape == (n,) and int(re_t[-1]) == e
    assert sorted(perm.tolist()) == list(range(e))
    row, _, _ = wo.rows_of(row_end)
    assert np.array_equal(col_t, row[perm]) and np.array_equal(col[perm], wo.rows_of(re_t)[0])
    s = np.concatenate([[0], re_t[:-1]]).astype(np.int64)
    for v in range(n):
        seg = col_t[s[v]:int(re_t[v])]
        assert (np.diff(seg.astype(np.int64)) >= 0).all()
    if e:
        assert re_t[-1] == re_t[-2]                          # node n - 1 has no out-edge: an empty transposed row
    rng = np.random.RandomState(gi)
    gy, w = rng.randn(n, 5), rng.randn(e)
    np.testing.assert_allclose(wo.forward(re_t, col_t, gy, w[perm]), wo.input_grad(row_end, col, gy, w, n),
                               rtol=1e-12, atol=1e-12)


def test_transpose_of_a_symmetric_sorted_graph_is_itself():
    rng = np.random.RandomState(5)
    n = 40
    a = rng.rand(n, n) < 0.15
    a = a | a.T
    row_end = np.cumsum(a.sum(axis=1)).astype(np.uint64)
    col = np.concatenate([np.nonzero(a[i])[0] for i in range(n)]).astype(np.uint32)
    re_t, col_t, _ = wo.transpose(row_end, col, n)
    assert np.array_equal(re_t, row_end) and np.array_equal(col_t, col)


@pytest.mark.parametrize("gi", range(3))
def test_gcn_edge_weights(gi):
    row_end, col = GRAPHS[gi]
    w = np.random.RandomState(gi).uniform(0.0, 3.0, size=col.shape[0])
    w[::7] = 0.0
    want = wo.gcn_edge_weights(row_end, col, w)
    got = datasets.gcn_edge_weights(row_end, col, w)
    assert got.dtype == np.float32
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=0)
    # all-ones weights on a graph where every source also has in-edges: 1 / sqrt(deg_i deg_j)
    row, _, t = wo.rows_of(row_end)
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    ones = wo.gcn_edge_weights(row_end, col, np.ones(col.shape[0]))
    ok = deg[col] > 0
    np.testing.assert_allclose(ones[ok], 1.0 / np.sqrt(deg[row] * deg[col])[ok], rtol=1e-12)
