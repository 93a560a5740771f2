"""The fp64 references of the exact backwards (exact_oracle.py) against torch autograd, on directed graphs with
duplicate edges, rows of in-degree 0 and nodes with no out-edge.  The GPU tests compare the kernels with these
references, so here they are checked once against an independent derivation of the gradient."""
import numpy as np
import torch

import attn_oracle as ao
import exact_oracle as xo


def directed_multigraph(n=60, e=400, seed=5):
    """(row_end, col, dst): sorted by destination, sources in random order within a row."""
    rng = np.random.RandomState(seed)
    dst = rng.randint(0, n - 4, size=e)                   # the last four rows have in-degree 0
    src = rng.randint(3, n, size=e)                       # nodes 0..2 have no out-edge
    src[1::5] = src[0::5][:src[1::5].shape[0]]            # duplicate edges
    dst[1::5] = dst[0::5][:dst[1::5].shape[0]]
    order = np.argsort(dst, kind="stable")
    dst, src = dst[order], src[order]
    re_ = np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64)
    return re_, src.astype(np.uint32), dst


def check_graph(re_, col, dst, n):
    pairs = dst.astype(np.int64) * n + col
    assert np.unique(pairs).shape[0] < pairs.shape[0], "no duplicate edge"
    assert (np.diff(np.concatenate([[0], re_.astype(np.int64)])) == 0).any(), "no row of in-degree 0"
    assert np.bincount(col.astype(np.int64), minlength=n).min() == 0, "no node without an out-edge"


def test_sum_backward_is_autograds():
    re_, col, dst = directed_multigraph()
    n = re_.shape[0]
    check_graph(re_, col, dst, n)
    rng = np.random.RandomState(1)
    x = torch.tensor(rng.randn(n, 7), dtype=torch.float64, requires_grad=True)
    gy = rng.randn(n, 7)
    _, deg = xo.edges(re_)
    src, d = torch.from_numpy(col.astype(np.int64)), torch.from_numpy(dst)
    # without and with the in-degree norm in front (the model's indegree_norm -> scatter_gather)
    for norm in (False, True):
        scale = torch.from_numpy(np.where(deg > 0, 1.0 / np.sqrt(np.maximum(deg, 1)), 0.0))[:, None]
        xin = x * scale if norm else x
        y = torch.zeros(n, 7, dtype=torch.float64).index_add(0, d, xin[src])
        (g,) = torch.autograd.grad(y, x, torch.from_numpy(gy))
        want = xo.sum_backward(re_, col, gy, n) * (scale.numpy() if norm else 1.0)
        assert np.allclose(g.numpy(), want, rtol=1e-12, atol=1e-12)
    # Q1 (the gather over the same CSR) is a different function here
    assert not np.allclose(xo.adjacency(re_, col, n) @ gy, xo.sum_backward(re_, col, gy, n))


def test_sum_epilogue_is_the_fp32_divide():
    re_, col, _ = directed_multigraph(seed=6)
    n = re_.shape[0]
    gy = (np.random.RandomState(2).randint(-64, 65, size=(n, 5)) / 16.0).astype(np.float32)
    s = xo.sum_backward(re_, col, gy, n).astype(np.float32)
    _, deg = xo.edges(re_)
    with np.errstate(divide="ignore", invalid="ignore"):
        normed = s / np.sqrt(deg.astype(np.float32))[:, None]
    got = xo.sum_backward_epi(re_, col, gy, n, xo.NORM | xo.RELU)
    assert np.array_equal(got, np.maximum(normed, np.float32(0)), equal_nan=True)
    assert np.isnan(got).any() or np.isinf(got).any()      # rows of in-degree 0 divide by 0, as roc_indegree_norm does


def test_minmax_backward_is_autograds():
    re_, col, dst = directed_multigraph(seed=7)
    n = re_.shape[0]
    rng = np.random.RandomState(3)
    xv = rng.randn(n, 6)                                  # no ties between distinct sources
    gy = rng.randn(n, 6)
    src, d = torch.from_numpy(col.astype(np.int64)), torch.from_numpy(dst)
    for aggr, how in ((1, "amax"), (2, "amin")):
        x = torch.tensor(xv, requires_grad=True)
        y = torch.zeros(n, 6, dtype=torch.float64).scatter_reduce(0, d[:, None].expand(-1, 6), x[src], how,
                                                                   include_self=False)
        (g,) = torch.autograd.grad(y, x, torch.from_numpy(gy))
        out, arg = xo.minmax_forward(re_, col, xv, aggr)
        assert np.array_equal(out, y.detach().numpy())
        # autograd splits a tie between a duplicate edge's twins, whose halves reach the same source: the whole once
        assert np.allclose(g.numpy(), xo.minmax_backward(re_, col, gy, arg, n), rtol=1e-12, atol=1e-12)
        # the gather over the same CSR counts a duplicate twice and sends gradients along reversed edges
        q1 = np.zeros((n, 6))
        for r in range(n):
            for e in range(int(re_[r - 1]) if r else 0, int(re_[r])):
                q1[r] += np.where(arg[col[e]] == r, gy[col[e]], 0.0)
        assert not np.allclose(q1, g.numpy())


def attn_torch(re_, col, dst, x, s, heads, slope):
    """The attention forward in torch fp64 on the edge list: the per-row softmax of LeakyReLU(s_dst + s_src) per
    head, weighting the sources' features."""
    n, h = x.shape
    F = h // heads
    i, j = torch.from_numpy(dst), torch.from_numpy(col.astype(np.int64))
    z = s[i, :heads] + s[j, heads:]
    y = torch.where(z > 0, z, slope * z)
    m = torch.full((n, heads), -np.inf, dtype=torch.float64).scatter_reduce(0, i[:, None].expand(-1, heads), y, "amax")
    ex = torch.exp(y - m.detach()[i])
    Z = torch.zeros(n, heads, dtype=torch.float64).index_add(0, i, ex)
    a = ex / Z[i]
    v = (a[:, :, None] * x[j].reshape(-1, heads, F)).reshape(-1, h)
    return torch.zeros(n, h, dtype=torch.float64).index_add(0, i, v)


def test_attn_backward_is_autograds():
    re_, col, dst = directed_multigraph(seed=8)
    n = re_.shape[0]
    rng = np.random.RandomState(4)
    for heads, h in ((1, 6), (2, 8), (4, 16)):
        xv, sv, gy = rng.randn(n, h), rng.randn(n, 2 * heads), rng.randn(n, h)
        x = torch.tensor(xv, requires_grad=True)
        s = torch.tensor(sv, requires_grad=True)
        y = attn_torch(re_, col, dst, x, s, heads, 0.2)
        gx, gs = torch.autograd.grad(y, (x, s), torch.from_numpy(gy))
        out, stats = ao.forward(re_, col, xv, sv, heads, 0.2)
        assert np.allclose(out, y.detach().numpy(), rtol=1e-12, atol=1e-12)
        ig, sg = xo.attn_backward(re_, col, xv, sv, out, stats, gy, heads, 0.2)
        assert np.allclose(ig, gx.numpy(), rtol=1e-10, atol=1e-12)
        assert np.allclose(sg, gs.numpy(), rtol=1e-10, atol=1e-12)
        # Q1 gets d s_dst right and the rest wrong
        qig, qsg = ao.backward(re_, col, xv, sv, out, stats, gy, heads, 0.2)
        assert np.allclose(qsg[:, :heads], gs.numpy()[:, :heads], rtol=1e-10, atol=1e-12)
        assert not np.allclose(qig, gx.numpy()) and not np.allclose(qsg[:, heads:], gs.numpy()[:, heads:])
