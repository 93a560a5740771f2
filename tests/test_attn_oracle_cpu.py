"""The attention aggregation's definition (tests/attn_oracle.py) against torch fp64 autograd of the same function:
the forward everywhere, all three backward outputs on symmetric graphs (where the CSR gathers are the true
adjoint), and the destination-score gradient also on a graph that is not symmetric.  The GPU suite then holds the
product's kernels to this oracle."""
import numpy as np
import pytest
import torch

import attn_oracle as ao
from roc_b200 import datasets
from sg_graphs import graph as sg_graph

SLOPE = 0.2


def graph(kind):
    if kind == "uniform":
        re, col = datasets.uniform_graph(1000, 4500, seed=1)
    elif kind == "rmat":
        re, col = datasets.rmat_graph(10, 8000, seed=3)          # symmetric, hub rows of degree >> 64
    else:
        return sg_graph(kind)
    return re.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


def torch_attention(row_end, col, x, s, heads, slope):
    """out[r] = sum_e softmax_e(LeakyReLU(s_dst[r] + s_src[col[e]])) x[col[e]] per head, from edge lists."""
    n = row_end.shape[0]
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dst = torch.from_numpy(np.repeat(np.arange(n), deg))
    src = torch.from_numpy(col.astype(np.int64))
    z = s[dst, :heads] + s[src, heads:]
    y = torch.nn.functional.leaky_relu(z, slope)
    m = torch.full((n, heads), -np.inf, dtype=torch.float64).scatter_reduce(
        0, dst.unsqueeze(1).expand(-1, heads), y, "amax", include_self=True).detach()
    ex = torch.exp(y - m[dst])
    Z = torch.zeros((n, heads), dtype=torch.float64).index_add(0, dst, ex)
    a = ex / Z[dst]
    F = x.shape[1] // heads
    msg = (a.unsqueeze(2) * x[src].view(-1, heads, F)).view(-1, x.shape[1])
    return torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, msg)


def case(kind, h, heads, seed):
    row_end, col = graph(kind)
    n = row_end.shape[0]
    rng = np.random.RandomState(seed)
    return row_end, col, rng.randn(n, h), rng.randn(n, 2 * heads), rng.randn(n, h)


def autograd(row_end, col, x, s, g, heads):
    xt = torch.from_numpy(x).requires_grad_(True)
    st = torch.from_numpy(s).requires_grad_(True)
    out = torch_attention(row_end, col, xt, st, heads, SLOPE)
    gx, gs = torch.autograd.grad(out, (xt, st), torch.from_numpy(g))
    return out.detach().numpy(), gx.numpy(), gs.numpy()


def close(a, b, what):
    scale = max(np.abs(b).max(), 1e-300)
    assert np.abs(a - b).max() <= 1e-10 * scale, "%s: max err %.3e (scale %.3e)" % (what, np.abs(a - b).max(), scale)


@pytest.mark.parametrize("kind", ["uniform", "rmat"])
@pytest.mark.parametrize("heads,h", [(1, 7), (1, 16), (4, 16), (4, 32)])
def test_oracle_matches_torch_autograd_on_symmetric_graphs(kind, heads, h):
    row_end, col, x, s, g = case(kind, h, heads, seed=h + heads)
    out, stats = ao.forward(row_end, col, x, s, heads, SLOPE)
    want, gx, gs = autograd(row_end, col, x, s, g, heads)
    close(out, want, "forward")
    in_grad, score_grad = ao.backward(row_end, col, x, s, out, stats, g, heads, SLOPE)
    close(in_grad, gx, "input gradient")
    close(score_grad[:, :heads], gs[:, :heads], "destination-score gradient")
    close(score_grad[:, heads:], gs[:, heads:], "source-score gradient")


@pytest.mark.parametrize("heads,h", [(1, 5), (2, 8)])
def test_destination_score_gradient_is_exact_on_a_ragged_graph(heads, h):
    """ragged is not symmetric and has rows of degree 0: only d s_dst is the true gradient there."""
    row_end, col, x, s, g = case("ragged", h, heads, seed=3)
    out, stats = ao.forward(row_end, col, x, s, heads, SLOPE)
    want, _, gs = autograd(row_end, col, x, s, g, heads)
    close(out, want, "forward")
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    assert (deg == 0).any()
    assert np.all(out[deg == 0] == 0) and np.all(stats[deg == 0] == 0), "a row of degree 0 gets 0, m = 0, 1/Z = 0"
    _, score_grad = ao.backward(row_end, col, x, s, out, stats, g, heads, SLOPE)
    close(score_grad[:, :heads], gs[:, :heads], "destination-score gradient")


def test_stats_hold_the_row_max_and_inverse_partition_function():
    row_end, col, x, s, _ = case("uniform", 4, 2, seed=5)
    _, stats = ao.forward(row_end, col, x, s, 2, SLOPE)
    v, e0 = 17, int(row_end[16])
    srcs = col[e0:int(row_end[v])].astype(np.int64)
    y = s[v, :2] + s[srcs, 2:]
    y = np.where(y > 0, y, SLOPE * y)
    assert np.allclose(stats[v, :2], y.max(0), rtol=0, atol=0)
    assert np.allclose(stats[v, 2:], 1.0 / np.exp(y - y.max(0)).sum(0), rtol=1e-14)
