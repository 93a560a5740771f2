"""The max / min ScatterGather definition (tests/minmax_oracle.c, its forward and backward) against torch's
scatter_reduce and autograd.  The reference has no max aggregation; these tests pin the oracle that the GPU suite
then holds the product's kernels to."""
import numpy as np
import pytest
import torch

import minmax_oracle as mmo
from oracle import oracle
from roc_b200 import datasets

NAMES = {mmo.AGGR_MAX: "amax", mmo.AGGR_MIN: "amin"}


def graph(kind):
    if kind == "uniform":
        re, col = datasets.uniform_graph(1000, 4500, seed=1)
    else:
        re, col = datasets.rmat_graph(12, 40000, seed=3)        # hub rows of degree >> 64
    return re.numpy().astype(np.uint64), col.numpy().astype(np.uint32)


def dst_of(row_end):
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    return np.repeat(np.arange(row_end.shape[0]), deg)


def torch_reduce(row_end, col, x, aggr):
    n, h = row_end.shape[0], x.shape[1]
    idx = torch.from_numpy(dst_of(row_end)).unsqueeze(1).expand(-1, h)
    src = torch.from_numpy(x)[torch.from_numpy(col.astype(np.int64))]
    return torch.zeros((n, h), dtype=torch.float32).scatter_reduce(0, idx, src, NAMES[aggr], include_self=False)


def first_extreme(row_end, col, x, aggr):
    """numpy: per row and feature, the source of the first edge holding the max / min (no NaN in x)."""
    n, h = row_end.shape[0], x.shape[1]
    arg = np.full((n, h), mmo.NOARG, dtype=np.uint32)
    s = 0
    for v in range(n):
        e = int(row_end[v])
        if e > s:
            vals = x[col[s:e]]
            k = np.argmax(vals, axis=0) if aggr == mmo.AGGR_MAX else np.argmin(vals, axis=0)
            arg[v] = col[s:e][k]
        s = e
    return arg


@pytest.mark.parametrize("kind", ["uniform", "rmat"])
@pytest.mark.parametrize("h", [1, 7, 64])
@pytest.mark.parametrize("aggr", [mmo.AGGR_MAX, mmo.AGGR_MIN])
def test_minmax_matches_torch_scatter_reduce(kind, h, aggr):
    row_end, col = graph(kind)
    n = row_end.shape[0]
    x = np.random.RandomState(h).randn(n, h).astype(np.float32)
    out, arg = mmo.forward(0, n - 1, 0, row_end, col, x, aggr)
    assert np.array_equal(out, torch_reduce(row_end, col, x, aggr).numpy()), "values must be exact"
    assert np.array_equal(arg, first_extreme(row_end, col, x, aggr))


def test_minmax_rules_on_a_hand_made_graph():
    # row 0: sources 1, 2, 3 with the max tied between 1 and 3 and the min tied between 2 and 3
    # row 1: all three sources equal            row 2: a NaN from source 2 after a finite value
    # row 3: -inf only                          row 4: no in-edge
    row_end = np.array([3, 6, 8, 9, 9], dtype=np.uint64)
    col = np.array([1, 2, 3, 0, 1, 4, 0, 2, 3], dtype=np.uint32)
    x = np.zeros((5, 2), dtype=np.float32)
    x[0] = [5, 5]; x[1] = [5, 5]; x[2] = [np.nan, 1]; x[3] = [-np.inf, 5]; x[4] = [5, 5]
    x[1, 1], x[2, 1], x[3, 1] = 7, -2, 7
    mx, amx = mmo.forward(0, 4, 0, row_end, col, x, mmo.AGGR_MAX)
    mn, amn = mmo.forward(0, 4, 0, row_end, col, x, mmo.AGGR_MIN)
    # row 0, feature 1: values 7, -2, 7 -> max 7 first at source 1; min -2 at source 2
    assert mx[0, 1] == 7 and amx[0, 1] == 1 and mn[0, 1] == -2 and amn[0, 1] == 2
    # row 0, feature 0: values 5, NaN, -inf -> NaN wins for both max and min (it propagates), taken at source 2
    assert np.isnan(mx[0, 0]) and amx[0, 0] == 2 and np.isnan(mn[0, 0]) and amn[0, 0] == 2
    # row 1: sources 0, 1, 4 all 5 in feature 0 -> the first edge's source
    assert mx[1, 0] == 5 and amx[1, 0] == 0 and mn[1, 0] == 5 and amn[1, 0] == 0
    # row 2: sources 0 (5) then 2 (NaN) -> NaN replaces the finite value
    assert np.isnan(mx[2, 0]) and amx[2, 0] == 2
    # row 3: -inf only -> -inf with the first (only) edge's source, not the empty-row marker
    assert mx[3, 0] == -np.inf and amx[3, 0] == 3 and mn[3, 0] == -np.inf
    # row 4: degree 0 -> 0 and 0xFFFFFFFF
    assert (mx[4] == 0).all() and (amx[4] == mmo.NOARG).all() and (amn[4] == mmo.NOARG).all()
    # a later NaN never replaces an earlier NaN: row 0 feature 0 has one NaN; two NaNs keep the first
    x2 = x.copy(); x2[1, 0] = np.nan
    _, a2 = mmo.forward(0, 4, 0, row_end, col, x2, mmo.AGGR_MAX)
    assert a2[0, 0] == 1


@pytest.mark.parametrize("kind", ["uniform", "rmat"])
@pytest.mark.parametrize("aggr", [mmo.AGGR_MAX, mmo.AGGR_MIN])
def test_minmax_backward_matches_torch_autograd(kind, aggr):
    """On a symmetric graph without duplicate edges and with tie-free inputs, torch's gradient of scatter_reduce
    (which splits a tie evenly) and the first-occurrence rule agree."""
    row_end, col = graph(kind)
    n, h = row_end.shape[0], 16
    rng = np.random.RandomState(5)
    # distinct values, none equal to the 0 torch starts from (its backward would split a tie with that, too)
    x = (rng.permutation(n * h).reshape(n, h).astype(np.float32) + 1) / (n * h)
    gy = rng.randn(n, h).astype(np.float32)
    xt = torch.from_numpy(x.astype(np.float64)).requires_grad_(True)
    idx = torch.from_numpy(dst_of(row_end)).unsqueeze(1).expand(-1, h)
    y = torch.zeros((n, h), dtype=torch.float64).scatter_reduce(0, idx, xt[torch.from_numpy(col.astype(np.int64))],
                                                                 NAMES[aggr], include_self=False)
    (y * torch.from_numpy(gy.astype(np.float64))).sum().backward()
    _, arg = mmo.forward(0, n - 1, 0, row_end, col, x, aggr)
    got = mmo.backward(0, n - 1, 0, row_end, col, gy, arg)
    assert np.allclose(got, xt.grad.numpy(), rtol=1e-6, atol=1e-6)
    # fp32 accumulation in edge order agrees to rounding
    got32 = mmo.backward(0, n - 1, 0, row_end, col, gy, arg, acc64=False)
    assert np.allclose(got32, got, rtol=1e-5, atol=1e-6)


def test_minmax_backward_sends_a_tied_gradient_to_the_first_source_only():
    # symmetric 3-vertex graph with self loops; every feature value equal -> every row picks its first source
    row_end = np.array([3, 6, 9], dtype=np.uint64)
    col = np.array([0, 1, 2] * 3, dtype=np.uint32)
    x = np.ones((3, 2), dtype=np.float32)
    _, arg = mmo.forward(0, 2, 0, row_end, col, x, mmo.AGGR_MAX)
    assert (arg == 0).all()
    gy = np.array([[1, 10], [2, 20], [4, 40]], dtype=np.float32)
    g = mmo.backward(0, 2, 0, row_end, col, gy, arg)
    assert np.array_equal(g, np.array([[7, 70], [0, 0], [0, 0]], dtype=np.float32))


def test_minmax_partition_slices_with_global_ids():
    row_end, col = graph("rmat")
    n, h = row_end.shape[0], 8
    x = np.random.RandomState(3).randn(n, h).astype(np.float32)
    gy = np.random.RandomState(4).randn(n, h).astype(np.float32)
    out, arg = mmo.forward(0, n - 1, 0, row_end, col, x, mmo.AGGR_MAX)
    gx = mmo.backward(0, n - 1, 0, row_end, col, gy, arg)
    k, vb, eb = oracle.partition(row_end, 3)
    for c in range(k):
        rl, rr, cl, cr = int(vb[c, 0]), int(vb[c, 1]), int(eb[c, 0]), int(eb[c, 1])
        o, a = mmo.forward(rl, rr, cl, row_end[rl:rr + 1], col[cl:cr + 1], x, mmo.AGGR_MAX)
        assert np.array_equal(o, out[rl:rr + 1]) and np.array_equal(a, arg[rl:rr + 1])
        g = mmo.backward(rl, rr, cl, row_end[rl:rr + 1], col[cl:cr + 1], gy, arg, self_base=rl)
        assert np.array_equal(g, gx[rl:rr + 1])
