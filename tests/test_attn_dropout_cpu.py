"""Attention dropout without a GPU: the numpy restatement of the keep mask (attn_dropout_oracle) pinned to the
oracle's Philox on sampled pairs, its keep fraction, the fp64 attention oracle with a mask against torch autograd of
the same masked function, build_gat(attn_dropout=)'s wiring on a recorder with no product behind it, and the refusals
of a rate outside [0, 1)."""
import math

import numpy as np
import pytest
import torch

import attn_dropout_oracle as ado
import attn_oracle as ao
from opgraph import Recorder
from oracle import oracle
from roc_b200.model import Model, build_gat


# ----------------------------------------------------------------------------------------------------- the mask ---
def test_mask_matches_the_oracle_philox():
    rng = np.random.RandomState(1)
    i = rng.randint(0, 2 ** 32, size=64, dtype=np.uint64).astype(np.uint32)
    j = rng.randint(0, 2 ** 32, size=64, dtype=np.uint64).astype(np.uint32)
    i[:4], j[:4] = [0, 1, 0, 4294967295], [0, 0, 1, 4294967295]
    for rate, seed, step in ((0.6, (7 << 32) | 3, 1), (0.1, 0, 5), (0.999, 2 ** 64 - 1, 2 ** 32 - 1), (0.0, 9, 2)):
        got = ado.keep_bytes(i, j, rate, seed, step)
        t = ado.thresh16(rate)
        for n in range(i.shape[0]):
            w = oracle.philox4x32_10([int(i[n]), int(j[n]), 0, step], [seed & 0xFFFFFFFF, seed >> 32])
            want = 0
            for k in range(8):
                half = (w[k // 2] & 0xFFFF) if k % 2 == 0 else (w[k // 2] >> 16)
                want |= (half >= t) << k
            assert int(got[n]) == want, (rate, seed, step, n)


def test_threshold_is_the_dropout_kernels():
    # T16 = round(rate * 65536) of the fp32 rate, at most 65535 (roc_dropout_fwd)
    for rate, want in ((0.0, 0), (0.5, 32768), (0.6, 39322), (0.1, 6554), (0.9999999, 65535)):
        assert ado.thresh16(rate) == want, rate


def test_keep_fraction_is_within_a_binomial_bound():
    rng = np.random.RandomState(2)
    n = 1 << 17                                   # x 8 lanes = 1,048,576 draws
    i, j = rng.randint(0, 1 << 22, n).astype(np.uint32), rng.randint(0, 1 << 22, n).astype(np.uint32)
    for rate in (0.1, 0.5, 0.6):
        kb = ado.keep_bytes(i, j, rate, 12345, 1)
        kept = int(np.unpackbits(kb).sum())
        p = 1.0 - ado.thresh16(rate) / 65536.0
        draws = 8 * n
        assert abs(kept - p * draws) <= 6 * math.sqrt(draws * p * (1 - p)), (rate, kept / draws, p)


def test_edge_orders_are_the_same_pairs():
    """The reverse-pair order and the transposed order hold the mask of the same pairs as the forward order."""
    row_end = np.array([2, 3, 6], dtype=np.uint64)
    col = np.array([0, 2, 0, 0, 1, 1], dtype=np.uint32)       # row 2 has a duplicate edge 2 <- 1
    fwd = ado.edge_keep(row_end, col, 0.5, 3, 4)
    rev = ado.edge_keep(row_end, col, 0.5, 3, 4, row_is_source=True)
    r, c = ado.edge_pairs(row_end, col)
    assert np.array_equal(fwd, ado.keep_bytes(r, c, 0.5, 3, 4)) and np.array_equal(rev, ado.keep_bytes(c, r, 0.5, 3, 4))
    assert fwd[4] == fwd[5]                                    # duplicates share a mask
    # the transposed CSR: row j lists the destinations of j's out-edges, its mask keyed by (dst <- j)
    order = np.lexsort((np.arange(col.shape[0]), c))
    t_end = np.cumsum(np.bincount(c, minlength=3)).astype(np.uint64)
    t_keep = ado.edge_keep(t_end, r[order].astype(np.uint32), 0.5, 3, 4, row_is_source=True)
    assert np.array_equal(t_keep, fwd[order])


# ---------------------------------------------------------------------------------------------- the fp64 oracle ---
def _sym_graph(n, e, seed):
    rng = np.random.RandomState(seed)
    a = rng.randint(0, n, e)
    b = rng.randint(0, n, e)
    pairs = set(zip(a.tolist(), b.tolist())) | set(zip(b.tolist(), a.tolist())) | {(v, v) for v in range(n)}
    pairs = sorted(pairs)
    row_end = np.cumsum(np.bincount([p[0] for p in pairs], minlength=n)).astype(np.uint64)
    return row_end, np.array([p[1] for p in pairs], dtype=np.uint32)


@pytest.mark.parametrize("heads,f", [(1, 5), (2, 4), (8, 4)])
def test_oracle_with_a_mask_matches_autograd(heads, f):
    n, slope, rate = 60, 0.2, 0.6
    row_end, col = _sym_graph(n, 150, heads)
    h = heads * f
    rng = np.random.RandomState(heads)
    x, s, gy = rng.randn(n, h), rng.randn(n, 2 * heads), rng.randn(n, h)
    m1 = ado.multipliers(ado.edge_keep(row_end, col, rate, 11, 3), heads, rate)
    m2 = ado.multipliers(ado.edge_keep(row_end, col, rate, 11, 3, row_is_source=True), heads, rate)
    out, stats = ado.forward(row_end, col, x, s, heads, slope, m1)
    ig, sg = ado.backward(row_end, col, x, s, out, stats, gy, heads, slope, m1, m2)
    # torch: the same masked function, differentiated
    r, c = (torch.from_numpy(v) for v in ado.edge_pairs(row_end, col))
    xt = torch.from_numpy(x).requires_grad_(True)
    st = torch.from_numpy(s).requires_grad_(True)
    z = st[r, :heads] + st[c, heads:]
    y = torch.where(z > 0, z, slope * z)
    ex = torch.exp(y)
    den = torch.zeros((n, heads), dtype=torch.float64).index_add(0, r, ex)
    a = ex / den[r] * torch.from_numpy(m1)
    msg = (a.unsqueeze(2) * xt[c].reshape(-1, heads, f)).reshape(-1, h)
    o = torch.zeros((n, h), dtype=torch.float64).index_add(0, r, msg)
    (o * torch.from_numpy(gy)).sum().backward()
    assert np.allclose(out, o.detach().numpy(), rtol=1e-12, atol=1e-12)
    assert np.allclose(ig, xt.grad.numpy(), rtol=1e-10, atol=1e-12)
    assert np.allclose(sg, st.grad.numpy(), rtol=1e-10, atol=1e-12)
    # with an all-keep mask of scale 1 it is attn_oracle's attention without dropout
    ones = np.ones((col.shape[0], heads))
    o0, st0 = ao.forward(row_end, col, x, s, heads, slope)
    o1, st1 = ado.forward(row_end, col, x, s, heads, slope, ones)
    assert np.allclose(o1, o0, rtol=1e-13, atol=1e-13) and np.array_equal(st1, st0)
    for a, b in zip(ado.backward(row_end, col, x, s, o0, st0, gy, heads, slope, ones, ones),
                    ao.backward(row_end, col, x, s, o0, st0, gy, heads, slope)):
        assert np.allclose(a, b, rtol=1e-12, atol=1e-12)
    assert np.allclose(ado.backward(row_end, col, x, s, o0, st0, gy, heads, slope, ones, ones, magnitude=True)[1],
                       ao.score_grad_magnitude(row_end, col, x, s, o0, st0, gy, heads, slope), rtol=1e-12, atol=1e-12)


# --------------------------------------------------------------------------------------------- the Python API ---
def test_build_gat_wiring_with_attn_dropout():
    layers = [24, 16, 32, 12]
    plain, ir = Recorder(None), Recorder(None)
    build_gat(plain, layers, 0.6, heads=[2, 8], scores="per_head", activation="elu")
    h = build_gat(ir, layers, 0.6, heads=[2, 8], scores="per_head", activation="elu", attn_dropout=0.6)
    gathers = [n for n in ir.nodes if n["kind"] == "attention_gather"]
    assert [n["out"] for n in gathers] == h["attn"]
    for g in gathers:
        assert g["attrs"]["dropout"] == 0.6 and g["attrs"]["key"] == g["layer"]     # seed 0, the op's position
    strip = lambda nodes: [(n["kind"], n["ins"], n["out"], {k: v for k, v in n["attrs"].items() if k != "dropout"})
                           for n in nodes]
    assert strip(ir.nodes) == strip(plain.nodes)
    assert all(n["attrs"]["dropout"] == 0.0 for n in plain.nodes if n["kind"] == "attention_gather")


def test_build_gat_defaults_call_attention_gather_as_before():
    """With attn_dropout = 0 the builder calls attention_gather with today's four arguments, so a recorder that knows
    only those builds the same model."""
    calls = []

    class Plain(Recorder):
        def attention_gather(self, t, scores, heads=1, negative_slope=0.2):
            calls.append((heads, negative_slope))
            return super().attention_gather(t, scores, heads, negative_slope)

    build_gat(Plain(None), [24, 16, 12], 0.5, heads=4, attn_dropout=0.0)
    build_gat(Plain(None), [24, 16, 12], 0.5, heads=4)
    assert calls == [(4, 0.2), (1, 0.2)] * 2


@pytest.mark.parametrize("rate", [-0.1, 1.0, 1.5, float("nan")])
def test_rates_outside_the_unit_interval_are_refused(rate):
    with pytest.raises(ValueError):
        build_gat(Recorder(None), [24, 16, 12], 0.5, heads=2, attn_dropout=rate)
    m = Model.__new__(Model)          # refused before the product is touched
    with pytest.raises(ValueError):
        m.attention_gather(0, 1, 2, 0.2, dropout=rate)
