"""Attention dropout's keep mask (include/roc_b200.h, roc_sg_attn_forward_dropout_planned) restated in vectorised
numpy: keep(i<-j,k) = 16-bit lane k of Philox4x32-10(counter = {i, j, 0, step}, key = {seed lo, seed hi}) >= T16,
lane k the low (k even) or high (k odd) half of word k // 2; and the attention aggregation with that dropout in fp64,
on attn_oracle's helpers.  No code shared with the product."""
import numpy as np

import attn_oracle as ao

M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 of uint32 arrays c0..c3 under the key (k0, k1) -> four uint32 arrays."""
    c = [np.asarray(v, dtype=np.uint32) for v in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0 = c[0].astype(np.uint64) * np.uint64(0xD2511F53)
        p1 = c[2].astype(np.uint64) * np.uint64(0xCD9E8D57)
        hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & M32).astype(np.uint32)
        hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & M32).astype(np.uint32)
        c = [hi1 ^ c[1] ^ np.uint32(k0), lo1, hi0 ^ c[3] ^ np.uint32(k1), lo0]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M32, (k1 + np.uint64(0xBB67AE85)) & M32
    return c


def thresh16(rate):
    t = float(np.float32(rate)) * 65536.0 + 0.5
    return 65535 if t >= 65535.0 else int(t)


def keep_bytes(i, j, rate, seed, step):
    """uint8 per pair (i <- j): bit k = keep(i<-j,k), all 8 lanes."""
    i, j = np.asarray(i, dtype=np.uint32), np.asarray(j, dtype=np.uint32)
    w = philox4x32_10(i, j, np.zeros_like(i), np.full_like(i, step), seed & 0xFFFFFFFF, seed >> 32)
    t = np.uint32(thresh16(rate))
    out = np.zeros(i.shape, dtype=np.uint8)
    for k in range(8):
        half = (w[k // 2] & np.uint32(0xFFFF)) if k % 2 == 0 else (w[k // 2] >> np.uint32(16))
        out |= ((half >= t).astype(np.uint8) << np.uint8(k))
    return out


def edge_pairs(row_end, col, col_left=0, self_base=0):
    """(row id, col id) of every edge in CSR order."""
    re = np.asarray(row_end, dtype=np.int64) - int(col_left)
    deg = np.diff(np.concatenate([[0], re]))
    r = np.repeat(np.arange(re.shape[0], dtype=np.int64), deg) + int(self_base)
    return r, np.asarray(col, dtype=np.int64)[:r.shape[0]]


def edge_keep(row_end, col, rate, seed, step, col_left=0, self_base=0, row_is_source=False):
    """roc_sg_attn_keep_mask restated: the keep byte of every edge in CSR order."""
    r, c = edge_pairs(row_end, col, col_left, self_base)
    return keep_bytes(c, r, rate, seed, step) if row_is_source else keep_bytes(r, c, rate, seed, step)


def multipliers(keep, heads, rate):
    """[E][heads] M = keep ? s : 0 with s = 1.0f / (1.0f - rate) in fp32, as fp64."""
    s = float(np.float32(1.0) / (np.float32(1.0) - np.float32(rate)))
    bits = (np.asarray(keep, dtype=np.uint8)[:, None] >> np.arange(heads, dtype=np.uint8)[None, :]) & 1
    return bits.astype(np.float64) * s


# ------------------------------------------------------------- the attention aggregation with dropout, fp64 ---
# attn_oracle's forward / backward with attention dropout: `drop` is M(i<-j,k) per edge in CSR order [E][heads]
# (multipliers above), `drop_rev` the same for the reverse pairs (j <- i).  m and Z stay the undropped softmax's; the
# backward's D is over the dropped output `out`.  Rows, ids and indexing are attn_oracle's.
def forward(row_end, col, x, s, heads, slope, drop, self_base=0, col_left=0):
    """-> out [nloc][H], stats [nloc][2*heads] (m | 1/Z), fp64."""
    x = np.asarray(x, dtype=np.float64)
    s = np.asarray(s, dtype=np.float64)
    re, deg, r, j, i = ao._edges(row_end, col, col_left, self_base)
    nloc = re.shape[0]
    y = ao._leaky(s[i, :heads] + s[j, heads:2 * heads], slope)
    m = np.full((nloc, heads), -np.inf)
    np.maximum.at(m, r, y)
    m[deg == 0] = 0.0
    ex = np.exp(y - m[r])
    Z = ao._row_sum(r, ex, nloc)
    iz = np.where(deg[:, None] > 0, 1.0 / np.where(Z > 0, Z, 1.0), 0.0)
    out = ao._weighted_gather(r, j, ex * iz[r] * drop, nloc, x, heads, x.shape[0])
    return out, np.concatenate([m, iz], axis=1)


def _alpha(s, stats, dst, src, heads, slope):
    m, iz = stats[:, :heads], stats[:, heads:2 * heads]
    z = s[dst, :heads] + s[src, heads:2 * heads]
    a = np.where(iz[dst] == 0, 0.0, np.exp(ao._leaky(z, slope) - m[dst]) * iz[dst])
    return a, np.where(z > 0, 1.0, slope)


def backward(row_end, col, x, s, out, stats, gy, heads, slope, drop, drop_rev, self_base=0, col_left=0,
             magnitude=False):
    """-> in_grad [nloc][H], score_grad [nloc][2*heads] (d s_dst | d s_src), fp64, as attn_oracle.backward (the
    gathers over the same CSR).  magnitude: the score gradients with every term replaced by its magnitude,
    sum_e a |l| (M sum_f |G X| + |D|), the scale of their fp32 rounding (attn_oracle.score_grad_magnitude)."""
    x, s, out, stats, gy = (np.asarray(v, dtype=np.float64) for v in (x, s, out, stats, gy))
    if magnitude:
        x, out, gy = np.abs(x), np.abs(out), np.abs(gy)
    re, deg, r, j, i = ao._edges(row_end, col, col_left, self_base)
    nloc = re.shape[0]
    F = x.shape[1] // heads
    D = (gy * out).reshape(gy.shape[0], heads, F).sum(-1)
    sign = 1.0 if magnitude else -1.0
    a1, l1 = _alpha(s, stats, i, j, heads, slope)
    a2, l2 = _alpha(s, stats, j, i, heads, slope)
    if magnitude:
        l1, l2 = np.abs(l1), np.abs(l2)
    dz1 = a1 * (drop * ao._per_head_dot(gy, i, x, j, heads) + sign * D[i]) * l1
    dz2 = a2 * (drop_rev * ao._per_head_dot(gy, j, x, i, heads) + sign * D[j]) * l2
    in_grad = ao._weighted_gather(r, j, a2 * drop_rev, nloc, gy, heads, gy.shape[0])
    return in_grad, np.concatenate([ao._row_sum(r, dz1, nloc), ao._row_sum(r, dz2, nloc)], axis=1)
