"""The element-wise error bound the Linear GEMM tests hold every kernel to, the data families they feed it, and a
numpy emulation of the tensor-core kernels' 3xTF32 arithmetic that calibrates the bound without a GPU
(tests/test_tf32_bound_cpu.py).

For an fp32 product C = A B^T with K terms per element, the fp64 reference ref_ij = sum_k a_ik b_jk and

    |got_ij - ref_ij| <= C_BOUND * (2^-20 * s_ij + 2^-21 * t_ij),
    s_ij = sqrt(sum_k (a_ik b_jk)^2),   t_ij = sum_g |P_ij(g)|,   P_ij(g) = sum_{k < 8 (g + 1)} a_ik b_jk.

The first term covers the hi / lo split of 3xTF32: the dropped lo*lo product and the truncation of lo to TF32 are
~2^-22 of each product, with random signs.  The second covers fp32 accumulation.  The tensor cores round each of the
three MMAs of a k8 step into the accumulator, each time by up to 2^-23 of the partial sum P(g).  On the H100 that
rounding truncates: with same-sign products the errors add up instead of cancelling, so they grow like K rather than
sqrt(K).  The SIMT kernels round to nearest after each of 8 fused multiply-adds per k8 step, which is 8 * 2^-24 of
the same partial sums.  t is the sum of |P| over the k8 steps, in the order the kernels run them.  With C_BOUND = 4,
the emulated 3xTF32 (truncating) and plain fp32 GEMMs stay under a quarter of the bound on every family.  Dropping any
one of the three MMAs overshoots it at least fourfold.  test_tf32_bound_cpu.py checks both.

dW accumulates K = the row count in split-K ranges; RefAccumulator(split=...) follows those ranges (see there).  The
power to reject a lost MMA depends on the range length, not on K: it is calibrated for ranges of 416 rows.  At
thousands of rows per range, a correct kernel's truncation comes within the bound's slack of a lost lo term.

A bound of the form C * (2^-20 s + sqrt(K) 2^-24 sum_k |a_ik b_jk|) models round-to-nearest accumulation.  At 602
terms of the same sign, the H100 exceeds it by 1.9x at C = 5, because its accumulation truncates.
"""
import math

import numpy as np
import torch

C_BOUND = 4.0
FAMILIES = ("random_sign", "positive", "scaled_rows", "zeros")


def family_data(family, rows, cols, gen, role, device):
    """fp32 [rows][cols] operand of one data family (torch, seeded by `gen`, which lives on `device`).
    role "a": the streaming operand (X or dY, one row per vertex); role "b": the weight.
      random_sign  standard normal
      positive     uniform [0, 1) in both operands: every product has the same sign
      scaled_rows  standard normal, each row of the streaming operand scaled by 2^e, e uniform in [-60, 60]
      zeros        standard normal with half the elements exactly 0, and every 7th streaming row all 0"""
    kw = dict(generator=gen, device=device, dtype=torch.float32)
    if family == "positive":
        return torch.rand((rows, cols), **kw)
    t = torch.randn((rows, cols), **kw)
    if family == "scaled_rows" and role == "a":
        e = torch.randint(-60, 61, (rows, 1), generator=gen, device=device).to(torch.float32)
        t = t * torch.exp2(e)
    elif family == "zeros":
        t = t * (torch.rand((rows, cols), **kw) < 0.5)
        if role == "a":
            t[::7] = 0.0
    elif family not in ("random_sign", "scaled_rows"):
        raise KeyError(family)
    return t


class RefAccumulator:
    """fp64 A B^T of fp32 operands and its bound, accumulated over chunks of K that start at multiples of 8.

    split = the K range each split-K partial sums (the dW kernels: vertices per split; a multiple of 8), None = one
    range.  The kernels accumulate each range on its own, then add the fp32 partials in range order.  So the partial
    sums P of the bound restart at every range, and the ranges combine as their errors do.  A range's error has a
    systematic part that follows the sign of its partial sums, u_z = sum_g P_z(g): same-sign data truncates the same
    way in every range.  Its remaining part is independent between ranges, so the ranges' sums t_z = sum_g |P_z(g)|
    add in quadrature.  The bound's accumulation term is max(|sum_z u_z|, sqrt(sum_z t_z^2)), which is t for a single
    range.  The reduction of the partials adds 2^-24 of each running sum S_z it rounds (r = sum_{z >= 1} |S_z|)."""

    def __init__(self, split=None):
        assert split is None or split % 8 == 0
        self.split_groups = None if split is None else split // 8
        self.p = self.ssq = None
        self.k = self.groups = 0

    def _close(self):
        """end of a split-K range: fold its partial sums into the running totals"""
        if self.in_range == 0:
            return
        self.tq += self.t * self.t
        self.u_all += self.u
        if self.ranges > 0:
            self.s = self.s + self.p
            self.r += self.s.abs()
        else:
            self.s = self.p.clone()
        self.ranges += 1
        self.p.zero_()
        self.t.zero_()
        self.u.zero_()
        self.in_range = 0

    def add(self, a, b):
        a, b = a.double(), b.double()
        k = a.shape[1]
        assert self.k % 8 == 0, "chunks of K must start at multiples of 8"
        if k % 8:
            a = torch.nn.functional.pad(a, (0, 8 - k % 8))
            b = torch.nn.functional.pad(b, (0, 8 - k % 8))
        m, n, groups = a.shape[0], b.shape[0], a.shape[1] // 8
        if self.p is None:
            z = a.new_zeros((m, n))
            self.p, self.ssq, self.t, self.u, self.tq, self.u_all, self.r = (z.clone() for _ in range(7))
            self.s = z.clone()
            self.ranges = self.in_range = 0
        self.ssq += (a * a) @ (b * b).T
        ag = a.reshape(m, groups, 8).permute(1, 0, 2)       # [groups][m][8]
        bg = b.reshape(n, groups, 8).permute(1, 2, 0)       # [groups][8][n]
        step = max(1, (1 << 29) // (8 * m * n))             # ~512 MB of per-group partial sums at a time
        g0 = 0
        while g0 < groups:
            g1 = min(groups, g0 + step)
            if self.split_groups is not None:               # never cross the end of a split-K range
                g1 = min(g1, g0 + self.split_groups - self.in_range)
            ps = torch.cumsum(torch.bmm(ag[g0:g1], bg[g0:g1]), 0) + self.p
            self.t += ps.abs().sum(0)
            self.u += ps.sum(0)
            self.p = ps[-1].clone()
            self.in_range += g1 - g0
            if self.split_groups is not None and self.in_range == self.split_groups:
                self._close()
            g0 = g1
        self.k += k
        return self

    def result(self):
        """(ref, bound), both fp64 [rows of A][rows of B]"""
        self._close()
        acc = torch.maximum(self.u_all.abs(), self.tq.sqrt())
        return self.s, bound(self.ssq.sqrt(), acc) + C_BOUND * 2.0 ** -24 * self.r


def bound(s, t):
    return C_BOUND * (2.0 ** -20 * s + 2.0 ** -21 * t)


def reference(a, b, chunk=1 << 16):
    """(ref, bound) of A B^T, computed in row chunks of A"""
    refs, bnds = [], []
    for r0 in range(0, a.shape[0], chunk):
        r, bd = RefAccumulator().add(a[r0:r0 + chunk], b).result()
        refs.append(r)
        bnds.append(bd)
    return torch.cat(refs), torch.cat(bnds)


def worst_ratio(got, ref, bnd):
    """max over elements of |got - ref| / bound; an element whose bound is 0 (all its products are 0) must be exact"""
    err = (got.double() - ref).abs()
    if bool((err[bnd == 0] != 0).any()):
        return math.inf
    r = torch.where(bnd > 0, err / torch.where(bnd > 0, bnd, torch.ones_like(bnd)), torch.zeros_like(err))
    return float(r.max()) if r.numel() else 0.0


# ---------------------------------------------------------------- numpy emulation of the kernels' arithmetic ---
def tf32(x):
    """fp32 truncated to TF32 (10 explicit mantissa bits): what the tensor cores read from an fp32 register"""
    return (np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def split(x):
    """hi = truncated x, lo = the exact fp32 remainder as the MMA sees it (truncated to TF32 again)"""
    x = np.asarray(x, dtype=np.float32)
    hi = tf32(x)
    return hi, tf32(x - hi)


# which of the three MMAs (lo_a*hi_b, hi_a*lo_b, hi_a*hi_b, in the kernels' issue order) a mode keeps
MODES = {
    "3xtf32": (True, True, True),
    "2xtf32_no_lo_hi": (False, True, True),
    "2xtf32_no_hi_lo": (True, False, True),
    "1xtf32": (False, False, True),
}


def round_toward_zero(x64):
    """fp64 -> fp32, truncating (the H100 tensor cores' accumulation, see the module docstring)"""
    f = x64.astype(np.float32)
    return np.where(np.abs(f.astype(np.float64)) > np.abs(x64), np.nextafter(f, np.float32(0)), f)


def emulate_split_k(a, b, split, mode):
    """emulate() of each range of `split` K-terms (the dW kernels' split-K), then the fp32 partials added in range
    order, rounded to nearest (k_splitk_reduce)"""
    total = None
    for k0 in range(0, a.shape[1], split):
        part = emulate(a[:, k0:k0 + split], b[:, k0:k0 + split], mode)
        total = part if total is None else (total.astype(np.float64) + part).astype(np.float32)
    return total


def emulate(a, b, mode):
    """fp32 C = A B^T the way the kernels compute it.  Tensor-core modes: for each k8 step, each kept MMA adds the
    exact sum of its 8 products (TF32 x TF32 is exact in fp32, and the sum is formed in fp64 here) to the fp32
    accumulator with one rounding toward zero.  "fp32": sequential fused multiply-adds in fp32, rounded to nearest, as
    the SIMT kernels do."""
    a = np.asarray(a, dtype=np.float32)
    b = np.asarray(b, dtype=np.float32)
    m, k = a.shape
    acc = np.zeros((m, b.shape[0]), dtype=np.float32)
    if mode == "fp32":
        a64, b64 = a.astype(np.float64), b.astype(np.float64)
        for kk in range(k):
            acc = (acc + np.outer(a64[:, kk], b64[:, kk])).astype(np.float32)
        return acc
    keep = MODES[mode]
    kp = (k + 7) // 8 * 8
    pa = np.zeros((m, kp), np.float32)
    pb = np.zeros((b.shape[0], kp), np.float32)
    pa[:, :k], pb[:, :k] = a, b
    ah, al = split(pa)
    bh, bl = split(pb)
    terms = [(al, bh), (ah, bl), (ah, bh)]
    for k0 in range(0, kp, 8):
        for on, (x, y) in zip(keep, terms):
            if on:
                part = x[:, k0:k0 + 8].astype(np.float64) @ y[:, k0:k0 + 8].astype(np.float64).T
                acc = round_toward_zero(acc.astype(np.float64) + part)
    return acc
