"""Synthetic inputs in the reference's formats (SURVEY Appendix C, §8d).

Graphs are symmetrised (the reference's backward multiplies by A, not A^T —
scattergather_kernel.cu:160-170 — which is the true adjoint only for symmetric
A), de-duplicated, given self loops (the `.add_self_edge.lux` convention,
gnn.cc:756) and sorted by (dst, src).  directed=True skips the symmetrisation, for
models trained with Model.set_exact_backward, whose backward runs over the transposed
graph.  CSR convention: rowEnd[v] = inclusive
prefix sum of in-degrees (u64), col[e] = source (u32).

Generators run on whatever torch device is passed (CPU in tests, the GPU in
bench.py — generation is setup, never inside a timed region).
"""
import os

import numpy as np
import torch


def _csr_from_pairs(src, dst, n, directed=False):
    """Symmetrise (unless directed) + self loops + dedup + sort by (dst, src).  src/dst: int64 tensors."""
    dev = src.device
    loops = torch.arange(n, device=dev, dtype=torch.int64)
    if directed:
        s = torch.cat([src, loops])
        d = torch.cat([dst, loops])
    else:
        s = torch.cat([src, dst, loops])
        d = torch.cat([dst, src, loops])
    key = torch.unique(d * n + s)          # sorted by dst then src, duplicates removed
    d = key // n
    s = key - d * n
    deg = torch.bincount(d, minlength=n)
    row_end = torch.cumsum(deg, 0)
    return row_end.to(torch.int64), s.to(torch.int32)


def uniform_graph(n, n_pairs, seed=1, device="cpu", directed=False):
    """directed=True keeps each pair's orientation (src -> dst): no reverse edges are added."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    src = torch.randint(0, n, (n_pairs,), generator=g, device=device, dtype=torch.int64)
    dst = torch.randint(0, n, (n_pairs,), generator=g, device=device, dtype=torch.int64)
    return _csr_from_pairs(src, dst, n, directed)


def rmat_graph(scale, n_pairs, seed=1, abcd=(0.57, 0.19, 0.19, 0.05), permute=True, device="cpu", directed=False):
    """R-MAT (Chakrabarti et al.) with Graph500's (a,b,c,d); n = 2^scale vertices,
    n_pairs undirected pairs drawn before symmetrisation / dedup.  directed=True keeps each pair's orientation
    (src -> dst): the graph gets no reverse edges, so it has about half the edges of the symmetric one."""
    n = 1 << scale
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    a, b, c, _ = abcd
    src = torch.zeros(n_pairs, dtype=torch.int64, device=device)
    dst = torch.zeros(n_pairs, dtype=torch.int64, device=device)
    for bit in range(scale):
        r = torch.rand(n_pairs, generator=g, device=device)
        sbit = r >= (a + b)
        dbit = ((r >= a) & (r < a + b)) | (r >= a + b + c)
        src |= sbit.to(torch.int64) << bit
        dst |= dbit.to(torch.int64) << bit
    if permute:
        perm = torch.randperm(n, generator=g, device=device)
        src, dst = perm[src], perm[dst]
    return _csr_from_pairs(src, dst, n, directed)


def powerlaw_graph(n, n_pairs, alpha=1.6, seed=1, device="cpu"):
    """Degree-shaped random graph: endpoint popularity ~ Zipf-like weights
    (used for the products-/Reddit-shaped configs)."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    w = (torch.arange(1, n + 1, device=device, dtype=torch.float64)) ** (-1.0 / alpha)
    cdf = torch.cumsum(w / w.sum(), 0)
    perm = torch.randperm(n, generator=g, device=device)
    u = torch.rand(n_pairs, generator=g, device=device, dtype=torch.float64)
    src = perm[torch.searchsorted(cdf, u).clamp_(max=n - 1)]
    dst = torch.randint(0, n, (n_pairs,), generator=g, device=device, dtype=torch.int64)
    return _csr_from_pairs(src, dst, n)


def node_data(n, in_dim, num_classes, seed=1, device="cpu"):
    """features ~ U(-1,1) fp32, labels uniform over classes, mask 66% Train / 10% Val / 24% Test."""
    g = torch.Generator(device=device)
    g.manual_seed(seed + 7)
    feats = torch.rand((n, in_dim), generator=g, device=device, dtype=torch.float32) * 2.0 - 1.0
    labels = torch.randint(0, num_classes, (n,), generator=g, device=device, dtype=torch.int32)
    u = torch.rand(n, generator=g, device=device)
    mask = torch.full((n,), 2, dtype=torch.int32, device=device)   # MASK_TEST
    mask[u < 0.76] = 1                                              # MASK_VAL
    mask[u < 0.66] = 0                                              # MASK_TRAIN
    return feats, labels, mask


def multilabel_node_data(n, in_dim, num_labels, seed=1, device="cpu", positive_rate=0.1):
    """Multi-label node data a model can learn: features ~ U(-1,1) fp32; labels y = (x @ R + noise > tau) as uint8
    [n][num_labels] 0/1, with R and the noise drawn from the seed and tau the (1 - positive_rate) quantile of all
    scores, so that about positive_rate of the labels are positive; mask 66% Train / 10% Val / 24% Test as node_data."""
    g = torch.Generator(device=device)
    g.manual_seed(seed + 11)
    feats = torch.rand((n, in_dim), generator=g, device=device, dtype=torch.float32) * 2.0 - 1.0
    r = torch.randn((in_dim, num_labels), generator=g, device=device, dtype=torch.float64) / np.sqrt(in_dim)
    noise = torch.randn((n, num_labels), generator=g, device=device, dtype=torch.float64) * 0.1
    score = feats.double() @ r + noise
    tau = torch.quantile(score.flatten()[: 1 << 24], 1.0 - positive_rate)
    labels = (score > tau).to(torch.uint8)
    u = torch.rand(n, generator=g, device=device)
    mask = torch.full((n,), 2, dtype=torch.int32, device=device)   # MASK_TEST
    mask[u < 0.76] = 1                                              # MASK_VAL
    mask[u < 0.66] = 0                                              # MASK_TRAIN
    return feats, labels, mask


def onehot(labels, num_classes):
    labels = np.asarray(labels)
    out = np.zeros((labels.shape[0], num_classes), dtype=np.float32)
    out[np.arange(labels.shape[0]), labels] = 1.0
    return out


# ------------------------------------------------------------- file formats ---
def write_lux(prefix, row_end, col_src):
    """<prefix>.add_self_edge.lux: u32 N, u64 E, u64 rowEnd[N], u32 src[E] (gnn.cc:756-801)."""
    row_end = np.ascontiguousarray(np.asarray(row_end), dtype=np.uint64)
    col_src = np.ascontiguousarray(np.asarray(col_src), dtype=np.uint32)
    with open(prefix + ".add_self_edge.lux", "wb") as f:
        f.write(np.uint32(row_end.shape[0]).tobytes())
        f.write(np.uint64(col_src.shape[0]).tobytes())
        f.write(row_end.tobytes())
        f.write(col_src.tobytes())


def read_lux(prefix):
    with open(prefix + ".add_self_edge.lux", "rb") as f:
        n = int(np.frombuffer(f.read(4), dtype=np.uint32)[0])
        e = int(np.frombuffer(f.read(8), dtype=np.uint64)[0])
        row_end = np.frombuffer(f.read(8 * n), dtype=np.uint64).copy()
        col = np.frombuffer(f.read(4 * e), dtype=np.uint32).copy()
    return n, e, row_end, col


def write_feats_bin(prefix, feats):
    np.ascontiguousarray(np.asarray(feats), dtype=np.float32).tofile(prefix + ".feats.bin")


def write_feats_csv(prefix, feats):
    with open(prefix + ".feats.csv", "w") as f:
        for row in np.asarray(feats):
            f.write(",".join(repr(float(v)) for v in row) + "\n")


def write_labels(prefix, labels):
    with open(prefix + ".label", "w") as f:
        for v in np.asarray(labels):
            f.write("%d\n" % int(v))


def write_mask(prefix, mask):
    names = {0: "Train", 1: "Val", 2: "Test", 3: "None"}
    with open(prefix + ".mask", "w") as f:
        for v in np.asarray(mask):
            f.write(names[int(v)] + "\n")


def write_dataset(prefix, row_end, col_src, feats, labels, mask):
    os.makedirs(os.path.dirname(prefix) or ".", exist_ok=True)
    write_lux(prefix, row_end, col_src)
    write_feats_bin(prefix, feats)
    write_labels(prefix, labels)
    write_mask(prefix, mask)


def gcn_edge_weights(row_end, col, w):
    """GCN's symmetric normalisation of edge weights: w_e / sqrt(d_i d_j) for edge e = (i <- j), where d is the
    weighted in-degree (the sum of a row's weights).  Weights are >= 0; an edge whose d_i d_j is 0 gets 0.  Computed
    once per graph in fp64 on the host and returned as fp32 in the CSR's edge order."""
    t = np.asarray(row_end, dtype=np.int64)
    deg = np.diff(np.concatenate([[0], t]))
    dst = np.repeat(np.arange(t.shape[0]), deg)
    w = np.asarray(w, dtype=np.float64)
    assert w.shape[0] == t[-1] and (w >= 0).all(), "one weight >= 0 per edge"
    d = np.bincount(dst, weights=w, minlength=t.shape[0])
    dd = d[dst] * d[np.asarray(col, dtype=np.int64)]
    out = np.zeros_like(w)
    np.divide(w, np.sqrt(dd), out=out, where=dd > 0)
    return out.astype(np.float32)
