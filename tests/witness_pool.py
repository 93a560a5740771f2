"""GraphSAGE-pool (roc_b200.model.build_sage_pool) derived independently in torch fp64 with autograd: no code shared
with the product or the oracle.  The aggregation picks, per row and feature, the FIRST source in CSR order holding
the max (min) explicitly and gathers it, so autograd sends the gradient to that one source (torch's own amax
backward would split ties)."""
import numpy as np
import torch


def first_extreme_sources(row_end, col, p, is_max):
    """[N][H] int64: per row and feature, the source of the first edge with the max / min of p (fp64, no NaN)."""
    n, h = row_end.shape[0], p.shape[1]
    out = np.zeros((n, h), dtype=np.int64)
    s = 0
    for v in range(n):
        e = int(row_end[v])
        if e > s:
            vals = p[col[s:e]]
            k = np.argmax(vals, axis=0) if is_max else np.argmin(vals, axis=0)
            out[v] = col[s:e][k]
        s = e
    return out


def sage_pool_witness(row_end, col, feats, labels, mask, layers, weights, is_max=True, args=None):
    """Logits, dL/dW (weights per layer: pool, neighbour, root), the chosen sources and the pooled values p per
    layer.  `args` (one [N][H] array per layer, or None) overrides the choice, e.g. with the product's own where fp32
    and fp64 disagree."""
    ws = [torch.from_numpy(w.astype(np.float64)).requires_grad_(True) for w in weights]
    t = torch.from_numpy(feats.astype(np.float64))
    L = len(layers) - 1
    chosen, pools = [], []
    for i in range(1, L + 1):
        wp, wn, wr = ws[3 * (i - 1): 3 * i]
        d = t                                                   # dropout rate 0
        p = torch.relu(d @ wp.T)
        src = args[i - 1] if args is not None else first_extreme_sources(row_end, col, p.detach().numpy(), is_max)
        src = np.asarray(src, dtype=np.int64)
        chosen.append(src)
        pools.append(p.detach().numpy())
        nb = p.gather(0, torch.from_numpy(src))                 # nb[v][h] = p[src[v][h]][h]
        z = nb @ wn.T + d @ wr.T
        t = torch.relu(z) if i != L else z
    logits = t
    train = torch.from_numpy(mask == 0)
    loss = torch.nn.functional.cross_entropy(logits[train], torch.from_numpy(labels.astype(np.int64))[train],
                                             reduction="sum")
    loss.backward()
    return logits.detach().numpy(), [w.grad.numpy() for w in ws], chosen, pools
