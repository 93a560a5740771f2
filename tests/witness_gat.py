"""GAT (roc_b200.model.build_gat) restated in torch fp64 with autograd from edge lists (scatter_reduce / index_add):
no code shared with the product or the attention oracle."""
import numpy as np
import torch


def attend(wh, sc, dst, src, n, heads, slope, drop=None):
    """Per head, the softmax over each row's in-edges of LeakyReLU(sc_dst[v] + sc_src[u]) applied to wh[u].  drop:
    [E][heads] multipliers of the softmax weights (attention dropout), or None."""
    z = sc[dst, :heads] + sc[src, heads:]
    y = torch.where(z > 0, z, slope * z)
    # the row max only shifts the exponent; the softmax, and so its gradient, does not depend on it
    m = torch.full((n, heads), -np.inf, dtype=torch.float64).scatter_reduce(
        0, dst.unsqueeze(1).expand(-1, heads), y.detach(), "amax", include_self=True)
    ex = torch.exp(y - m[dst])
    den = torch.zeros((n, heads), dtype=torch.float64).index_add(0, dst, ex)
    a = ex / den[dst]
    if drop is not None:
        a = a * torch.from_numpy(np.asarray(drop, dtype=np.float64))
    f = wh.shape[1] // heads
    msg = (a.unsqueeze(2) * wh[src].reshape(-1, heads, f)).reshape(-1, wh.shape[1])
    return torch.zeros((n, wh.shape[1]), dtype=torch.float64).index_add(0, dst, msg)


def edge_lists(row_end, col):
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    return torch.from_numpy(np.repeat(np.arange(row_end.shape[0]), deg)), torch.from_numpy(col.astype(np.int64))


def train_loss(logits, labels, mask):
    """The summed cross-entropy over the train rows."""
    train = torch.from_numpy(mask == 0)
    return torch.nn.functional.cross_entropy(logits[train], torch.from_numpy(labels.astype(np.int64))[train],
                                             reduction="sum")


def gat_witness(row_end, col, feats, labels, mask, layers, weights, heads, slope=0.2):
    """Logits and dL/dW (weights per layer: feature Linear, score Linear; W_mem[o][i]) of one step at dropout 0, with
    the summed cross-entropy over the train rows.  heads: one head count per hidden layer (the last layer has one)."""
    ws = [torch.from_numpy(w.astype(np.float64)).requires_grad_(True) for w in weights]
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    hs = list(heads) + [1]
    t = torch.from_numpy(feats.astype(np.float64))
    L = len(layers) - 1
    for i in range(L):
        wh = t @ ws[2 * i].T
        sc = wh @ ws[2 * i + 1].T
        t = attend(wh, sc, dst, src, n, hs[i], slope)
        if i != L - 1:
            t = torch.relu(t)
    train_loss(t, labels, mask).backward()
    return t.detach().numpy(), [w.grad.numpy() for w in ws]
