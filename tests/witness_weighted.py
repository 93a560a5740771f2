"""The weighted GCN (roc_b200.model.build_gcn_weighted) restated in torch fp64 with autograd over edge lists
(index_add): no code shared with the product or the weighted oracle."""
import numpy as np
import torch

from witness_gat import edge_lists, train_loss


def gcn_weighted_witness(row_end, col, feats, labels, mask, layers, weights, edge_w):
    """Logits, dL/dW per layer (W_mem[o][i]) and dL/d(edge weights) of one step at dropout 0, with the summed
    cross-entropy over the train rows; every layer aggregates with the same edge weights."""
    ws = [torch.from_numpy(w.astype(np.float64)).requires_grad_(True) for w in weights]
    ew = torch.from_numpy(np.asarray(edge_w, dtype=np.float64)).requires_grad_(True)
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    t = torch.from_numpy(feats.astype(np.float64))
    L = len(layers) - 1
    for i in range(L):
        h = t @ ws[i].T
        t = torch.zeros((n, h.shape[1]), dtype=torch.float64).index_add(0, dst, ew[:, None] * h[src])
        if i != L - 1:
            t = torch.relu(t)
    train_loss(t, labels, mask).backward()
    return t.detach().numpy(), [w.grad.numpy() for w in ws], ew.grad.numpy()
