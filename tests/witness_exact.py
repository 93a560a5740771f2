"""GCN and GraphSAGE-mean (roc_b200.model.build_gcn / build_sage_mean) restated in torch fp64 with autograd over edge
lists (index_add), so that a duplicate edge counts twice in the aggregation and in the in-degree, as in the product:
no code shared with the product or the oracles.  witness.torch_witness builds a dense A by assignment, which counts a
duplicate once; this one is for multigraphs."""
import numpy as np
import torch

from witness_gat import edge_lists, train_loss


def gcn_sage_witness(kind, row_end, col, feats, labels, mask, layers, weights):
    """Logits and dL/dW (W_mem[o][i], in parameter order) of one step at dropout 0 for kind "gcn" or "sage_mean",
    with the summed cross-entropy over the train rows."""
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dinv = torch.from_numpy(1.0 / np.sqrt(deg.astype(np.float64))).unsqueeze(1)
    ws = [torch.from_numpy(w.astype(np.float64)).requires_grad_(True) for w in weights]

    def agg(h):                                          # sum over in-edges, duplicates counted
        return torch.zeros((n, h.shape[1]), dtype=torch.float64).index_add(0, dst, h[src])

    t = torch.from_numpy(feats.astype(np.float64))
    L = len(layers) - 1
    wi = 0
    for i in range(1, L + 1):
        d = t                                            # dropout rate 0
        if kind == "gcn":
            z = agg((d @ ws[wi].T) * dinv) * dinv
            wi += 1
            if i != L:
                z = torch.relu(z)
            if len(layers) > 3:                          # the residual branch
                z = z + d @ ws[wi].T
                wi += 1
            t = z
        else:
            z = agg(d @ ws[wi].T) * dinv * dinv + d @ ws[wi + 1].T
            wi += 2
            t = torch.relu(z) if i != L else z
    train_loss(t, labels, mask).backward()
    return t.detach().numpy(), [w.grad.numpy() for w in ws]
