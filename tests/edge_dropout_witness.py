"""Edge dropout of the sum ScatterGather (include/roc_b200.h, roc_sg_forward_dropout_planned) restated: the keep bit
of every edge, and a torch fp64 autograd interpreter of the GCN and APPNP graphs that model scripts with
Model.scatter_gather(dropout=) build, as opgraph.Recorder records them.  No code shared with the product.

keep(i<-j) is bit 0 of attention dropout's keep byte of the pair (attn_dropout_oracle.keep_bytes); a kept edge's row
is weighted by s = 1.0f / (1.0f - rate) (fp32), a dropped one's by 0, and the degrees are the full graph's."""
import numpy as np
import torch

import attn_dropout_oracle as ado
import opgraph          # a module import: opgraph imports this module too
from oracle import oracle
from roc_b200 import _lib
from witness_gat import edge_lists, train_loss


def drop_scale(rate):
    """s = 1.0f / (1.0f - rate) in fp32, as a double"""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(rate)))


def edge_keep(row_end, col, rate, key, step, col_left=0, self_base=0, row_is_source=False):
    """bool [E]: keep bit of every edge in CSR order, for the pair (row <- col), or (col <- row) with row_is_source"""
    b = ado.edge_keep(row_end, col, rate, key, step, col_left, self_base, row_is_source)
    return (b & 1).astype(bool)


def edge_weights(keep, rate):
    """fp32 [E]: keep ? s : 0, the weights under which the weighted sum is the dropped sum"""
    return np.where(keep, np.float32(drop_scale(rate)), np.float32(0.0)).astype(np.float32)


def witness(ir, graph, feats, labels, mask, weights, step=1, relu_masks=None, training=True):
    """One training step of the recorded graph in fp64 (the ops of build_gcn and build_appnp): the logits, dL/dW
    (W_mem[o][i] per parameter) and each dropped scatter_gather's keep bits ({layer: bool [E]}).  graph: (row_end,
    col); step: the product's train step (its dropout masks); relu_masks {layer: product output > 0}, taken where fp32
    and fp64 tie.  training=False: no dropout of either kind and nothing differentiated.  The gradient is autograd's,
    the true adjoint on any graph."""
    row_end, col = np.asarray(graph[0]), np.asarray(graph[1])
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dinv = torch.from_numpy(1.0 / np.sqrt(deg.astype(np.float64))).unsqueeze(1)
    relu_masks = relu_masks or {}
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(training) for w in weights]
    val = {ir.leaves[0]: torch.from_numpy(np.asarray(feats, dtype=np.float64))}
    loss, logits, masks = None, None, {}
    for node in ir.nodes:
        k, a, ins, what = node["kind"], node["attrs"], node["ins"], "layer %d (%s)" % (node["layer"], node["kind"])
        x = val.get(ins[0])
        if k == "linear":
            y = x @ ws[a["param"]].T
            if a["activation"] == _lib.AC_MODE_RELU:
                y = opgraph._relu_with_mask(y, relu_masks.get(node["layer"]), what)
        elif k == "indegree_norm":
            y = x * dinv
        elif k == "scatter_gather":
            rows = x[src]
            if a.get("dropout", 0.0) > 0 and training:
                keep = edge_keep(row_end, col, a["dropout"], a["key"], step)
                masks[node["layer"]] = keep
                rows = rows * torch.from_numpy(keep.astype(np.float64) * drop_scale(a["dropout"])).unsqueeze(1)
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, rows)
        elif k == "relu":
            y = opgraph._relu_with_mask(x, relu_masks.get(node["layer"]), what)
        elif k == "add":
            y = x + val[ins[1]]
        elif k == "scaled_add":
            y = a["alpha"] * x + a["beta"] * val[ins[1]]
        elif k == "dropout":
            if a["rate"] > 0 and training:
                keep = oracle.dropout_mask(0, n, x.shape[1], a["rate"], a["key"], step)
                y = x * torch.from_numpy(keep.astype(np.float64) * drop_scale(a["rate"]))
            else:
                y = x
        elif k == "softmax_cross_entropy":
            logits = x
            if training:
                loss = train_loss(x, np.asarray(labels), np.asarray(mask))
            continue
        else:
            raise AssertionError("unknown op " + k)
        val[node["out"]] = y
    if loss is not None and loss.requires_grad:
        loss.backward()
    return dict(logits=logits.detach().numpy(), masks=masks,
                dW=[w.grad.numpy() if w.grad is not None else np.zeros(w.shape) for w in ws])
