"""APPNP and GCNII (roc_b200.model.build_appnp / build_gcnii) as recorded op graphs, and a torch fp64 autograd
interpreter of them: no code shared with the product.

The graphs are recorded by opgraph.Recorder; a scaled_add node has attrs alpha / beta, the fp32 coefficients the
product was given, as doubles.  witness() runs the ops the two builders use (linear, dropout, indegree_norm,
scatter_gather, relu, scaled_add and the two losses) from edge lists."""
import numpy as np
import torch

from oracle import oracle
from opgraph import _relu_with_mask
from roc_b200 import _lib
from witness_gat import edge_lists, train_loss


def bce_train_loss(x, labels, mask):
    train = torch.from_numpy(np.asarray(mask) == _lib.MASK_TRAIN)
    y = torch.from_numpy(np.asarray(labels, dtype=np.float64))
    return torch.nn.functional.binary_cross_entropy_with_logits(x[train], y[train], reduction="sum")


def witness(ir, graph, feats, labels, mask, weights, step=1, relu_masks=None, training=True, loss_fn=train_loss):
    """One training step of the recorded graph in fp64: the logits and dL/dW (W_mem[o][i] per parameter).  graph:
    (row_end, col); step: the product's train step (dropout masks); relu_masks {layer: product output > 0}, taken where
    fp32 and fp64 tie.  training=False: dropout is a copy and nothing is differentiated."""
    row_end, col = np.asarray(graph[0]), np.asarray(graph[1])
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dinv = torch.from_numpy(1.0 / np.sqrt(deg.astype(np.float64))).unsqueeze(1)
    relu_masks = relu_masks or {}
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(training) for w in weights]
    val = {ir.leaves[0]: torch.from_numpy(np.asarray(feats, dtype=np.float64))}
    loss, logits = None, None
    for node in ir.nodes:
        k, a, ins, what = node["kind"], node["attrs"], node["ins"], "layer %d (%s)" % (node["layer"], node["kind"])
        x = val.get(ins[0])
        if k == "linear":
            y = x @ ws[a["param"]].T
            if a["activation"] == _lib.AC_MODE_RELU:
                y = _relu_with_mask(y, relu_masks.get(node["layer"]), what)
        elif k == "indegree_norm":
            y = x * dinv
        elif k == "scatter_gather":
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, x[src])
        elif k == "relu":
            y = _relu_with_mask(x, relu_masks.get(node["layer"]), what)
        elif k == "scaled_add":
            y = a["alpha"] * x + a["beta"] * val[ins[1]]
        elif k == "dropout":
            if a["rate"] > 0 and training:
                keep = oracle.dropout_mask(0, n, x.shape[1], a["rate"], a["key"], step)
                scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(a["rate"])))
                y = x * torch.from_numpy(keep.astype(np.float64) * scale)
            else:
                y = x
        elif k in ("softmax_cross_entropy", "sigmoid_cross_entropy"):
            logits = x
            if training:
                loss = loss_fn(x, np.asarray(labels), np.asarray(mask))
            continue
        else:
            raise AssertionError("unknown op " + k)
        val[node["out"]] = y
    if loss is not None and loss.requires_grad:
        loss.backward()
    return dict(logits=logits.detach().numpy(),
                dW=[w.grad.numpy() if w.grad is not None else np.zeros(w.shape) for w in ws])
