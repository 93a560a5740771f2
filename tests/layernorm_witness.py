"""Layer normalisation (roc_layernorm_*, Model.layer_norm) restated in torch fp64 with autograd, no code shared with the
product: the kernel's forward and backward through torch.nn.functional.layer_norm; DeeperGCN with layer norm, built
from softmax_aggr_witness.softmax_aggr with its block structure restated; and an interpreter of a recorded GCN / GAT /
GraphSAGE op graph (tests/opgraph.py's Recorder) with layer_norm nodes, at dropout 0."""
import numpy as np
import torch

from softmax_aggr_witness import softmax_aggr
from witness_gat import attend, edge_lists, train_loss

LN_EPS = float(np.float32(1e-5))


def kernel_witness(x, gy, gamma, beta, eps=LN_EPS, relu=False):
    """y, and dx, dgamma, dbeta of sum(y * gy), for fp32 / fp64 [N][H] x and gy, in fp64 on x's device.  With relu, y
    is relu(layer_norm(x)) and the gradient is masked by the pre-relu value > 0, as torch's relu is."""
    tx = x.detach().double().clone().requires_grad_(True)
    tg = gamma.detach().double().clone().requires_grad_(True)
    tb = beta.detach().double().clone().requires_grad_(True)
    pre = torch.nn.functional.layer_norm(tx, (tx.shape[1],), tg, tb, eps)
    y = torch.relu(pre) if relu else pre
    (y * gy.detach().double()).sum().backward()
    return dict(y=y.detach(), pre=pre.detach(), dx=tx.grad, dgamma=tg.grad, dbeta=tb.grad)


def deepergcn_witness(row_end, col, feats, labels, mask, layers, weights, depth, learn_temperature=True,
                      temperature=1.0, expansion=2, loss_fn=train_loss):
    """Logits and the gradient of every parameter, in Model order, of one training step of
    build_deepergcn(norm="layer_norm") at dropout 0.  The parameters are as get_parameter returns them: a Linear's W as
    (out, in), a layer_norm's gamma and beta as (1, H), each learned t as (1, 1).  Model order: the encoder's W, then
    per layer its t (learn_temperature), the expansion Linear's W, the conv's layer_norm, the second Linear's W, with
    layers 2.. first taking the pre-conv layer_norm; then the head's layer_norm and W.  Returns (logits, grads)."""
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(True) for w in weights]
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    k = [0]

    def take():
        k[0] += 1
        return ws[k[0] - 1]

    def norm_relu(t):                      # res+: LayerNorm, then ReLU
        g, b = take(), take()
        return torch.relu(torch.nn.functional.layer_norm(t, (t.shape[1],), g[0], b[0], LN_EPS))

    def genconv(h):                        # GENConv: softmax aggregation of relu(h), the root added, the MLP
        t = take()[0, 0] if learn_temperature else torch.tensor(float(np.float32(temperature)), dtype=torch.float64)
        a = softmax_aggr(torch.relu(h), t, dst, src, n)[0]
        z = norm_relu((a + h) @ take().T)
        return z @ take().T

    x = torch.from_numpy(np.asarray(feats, dtype=np.float64))
    t = genconv(x @ take().T)
    for _ in range(2, depth + 1):
        t = t + genconv(norm_relu(t))
    logits = norm_relu(t) @ take().T
    assert k[0] == len(ws)
    loss_fn(logits, labels, mask).backward()
    return logits.detach().numpy(), [w.grad.numpy() for w in ws]


def graph_witness(ir, graph, feats, labels, mask, weights, training=True, loss_fn=train_loss):
    """A recorded op graph (linear, layer_norm, indegree_norm, sum scatter_gather, attention_gather, attention_scores,
    relu, elu, add, dropout at rate 0 and the softmax loss) in fp64 with autograd.  layer_norm nodes carry gamma / beta
    parameter indices and eps.  Returns dict(logits, dW)."""
    row_end, col = np.asarray(graph[0]), np.asarray(graph[1])
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    deg = np.diff(np.concatenate([[0], row_end.astype(np.int64)]))
    dinv = torch.from_numpy(1.0 / np.sqrt(deg.astype(np.float64))).unsqueeze(1)
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(training) for w in weights]
    val = {ir.leaves[0]: torch.from_numpy(np.asarray(feats, dtype=np.float64))}
    loss, logits = None, None
    for node in ir.nodes:
        k, a, ins = node["kind"], node["attrs"], node["ins"]
        x = val.get(ins[0])
        if k == "linear":
            y = x @ ws[a["param"]].T
        elif k == "layer_norm":
            y = torch.nn.functional.layer_norm(x, (x.shape[1],), ws[a["gamma"]][0], ws[a["beta"]][0], a["eps"])
        elif k == "indegree_norm":
            y = x * dinv
        elif k == "scatter_gather":
            y = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, x[src])
        elif k == "attention_scores":
            hd, w = a["heads"], ws[a["param"]]
            xv = x.reshape(n, hd, -1)
            y = torch.cat([(xv * w[:hd]).sum(2), (xv * w[hd:]).sum(2)], 1)
        elif k == "attention_gather":
            y = attend(x, val[ins[1]], dst, src, n, a["heads"], a["slope"])
        elif k == "relu":
            y = torch.relu(x)
        elif k == "elu":
            y = torch.nn.functional.elu(x)
        elif k == "add":
            y = x + val[ins[1]]
        elif k == "dropout":
            assert a["rate"] == 0 or not training, "the witness runs at dropout 0"
            y = x
        elif k == "softmax_cross_entropy":
            logits = x
            if training:
                loss = loss_fn(x, np.asarray(labels), np.asarray(mask))
            continue
        else:
            raise AssertionError("layernorm_witness: unsupported op " + k)
        val[node["out"]] = y
    if loss is not None:
        loss.backward()
    return dict(logits=logits.detach().numpy(),
                dW=[w.grad.numpy() if w.grad is not None else np.zeros(w.shape) for w in ws] if training else None)
