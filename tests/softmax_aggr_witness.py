"""The softmax aggregation (Model.softmax_gather, roc_sg_softmax_*) and DeeperGCN (roc_b200.model.build_deepergcn)
restated in torch fp64 with autograd from edge lists: a per-edge scatter softmax per column, no code shared with the
product."""
import numpy as np
import torch

from witness_gat import edge_lists, train_loss

BN_EPS = float(np.float32(1e-5))


def softmax_aggr(x, t, dst, src, n):
    """y[v][f] = sum_u p_u x[u][f], p = softmax over v's in-edges of t * x[u][f] (y = 0 for a row of degree 0).  x: [N][H]
    fp64, t: a 0-d fp64 tensor.  Returns (y, m, Z) with m, Z per (row, column); a row of degree 0 has Z = 0."""
    z = t * x[src]
    # the row max only shifts the exponent; the softmax, and so its gradient, does not depend on it
    m = torch.full((n, x.shape[1]), -np.inf, dtype=torch.float64).scatter_reduce(
        0, dst.unsqueeze(1).expand(-1, x.shape[1]), z.detach(), "amax", include_self=True)
    ex = torch.exp(z - m[dst])
    den = torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, ex)
    p = ex / den[dst]
    return torch.zeros((n, x.shape[1]), dtype=torch.float64).index_add(0, dst, p * x[src]), m, den


def kernel_witness(row_end, col, x, t, gy):
    """y, m, 1/Z (0 | 0 for a row of degree 0), dx and dt of sum(y * gy), all fp64 numpy; x, gy: [N][H], t a float."""
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    tx = torch.tensor(np.asarray(x, dtype=np.float64), requires_grad=True)
    tt = torch.tensor(float(t), dtype=torch.float64, requires_grad=True)
    y, m, den = softmax_aggr(tx, tt, dst, src, n)
    (y * torch.from_numpy(np.asarray(gy, dtype=np.float64))).sum().backward()
    m, den = m.detach(), den.detach()
    deg0 = den == 0
    m = torch.where(deg0, torch.zeros_like(m), m)
    iz = torch.where(deg0, torch.zeros_like(den), 1.0 / torch.where(deg0, torch.ones_like(den), den))
    return dict(out=y.detach().numpy(), m=m.numpy(), iz=iz.numpy(), dx=tx.grad.numpy(), dt=float(tt.grad))


def model_witness(row_end, col, feats, labels, mask, layers, weights, depth, learn_temperature=True,
                  temperature=1.0, norm="batch", expansion=2, loss_fn=train_loss, bf16_features=False,
                  training=True, bn_running=None):
    """Logits and the gradient of every parameter, in Model order, of one step of build_deepergcn at dropout 0.  The
    parameters are as get_parameter returns them: a Linear's W as (out, in), a batch_norm's gamma and beta as (1, H),
    each learned t as (1, 1).  Model order: the encoder's W, then per layer its t (learn_temperature), the expansion
    Linear's W, the conv's batch_norm (norm="batch"), the second Linear's W, with layers 2.. first taking the
    pre-conv batch_norm; then the head's batch_norm and W.  norm="batch" normalises with the batch statistics (biased
    variance, eps = fp32 1e-5) when training, else with bn_running, a list of (mean, var) per batch_norm in model
    order.  bf16_features: the input features as their bf16 rounding (RNE)."""
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(True) for w in weights]
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    x = torch.from_numpy(np.asarray(feats, dtype=np.float32))
    x = (x.to(torch.bfloat16) if bf16_features else x).to(torch.float64)
    k = [0]
    nb = [0]

    def take():
        k[0] += 1
        return ws[k[0] - 1]

    def norm_relu(t):
        if norm == "batch":
            g, b = take(), take()
            if training:
                t = torch.nn.functional.batch_norm(t, None, None, g[0], b[0], training=True, eps=BN_EPS)
            else:
                mean, var = (torch.from_numpy(np.asarray(v, dtype=np.float64)) for v in bn_running[nb[0]])
                t = torch.nn.functional.batch_norm(t, mean, var, g[0], b[0], training=False, eps=BN_EPS)
            nb[0] += 1
        return torch.relu(t)

    def genconv(h):
        t = take()[0, 0] if learn_temperature else torch.tensor(float(np.float32(temperature)), dtype=torch.float64)
        a = softmax_aggr(torch.relu(h), t, dst, src, n)[0]
        w1 = take()
        z = (a + h) @ w1.T
        z = norm_relu(z)
        return z @ take().T

    t = x @ take().T
    t = genconv(t)
    for _ in range(2, depth + 1):
        t = t + genconv(norm_relu(t))
    logits = norm_relu(t) @ take().T
    assert k[0] == len(ws)
    if training:
        loss_fn(logits, labels, mask).backward()
        return logits.detach().numpy(), [w.grad.numpy() for w in ws]
    return logits.detach().numpy(), None
