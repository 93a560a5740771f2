"""The graph transformer (roc_b200.model.build_graph_transformer, Model.dot_attention_gather) restated in torch fp64
with autograd from edge lists: no code shared with the product."""
import numpy as np
import torch

from witness_gat import edge_lists, train_loss

EPS = float(np.float32(1e-5))       # batch_norm's and layer_norm's default eps, as the fp32 the product holds


def dot_scale(f):
    """1 / sqrt(F) computed in double and rounded once to fp32, as the host default"""
    return float(np.float32(1.0 / np.sqrt(f)))


def dot_attend(q, k, v, dst, src, n, heads, scale):
    """Per head, the softmax over each row's in-edges u of s = scale * q[v] . k[u], applied to v[u].  Returns (out, m,
    Z) with m, Z per (row, head); a row of degree 0 gets out 0."""
    f = q.shape[1] // heads
    s = scale * (q[dst].reshape(-1, heads, f) * k[src].reshape(-1, heads, f)).sum(2)
    # the row max only shifts the exponent; the softmax, and so its gradient, does not depend on it
    m = torch.full((n, heads), -np.inf, dtype=torch.float64).scatter_reduce(
        0, dst.unsqueeze(1).expand(-1, heads), s.detach(), "amax", include_self=True)
    ex = torch.exp(s - m[dst])
    den = torch.zeros((n, heads), dtype=torch.float64).index_add(0, dst, ex)
    p = ex / den[dst]
    msg = (p.unsqueeze(2) * v[src].reshape(-1, heads, f)).reshape(-1, q.shape[1])
    return torch.zeros((n, q.shape[1]), dtype=torch.float64).index_add(0, dst, msg), m, den


def kernel_witness(row_end, col, q, k, v, gy, heads, scale):
    """out, m, 1/Z and the gradients (dq, dk, dv) of sum(out * gy), all fp64 numpy.  q, k, v, gy: [N][H].  Pass the
    same array more than once for a shared input: the first of its names then holds the whole gradient, the later ones
    None."""
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    ts, seen = [], {}
    for x in (q, k, v):
        if id(x) not in seen:
            seen[id(x)] = torch.tensor(np.asarray(x, dtype=np.float64), requires_grad=True)
            ts.append(seen[id(x)])
        else:
            ts.append(None)
    tq, tk, tv = (seen[id(x)] for x in (q, k, v))
    out, m, den = dot_attend(tq, tk, tv, dst, src, n, heads, scale)
    (out * torch.from_numpy(np.asarray(gy, dtype=np.float64))).sum().backward()
    m, den = m.detach(), den.detach()
    deg0 = den == 0
    m = torch.where(deg0, torch.zeros_like(m), m)
    iz = torch.where(deg0, torch.zeros_like(den), 1.0 / torch.where(deg0, torch.ones_like(den), den))
    grads = [t.grad.numpy() if t is not None else None for t in ts]
    return dict(out=out.detach().numpy(), m=m.numpy(), iz=iz.numpy(), dq=grads[0], dk=grads[1], dv=grads[2])


def model_witness(row_end, col, feats, labels, mask, layers, weights, heads, root_weight=True, activation="relu",
                  loss_fn=train_loss, norm=None):
    """Logits and the gradient of every parameter (in Model order: per layer the q, k and v Linears, the skip Linear
    when root_weight, then with a norm on a hidden layer its gamma and beta as (1, H)) of one training step at dropout
    0.  norm="batch" normalises with the batch statistics (biased variance), norm="layer_norm" each row; both with
    eps = fp32 1e-5."""
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(True) for w in weights]
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    hs = list(heads) + [1]
    t = torch.from_numpy(np.asarray(feats, dtype=np.float32)).to(torch.float64)
    L = len(layers) - 1
    k = 0
    for i in range(L):
        q, kk, v = (t @ ws[k + j].T for j in range(3))
        k += 3
        out = dot_attend(q, kk, v, dst, src, n, hs[i], dot_scale(layers[i + 1] // hs[i]))[0]
        if root_weight:
            out = out + t @ ws[k].T
            k += 1
        t = out
        if i != L - 1:
            if norm == "batch":
                t = torch.nn.functional.batch_norm(t, None, None, ws[k][0], ws[k + 1][0], training=True, eps=EPS)
                k += 2
            elif norm == "layer_norm":
                t = torch.nn.functional.layer_norm(t, (t.shape[1],), ws[k][0], ws[k + 1][0], EPS)
                k += 2
            t = torch.nn.functional.elu(t) if activation == "elu" else torch.relu(t)
    loss_fn(t, labels, mask).backward()
    return t.detach().numpy(), [w.grad.numpy() for w in ws]
