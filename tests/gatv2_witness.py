"""GATv2 (roc_b200.model.build_gatv2, Model.dynamic_attention_gather) restated in torch fp64 with autograd from edge
lists: no code shared with the product."""
import numpy as np
import torch

from witness_gat import edge_lists, train_loss


def dynamic_attend(xl, xr, a, dst, src, n, heads, slope):
    """Per head, the softmax over each row v's in-edges u of e = sum_f a[k][f] LeakyReLU(xl[u] + xr[v]) applied to
    xl[u].  a: [heads][F].  Returns (out, m, Z) with m, Z per (row, head); a row of degree 0 gets out 0."""
    f = xl.shape[1] // heads
    z = xl[src] + xr[dst]
    lz = torch.where(z > 0, z, slope * z)
    e = (lz.reshape(-1, heads, f) * a.reshape(1, heads, f)).sum(2)
    # the row max only shifts the exponent; the softmax, and so its gradient, does not depend on it
    m = torch.full((n, heads), -np.inf, dtype=torch.float64).scatter_reduce(
        0, dst.unsqueeze(1).expand(-1, heads), e.detach(), "amax", include_self=True)
    ex = torch.exp(e - m[dst])
    den = torch.zeros((n, heads), dtype=torch.float64).index_add(0, dst, ex)
    p = ex / den[dst]
    msg = (p.unsqueeze(2) * xl[src].reshape(-1, heads, f)).reshape(-1, xl.shape[1])
    return torch.zeros((n, xl.shape[1]), dtype=torch.float64).index_add(0, dst, msg), m, den


def kernel_witness(row_end, col, xl, xr, a, gy, heads, slope):
    """out, m, 1/Z and the gradients (dxl, dxr, da) of sum(out * gy), all fp64 numpy.  xl, xr, gy: [N][H]; a:
    [heads][F].  Pass the same array as xl and xr for a shared input: dxl then holds the whole gradient, dxr None."""
    shared = xl is xr
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    tl = torch.tensor(np.asarray(xl, dtype=np.float64), requires_grad=True)
    tr = tl if shared else torch.tensor(np.asarray(xr, dtype=np.float64), requires_grad=True)
    ta = torch.tensor(np.asarray(a, dtype=np.float64), requires_grad=True)
    out, m, den = dynamic_attend(tl, tr, ta, dst, src, n, heads, slope)
    (out * torch.from_numpy(np.asarray(gy, dtype=np.float64))).sum().backward()
    m, den = m.detach(), den.detach()
    deg0 = (den == 0)
    m = torch.where(deg0, torch.zeros_like(m), m)
    iz = torch.where(deg0, torch.zeros_like(den), 1.0 / torch.where(deg0, torch.ones_like(den), den))
    return dict(out=out.detach().numpy(), m=m.numpy(), iz=iz.numpy(), dxl=tl.grad.numpy(),
                dxr=None if shared else tr.grad.numpy(), da=ta.grad.numpy())


def model_witness(row_end, col, feats, labels, mask, layers, weights, heads, share_weights=False, slope=0.2,
                  activation="relu", loss_fn=train_loss, norm=None, bf16_features=False):
    """Logits and the gradient of every parameter (in Model order: per layer the xl Linear, the xr Linear unless
    share_weights, then a as get_parameter returns it, (F, heads), then with norm="batch" on a hidden layer the
    batch_norm's gamma and beta as (1, H)) of one training step at dropout 0.  norm="batch" normalises with the batch
    statistics (biased variance, eps = fp32 1e-5).  bf16_features: the input features as their bf16 rounding (RNE)."""
    ws = [torch.from_numpy(np.asarray(w, dtype=np.float64)).requires_grad_(True) for w in weights]
    n = row_end.shape[0]
    dst, src = edge_lists(row_end, col)
    hs = list(heads) + [1]
    t = torch.from_numpy(np.asarray(feats, dtype=np.float32))
    t = (t.to(torch.bfloat16) if bf16_features else t).to(torch.float64)
    L = len(layers) - 1
    k = 0
    for i in range(L):
        xl = t @ ws[k].T
        k += 1
        if share_weights:
            xr = xl
        else:
            xr = t @ ws[k].T
            k += 1
        a = ws[k].T                     # get_parameter gives (F, heads)
        k += 1
        t = dynamic_attend(xl, xr, a, dst, src, n, hs[i], slope)[0]
        if i != L - 1 and norm == "batch":
            t = torch.nn.functional.batch_norm(t, None, None, ws[k][0], ws[k + 1][0], training=True,
                                               eps=float(np.float32(1e-5)))
            k += 2
        if i != L - 1:
            t = torch.nn.functional.elu(t) if activation == "elu" else torch.relu(t)
    loss_fn(t, labels, mask).backward()
    return t.detach().numpy(), [w.grad.numpy() for w in ws]
