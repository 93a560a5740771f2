"""Batch normalisation without a GPU: the builders' wiring with norm="batch" on a recorder with no product behind it,
the refusal of an unknown norm, and the fp64 reference the GPU tests check against (bn_forward / bn_backward) against
torch.nn.functional.batch_norm's forward and autograd in fp64.

The reference lives here so that tests/test_batchnorm_gpu.py can import it."""
import numpy as np
import pytest
import torch

from opgraph import Recorder
from roc_b200.model import build_gat, build_gcn, build_gcn_weighted, build_sage_mean, build_sage_pool


# ---------------------------------------------------------------------------------------- the fp64 reference ---
def bn_forward(x, gamma, beta, run_mean, run_var, training=True, eps=1e-5, momentum=0.1):
    """torch.nn.BatchNorm1d's forward in fp64 on [N][H] tensors (any device): returns y (before any relu), a, b (the
    affine map y = x a + b), the batch mean and biased variance (None in eval), and the new running statistics."""
    x = x.double()
    g, bt = gamma.double(), beta.double()
    rm, rv = run_mean.double(), run_var.double()
    if training:
        n = x.shape[0]
        mean = x.mean(0)
        var = ((x - mean) ** 2).mean(0)
        rm = (1 - momentum) * rm + momentum * mean
        rv = (1 - momentum) * rv + momentum * var * n / (n - 1)
        use_m, use_v = mean, var
    else:
        mean = var = None
        use_m, use_v = rm, rv
    a = g / torch.sqrt(use_v + eps)
    b = bt - use_m * a
    return dict(y=(x - use_m) * a + bt, a=a, b=b, mean=mean, var=var, run_mean=rm, run_var=rv)


def bn_backward(x, g, gamma, mean, var, eps=1e-5):
    """The training backward in fp64 from the output gradient g (already relu-masked): dx, dgamma, dbeta, and the terms
    A g, B x, C whose sum is dx (A = gamma invstd, B = -A invstd dgamma / N, C = -A dbeta / N - B mean)."""
    x, g = x.double(), g.double()
    n = x.shape[0]
    s = 1.0 / torch.sqrt(var + eps)
    xhat = (x - mean) * s
    dbeta = g.sum(0)
    dgamma = (g * xhat).sum(0)
    A = gamma.double() * s
    B = -A * s * dgamma / n
    C = -A * dbeta / n - B * mean
    return dict(dx=A * (g - dbeta / n - xhat * dgamma / n), dgamma=dgamma, dbeta=dbeta, Ag=A * g, Bx=B * x,
                C=C.expand_as(x), gxhat=g * xhat)


@pytest.mark.parametrize("rows,h", [(2, 1), (3, 5), (100, 7), (257, 16)])
@pytest.mark.parametrize("shift", [0.0, 1e4])
def test_reference_matches_torch_batch_norm(rows, h, shift):
    gen = torch.Generator().manual_seed(rows * 31 + h)
    x = torch.randn(rows, h, generator=gen, dtype=torch.float64) + shift
    x[:, 0] = 2.5                                      # a constant column: var 0
    gamma = torch.rand(h, generator=gen, dtype=torch.float64) + 0.5
    beta = torch.randn(h, generator=gen, dtype=torch.float64)
    rm0 = torch.randn(h, generator=gen, dtype=torch.float64)
    rv0 = torch.rand(h, generator=gen, dtype=torch.float64) + 0.5
    go = torch.randn(rows, h, generator=gen, dtype=torch.float64)
    for training in (True, False):
        xr, gr, br = x.clone().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        rm, rv = rm0.clone(), rv0.clone()
        y = torch.nn.functional.batch_norm(xr, rm, rv, gr, br, training=training, momentum=0.1, eps=1e-5)
        ours = bn_forward(x, gamma, beta, rm0, rv0, training=training)
        assert torch.allclose(ours["y"], y.detach(), rtol=1e-12, atol=1e-9)
        assert torch.allclose(ours["y"], x * ours["a"] + ours["b"], rtol=1e-12, atol=1e-9 * (1 + shift))
        assert torch.allclose(ours["run_mean"], rm, rtol=1e-14, atol=1e-14)
        assert torch.allclose(ours["run_var"], rv, rtol=1e-14, atol=1e-14)
        if training:
            y.backward(go)
            bwd = bn_backward(x, go, gamma, ours["mean"], ours["var"])
            assert torch.allclose(bwd["dx"], xr.grad, rtol=1e-9, atol=1e-9)
            assert torch.allclose(bwd["Ag"] + bwd["Bx"] + bwd["C"], xr.grad, rtol=1e-9, atol=1e-8 * (1 + shift))
            assert torch.allclose(bwd["dgamma"], gr.grad, rtol=1e-10, atol=1e-10)
            assert torch.allclose(bwd["dbeta"], br.grad, rtol=1e-12, atol=1e-12)


def test_running_statistics_recurrence():
    """three training forwards chain run_mean / run_var from 0 / 1 as torch's module does"""
    gen = torch.Generator().manual_seed(3)
    bn = torch.nn.BatchNorm1d(6).double()
    rm, rv = torch.zeros(6, dtype=torch.float64), torch.ones(6, dtype=torch.float64)
    for _ in range(3):
        x = torch.randn(50, 6, generator=gen, dtype=torch.float64) * 3 + 1
        bn(x)
        r = bn_forward(x, bn.weight.detach(), bn.bias.detach(), rm, rv)
        rm, rv = r["run_mean"], r["run_var"]
    assert torch.allclose(rm, bn.running_mean) and torch.allclose(rv, bn.running_var)


# ------------------------------------------------------------------------------------------ builders' wiring ---
BUILDERS = {
    "gcn": lambda ir, **kw: build_gcn(ir, [24, 16, 12], 0.5, **kw),
    "gcn4": lambda ir, **kw: build_gcn(ir, [24, 16, 16, 12], 0.5, **kw),
    "sage_mean": lambda ir, **kw: build_sage_mean(ir, [24, 16, 16, 12], 0.5, **kw),
    "sage_pool": lambda ir, **kw: build_sage_pool(ir, [24, 16, 12], 0.5, **kw),
    "gat": lambda ir, **kw: build_gat(ir, [24, 16, 12], 0.5, heads=2, **kw),
    "gcn_weighted": lambda ir, edge_weights=(), **kw: build_gcn_weighted(ir, [24, 16, 12], 0.5, edge_weights, **kw),
}


HIDDEN = {"gcn": 1, "gcn4": 2, "sage_mean": 2, "sage_pool": 1, "gat": 1, "gcn_weighted": 1}


def _consumers(ir, t):
    return [n for n in ir.nodes if t in n["ins"]]


@pytest.mark.parametrize("name", list(BUILDERS))
def test_builder_puts_batch_norm_before_every_hidden_relu(name):
    plain, ir = Recorder(None), Recorder(None)
    BUILDERS[name](plain)
    h = BUILDERS[name](ir, norm="batch")
    bns = [n for n in ir.nodes if n["kind"] == "batch_norm"]
    assert len(bns) == HIDDEN[name] and h["bns"] == [n["out"] for n in bns]
    producer = {n["out"]: n for n in ir.nodes}
    for r in h.get("relu_outs", []):                    # every hidden layer's relu reads a batch_norm
        assert producer[producer[r]["ins"][0]]["kind"] == "batch_norm"
    for n in bns:
        (c,) = _consumers(ir, n["out"])                 # read by exactly one op: its relu
        assert c["kind"] == "relu"
        assert n["attrs"]["beta"] == n["attrs"]["gamma"] + 1
    # two parameters per batch_norm, and every other node as without norm
    assert ir.params == plain.params + 2 * len(bns)
    assert [n["kind"] for n in ir.nodes if n["kind"] != "batch_norm"] == [n["kind"] for n in plain.nodes]
    # the last layer has none: nothing between the last relu-free layer and the loss is a batch_norm
    loss = ir.nodes[-1]
    assert producer[loss["ins"][0]]["kind"] != "batch_norm"
    last_relu = max(n["layer"] for n in ir.nodes if n["kind"] == "relu")
    assert all(n["layer"] < last_relu for n in bns)
    if name.startswith("gcn") and name != "gcn_weighted":
        for n in bns:                                   # after the second indegree_norm
            assert producer[n["ins"][0]]["kind"] == "indegree_norm"
    if name == "gcn4":                                  # the relu after each BN feeds the residual add
        for n in bns:
            (r,) = _consumers(ir, n["out"])
            assert any(c["kind"] == "add" for c in _consumers(ir, r["out"]))


@pytest.mark.parametrize("name", list(BUILDERS))
@pytest.mark.parametrize("bad", ["layer", "Batch", "", 1])
def test_builder_refuses_an_unknown_norm(name, bad):
    with pytest.raises(ValueError):
        BUILDERS[name](Recorder(None), norm=bad)
