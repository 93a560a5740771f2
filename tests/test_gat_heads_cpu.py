"""Per-head GAT scores and ELU without a GPU: the fp64 references the GPU tests check against (scores_ref /
scores_bwd_ref, elu_ref / elu_bwd_ref) against torch; build_gat's wiring for every scores x activation on a recorder
with no product behind it; the refusal of unknown values; and a register / spill check of every new kernel.

The references live here so that tests/test_gat_heads_gpu.py can import them."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from conftest import ROOT
from opgraph import Recorder
from roc_b200.model import build_gat


# ---------------------------------------------------------------------------------------- the fp64 references ---
def scores_ref(x, a, heads):
    """S [rows][2 * heads] = [s_dst | s_src] in fp64 from x [rows][H] and a [2 * heads][F] (numpy or torch), and the
    bound's sum: B[v][j] = sum_f |a[j][f] x[v][kF + f]| for the head k of output j."""
    x, a = torch.as_tensor(x).double(), torch.as_tensor(a).double()
    rows, h = x.shape
    f = h // heads
    xv = x.reshape(rows, heads, f)
    s = torch.cat([(xv * a[:heads]).sum(2), (xv * a[heads:]).sum(2)], 1)
    b = torch.cat([(xv.abs() * a[:heads].abs()).sum(2), (xv.abs() * a[heads:].abs()).sum(2)], 1)
    return s, b


def scores_bwd_ref(x, a, ds, heads):
    """The backward in fp64: dx [rows][H], da [2 * heads][F], and the bound terms: |gd ad| + |gs as| per element of dx,
    sum_v |g x| per element of da."""
    x, a, ds = torch.as_tensor(x).double(), torch.as_tensor(a).double(), torch.as_tensor(ds).double()
    rows, h = x.shape
    f = h // heads
    gd, gs = ds[:, :heads, None], ds[:, heads:, None]
    t1, t2 = gd * a[:heads], gs * a[heads:]                  # [rows][heads][F]
    xv = x.reshape(rows, heads, f)
    da = torch.cat([(gd * xv).sum(0), (gs * xv).sum(0)], 0)
    da_abs = torch.cat([(gd * xv).abs().sum(0), (gs * xv).abs().sum(0)], 0)
    return dict(dx=(t1 + t2).reshape(rows, h), dx_abs=(t1.abs() + t2.abs()).reshape(rows, h), da=da, da_abs=da_abs)


def elu_ref(x):
    """ELU (alpha 1) in fp64: x > 0 ? x : expm1(x), NaN kept"""
    x = torch.as_tensor(x).double()
    return torch.where(x > 0, x, torch.expm1(x))


def elu_bwd_ref(y, g):
    """dx = g * (y > 0 ? 1 : y + 1) in fp64, from the output y (NaN where y is NaN)"""
    y, g = torch.as_tensor(y).double(), torch.as_tensor(g).double()
    return g * torch.where(y > 0, torch.ones_like(y), y + 1)


@pytest.mark.parametrize("rows,heads,f", [(1, 1, 1), (7, 1, 3), (50, 2, 4), (33, 3, 5), (20, 8, 8), (9, 1, 41)])
def test_scores_reference_matches_torch(rows, heads, f):
    gen = torch.Generator().manual_seed(rows * 13 + heads * 7 + f)
    wh = torch.randn(rows, heads * f, generator=gen, dtype=torch.float64, requires_grad=True)
    a = torch.randn(2 * heads, f, generator=gen, dtype=torch.float64, requires_grad=True)
    go = torch.randn(rows, 2 * heads, generator=gen, dtype=torch.float64)
    v = wh.view(rows, heads, f)
    want = torch.cat([torch.einsum("rkf,kf->rk", v, a[:heads]), torch.einsum("rkf,kf->rk", v, a[heads:])], 1)
    s, b = scores_ref(wh.detach(), a.detach(), heads)
    assert torch.allclose(s, want.detach(), rtol=1e-12, atol=1e-12)
    assert bool((s.abs() <= b + 1e-12).all())
    want.backward(go)
    r = scores_bwd_ref(wh.detach(), a.detach(), go, heads)
    assert torch.allclose(r["dx"], wh.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(r["da"], a.grad, rtol=1e-12, atol=1e-12)
    assert bool((r["dx"].abs() <= r["dx_abs"] + 1e-12).all()) and bool((r["da"].abs() <= r["da_abs"] + 1e-12).all())


def test_elu_reference_matches_torch():
    x = torch.tensor([0.0, -0.0, 1.5, -1.5, -25.0, 1e-40, -1e-40, float("inf"), float("-inf"), 3e38, -1e-3],
                     dtype=torch.float64)
    x = torch.cat([x, torch.randn(200, generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 5])
    assert torch.equal(elu_ref(x), torch.nn.functional.elu(x))
    assert torch.isnan(elu_ref(torch.tensor([float("nan")]))).all()
    xr = x[torch.isfinite(x)].clone().requires_grad_(True)
    g = torch.randn(xr.shape, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    torch.nn.functional.elu(xr).backward(g)
    y = elu_ref(xr.detach())
    # torch's input-form backward takes exp(x), ours y + 1: they differ by fp64 rounding of y + 1 (absolute in y)
    assert bool(((elu_bwd_ref(y, g) - xr.grad).abs() <= 4 * 2.0 ** -53 * g.abs() * (y.abs() + 1)).all())


# ------------------------------------------------------------------------------------------ build_gat's wiring ---
@pytest.mark.parametrize("scores", ["dense", "per_head"])
@pytest.mark.parametrize("activation", ["relu", "elu"])
@pytest.mark.parametrize("heads", [1, 4, [2, 8]])
def test_build_gat_wiring(scores, activation, heads):
    layers = [24, 16, 32, 12] if isinstance(heads, list) else [24, 16, 12]
    plain, ir = Recorder(None), Recorder(None)
    build_gat(plain, layers, 0.5, heads=heads)
    h = build_gat(ir, layers, 0.5, heads=heads, scores=scores, activation=activation)
    hs = (heads if isinstance(heads, list) else [heads] * (len(layers) - 2)) + [1]
    producer = {n["out"]: n for n in ir.nodes}
    # the score op of every layer reads wh and feeds the attention_gather's scores
    gathers = [n for n in ir.nodes if n["kind"] == "attention_gather"]
    assert len(gathers) == len(layers) - 1 and [n["out"] for n in gathers] == h["attn"]
    for g, k, wh, sc in zip(gathers, hs, h["attn_ins"], h["scores"]):
        assert g["ins"] == [wh, sc] and g["attrs"]["heads"] == k
        s = producer[sc]
        assert s["ins"] == [wh] and ir.width[sc] == 2 * k
        if scores == "per_head":
            assert s["kind"] == "attention_scores" and s["attrs"]["heads"] == k
        else:
            assert s["kind"] == "linear" and s["attrs"]["out_dim"] == 2 * k
    # every hidden activation is the chosen one, reads an attention output, and the last layer has none
    acts = [n for n in ir.nodes if n["kind"] in ("relu", "elu")]
    assert [n["kind"] for n in acts] == [activation] * (len(layers) - 2) and [n["out"] for n in acts] == h["relu_outs"]
    for n in acts:
        assert producer[n["ins"][0]]["kind"] == "attention_gather"
    # the same parameters in the same order, and otherwise the default model's nodes
    assert ir.params == plain.params
    swap = {"attention_scores": "linear", "elu": "relu"}
    assert [swap.get(n["kind"], n["kind"]) for n in ir.nodes] == [n["kind"] for n in plain.nodes]
    if scores == "dense" and activation == "relu":
        assert [(n["kind"], n["ins"], n["out"], n["attrs"]) for n in ir.nodes] == \
            [(n["kind"], n["ins"], n["out"], n["attrs"]) for n in plain.nodes]


def test_build_gat_with_batch_norm_puts_it_before_the_elu():
    ir = Recorder(None)
    h = build_gat(ir, [24, 16, 12], 0.5, heads=2, scores="per_head", activation="elu", norm="batch")
    producer = {n["out"]: n for n in ir.nodes}
    (e,) = [n for n in ir.nodes if n["kind"] == "elu"]
    assert producer[e["ins"][0]]["kind"] == "batch_norm" and h["bns"] == [e["ins"][0]]


@pytest.mark.parametrize("kw", [dict(scores="perhead"), dict(scores=""), dict(scores=None), dict(activation="ELU"),
                                dict(activation="gelu"), dict(activation=None)])
def test_build_gat_refuses_unknown_values(kw):
    with pytest.raises(ValueError):
        build_gat(Recorder(None), [24, 16, 12], 0.5, heads=2, **kw)


# -------------------------------------------------------------------------------------------------- the kernels ---
def _ptxas(tmp_path, src):
    nvcc = os.path.join(os.environ.get("CUDA", "/usr/local/cuda"), "bin", "nvcc")
    if not os.path.exists(nvcc):
        nvcc = shutil.which("nvcc")
    if not nvcc:
        pytest.skip("no nvcc")
    p = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                        "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "roc_b200", "csrc"), "-c",
                        os.path.join(ROOT, "roc_b200", "csrc", src), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True, check=True)
    return re.split(r"Compiling entry function", p.stderr)


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    blocks = _ptxas(tmp_path, "attn_scores.cu")
    mine = [b for b in blocks if "k_attn_scores" in b.split("\n")[0]]
    assert len(mine) == 9, "fwd and bwd x fp32 / bf16 x vector / element loads, and the finalize"
    # the ELU forward and backward maps (OP_ELU_F = 6, OP_ELU_B = 7) at both vector widths
    elu = [b for b in _ptxas(tmp_path, "elementwise.cu") if re.search(r"k_mapILi[67]E", b.split("\n")[0])]
    assert len(elu) == 6, "forward at 2 widths, backward at 2 widths x accumulate"
    for b in mine + elu:
        assert "0 bytes spill stores, 0 bytes spill loads" in b, b
        regs = int(re.search(r"Used (\d+) registers", b).group(1))
        assert regs <= 128, b       # 256 threads per CTA
