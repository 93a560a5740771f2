"""CPU checks of the multi-label sigmoid cross-entropy: the metrics struct's ctypes layout, the label packing, the fp64
oracle against torch, the synthetic multi-label data, and the kernel's register budget."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from multilabel_oracle import element_loss, sigmoid_xent, unpack_multilabels
from roc_b200 import _lib, datasets
from roc_b200.model import pack_multilabels


def test_multilabel_metrics_layout_matches_the_header(tmp_path):
    """MultilabelMetrics has roc_multilabel_metrics' C layout: a C program prints sizeof / offsetof of every field."""
    py = _lib.MultilabelMetrics
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "roc_b200.h"', 'int main(void) {',
            '  printf("%zu\\n", sizeof(roc_multilabel_metrics));']
    prog += ['  printf("%%zu\\n", offsetof(roc_multilabel_metrics, %s));' % f for f, _ in py._fields_]
    prog += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out[0] == C.sizeof(py) == 144
    assert [getattr(py, f).offset for f, _ in py._fields_] == out[1:]


@pytest.mark.parametrize("c", [1, 5, 31, 32, 33, 64, 112, 129])
def test_pack_multilabels_round_trips(c):
    rng = np.random.RandomState(c)
    y = rng.rand(37, c) < 0.3
    bits = pack_multilabels(y)
    w = (c + 31) // 32
    assert bits.dtype == np.uint32 and bits.shape == (37, w) and bits.flags["C_CONTIGUOUS"]
    assert np.array_equal(unpack_multilabels(bits, c), y.astype(np.uint8))
    # the layout itself: bit c % 32 of word c // 32, nothing past C
    for r in range(5):
        for k in range(c):
            assert ((int(bits[r, k // 32]) >> (k % 32)) & 1) == int(y[r, k])
        if c % 32:
            assert int(bits[r, -1]) >> (c % 32) == 0
    assert np.array_equal(pack_multilabels(y.astype(np.uint8)), bits)      # 0/1 ints pack as bools do


def test_oracle_loss_matches_torch_bce():
    rng = np.random.RandomState(3)
    special = np.array([0.0, -0.0, 1e-3, -1e-3, 20.0, -20.0, 100.0, -100.0, 1e30, -1e30], dtype=np.float32)
    z = np.concatenate([rng.randn(200, 41).astype(np.float32) * 4, np.tile(special, (200, 5))[:, :41]])
    y = rng.rand(400, 41) < 0.2
    want = torch.nn.functional.binary_cross_entropy_with_logits(
        torch.from_numpy(z.astype(np.float64)), torch.from_numpy(y.astype(np.float64)), reduction="none").numpy()
    # torch takes log(1 + e^-|z|) where the oracle takes log1p: they differ by ~1e-16 absolute where the loss is tiny
    assert np.allclose(element_loss(z, y), want, rtol=1e-13, atol=1e-14)
    mask = rng.randint(0, 4, size=400)
    g, m = sigmoid_xent(z, y, mask)
    zt = torch.from_numpy(z.astype(np.float64)).requires_grad_(True)
    train = torch.from_numpy(mask == 0)
    torch.nn.functional.binary_cross_entropy_with_logits(zt[train], torch.from_numpy(y.astype(np.float64))[train],
                                                         reduction="sum").backward()
    assert np.allclose(g, zt.grad.numpy(), rtol=0, atol=1e-15)
    for s in range(3):
        r = mask == s
        assert m["rows"][s] == r.sum()
        assert np.isclose(m["loss"][s], want[r].sum(), rtol=1e-13)
        pred = z[r] > 0
        assert m["tp"][s] + m["fn"][s] == y[r].sum()
        assert m["tp"][s] + m["fp"][s] == pred.sum()
        assert m["exact"][s] == sum(np.array_equal(p, t) for p, t in zip(pred, y[r]))
    # z == 0 (either sign) and NaN are negative predictions
    _, m0 = sigmoid_xent(np.array([[0.0, -0.0, np.nan]], np.float32), np.array([[0, 0, 0]]), np.array([0]))
    assert m0["fp"][0] == 0 and m0["exact"][0] == 1


def test_oracle_fused_norm_divides_by_sqrt_degree():
    rng = np.random.RandomState(5)
    z = rng.randn(50, 7).astype(np.float32)
    y = rng.rand(50, 7) < 0.5
    mask = np.zeros(50, dtype=np.int32)
    deg = rng.randint(1, 9, size=50)
    g0, _ = sigmoid_xent(z, y, mask)
    g1, _ = sigmoid_xent(z, y, mask, deg)
    assert np.allclose(g1 * np.sqrt(deg)[:, None], g0, rtol=1e-14)


def test_multilabel_node_data_is_deterministic_with_the_stated_rate():
    a = datasets.multilabel_node_data(5000, 32, 112, seed=3)
    b = datasets.multilabel_node_data(5000, 32, 112, seed=3)
    c = datasets.multilabel_node_data(5000, 32, 112, seed=4)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert not torch.equal(a[1], c[1])
    feats, labels, mask = a
    assert feats.shape == (5000, 32) and feats.dtype == torch.float32
    assert float(feats.min()) >= -1.0 and float(feats.max()) <= 1.0
    assert labels.shape == (5000, 112) and set(np.unique(labels.numpy())) <= {0, 1}
    assert abs(float(labels.double().mean()) - 0.1) < 0.01
    m = mask.numpy()
    assert set(np.unique(m)) == {0, 1, 2}
    assert abs((m == 0).mean() - 0.66) < 0.03 and abs((m == 1).mean() - 0.10) < 0.02
    # the labels depend on the features: a least-squares fit on them beats the all-negative predictor's F1 of 0
    x = np.c_[feats.numpy().astype(np.float64), np.ones(5000)]
    w = np.linalg.lstsq(x, labels.numpy().astype(np.float64) - 0.5, rcond=None)[0]
    pred = x @ w > np.quantile(x @ w, 0.9)
    y = labels.numpy().astype(bool)
    tp = (pred & y).sum()
    assert 2 * tp / (2 * tp + (pred & ~y).sum() + (~pred & y).sum()) > 0.5


def test_sigmoid_kernel_compiles_for_sm90a_without_spills(tmp_path):
    nvcc = os.path.join(os.environ.get("CUDA", "/usr/local/cuda"), "bin", "nvcc")
    if not os.path.exists(nvcc):
        nvcc = shutil.which("nvcc")
    if not nvcc:
        pytest.skip("no nvcc")
    p = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                        "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "roc_b200", "csrc"), "-c",
                        os.path.join(ROOT, "roc_b200", "csrc", "elementwise.cu"), "-o", str(tmp_path / "ew.o")],
                       capture_output=True, text=True, check=True)
    blocks = re.split(r"Compiling entry function", p.stderr)
    mine = [b for b in blocks if "k_sigmoid_xent" in b.split("\n")[0]]
    assert len(mine) == 12, "2 vector widths x 6 row widths"
    for b in mine:
        assert "0 bytes spill stores, 0 bytes spill loads" in b, b
        regs = int(re.search(r"Used (\d+) registers", b).group(1))
        assert regs <= 64, b      # __launch_bounds__(256, 4)
