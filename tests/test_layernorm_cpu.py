"""Layer normalisation without a GPU: the fp64 witness of tests/layernorm_witness.py against a numpy per-row restatement
of the formulas in include/roc_b200.h (the closed-form dx included); every builder's op graph with norm="layer_norm"
on a recorder against its norm="batch" graph; Model.layer_norm's ValueErrors; the entry points declared and bound;
and a check that the new kernels compiled without local memory or a stack frame."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from layernorm_witness import LN_EPS, kernel_witness
from opgraph import Recorder
from roc_b200 import _lib
from roc_b200.model import (Model, build_deepergcn, build_gat, build_gatv2, build_gcn, build_gcn_weighted,
                            build_sage_mean, build_sage_pool)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rows(x, gy, gamma, beta, eps, relu):
    """include/roc_b200.h's formulas, one row at a time, in fp64"""
    n, h = x.shape
    y, dx = np.zeros((n, h)), np.zeros((n, h))
    dgamma, dbeta = np.zeros(h), np.zeros(h)
    for r in range(n):
        mu = x[r].sum() / h
        var = ((x[r] - mu) ** 2).sum() / h
        rstd = 1.0 / np.sqrt(var + eps)
        xhat = (x[r] - mu) * rstd
        pre = xhat * gamma + beta
        y[r] = np.where(pre > 0, pre, 0.0) if relu else pre
        g = np.where(pre > 0, gy[r], 0.0) if relu else gy[r]
        gh = g * gamma
        dx[r] = rstd * (gh - gh.mean() - xhat * (gh * xhat).mean())
        dgamma += g * xhat
        dbeta += g
    return y, dx, dgamma, dbeta


@pytest.mark.parametrize("h", [1, 2, 5, 33])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("shift", [0.0, 1e4])
def test_witness_matches_the_row_formulas(h, relu, shift):
    rng = np.random.RandomState(h * 7 + int(relu))
    x = rng.standard_normal((9, h)) + shift
    x[3] = 2.5                                   # a constant row: var 0
    gy = rng.standard_normal((9, h))
    gamma, beta = rng.rand(h) + 0.5, rng.standard_normal(h)
    w = kernel_witness(torch.from_numpy(x), torch.from_numpy(gy), torch.from_numpy(gamma), torch.from_numpy(beta),
                       LN_EPS, relu)
    y, dx, dgamma, dbeta = _rows(x, gy, gamma, beta, LN_EPS, relu)
    np.testing.assert_allclose(w["y"].numpy(), y, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(w["dx"].numpy(), dx, rtol=1e-7, atol=1e-7)
    np.testing.assert_allclose(w["dgamma"].numpy(), dgamma, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(w["dbeta"].numpy(), dbeta, rtol=1e-12, atol=1e-12)
    if h == 1:                                   # y = beta and dx = 0
        np.testing.assert_allclose(w["pre"].numpy()[:, 0], beta[0], rtol=0, atol=0)
        assert not dx.any() and np.abs(w["dx"].numpy()).max() < 1e-12


# ------------------------------------------------------------------------------------------ builders' wiring ---
BUILDERS = {
    "gcn": lambda ir, **kw: build_gcn(ir, [24, 16, 12], 0.5, **kw),
    "gcn4": lambda ir, **kw: build_gcn(ir, [24, 16, 16, 12], 0.5, **kw),
    "sage_mean": lambda ir, **kw: build_sage_mean(ir, [24, 16, 16, 12], 0.5, **kw),
    "sage_pool": lambda ir, **kw: build_sage_pool(ir, [24, 16, 12], 0.5, **kw),
    "gat": lambda ir, **kw: build_gat(ir, [24, 16, 12], 0.5, heads=2, **kw),
    "gat_per_head": lambda ir, **kw: build_gat(ir, [24, 16, 12], 0.5, heads=2, scores="per_head", activation="elu",
                                               **kw),
    "gatv2": lambda ir, **kw: build_gatv2(ir, [24, 16, 12], 0.5, heads=2, **kw),
    "gcn_weighted": lambda ir, **kw: build_gcn_weighted(ir, [24, 16, 12], 0.5, (), **kw),
    "deepergcn": lambda ir, **kw: build_deepergcn(ir, [24, 16, 12], 0.5, 3, **kw),
}


@pytest.mark.parametrize("name", list(BUILDERS))
def test_layer_norm_sits_where_batch_norm_does(name):
    bn, ln = Recorder(None), Recorder(None)
    hb = BUILDERS[name](bn, norm="batch")
    hl = BUILDERS[name](ln, norm="layer_norm")
    assert [n["kind"] for n in ln.nodes] == [("layer_norm" if n["kind"] == "batch_norm" else n["kind"])
                                             for n in bn.nodes]
    assert [n["ins"] for n in ln.nodes] == [n["ins"] for n in bn.nodes]
    assert ln.params == bn.params
    lns, bns = [n for n in ln.nodes if n["kind"] == "layer_norm"], [n for n in bn.nodes if n["kind"] == "batch_norm"]
    assert lns and [(n["attrs"]["gamma"], n["attrs"]["beta"]) for n in lns] == \
        [(n["attrs"]["gamma"], n["attrs"]["beta"]) for n in bns]
    assert hl["bns"] == [n["out"] for n in lns] and len(hl["bns"]) == len(hb["bns"])
    assert all(n["attrs"]["eps"] == float(np.float32(1e-5)) for n in lns)


@pytest.mark.parametrize("name", list(BUILDERS))
def test_defaults_are_unchanged(name):
    """no builder puts a layer_norm in unless asked"""
    ir = Recorder(None)
    BUILDERS[name](ir)
    assert all(n["kind"] != "layer_norm" for n in ir.nodes)


@pytest.mark.parametrize("name", list(BUILDERS))
@pytest.mark.parametrize("bad", ["layer", "LayerNorm", "layernorm", "Layer_norm"])
def test_other_spellings_are_refused(name, bad):
    with pytest.raises(ValueError):
        BUILDERS[name](Recorder(None), norm=bad)


@pytest.mark.parametrize("eps", [-1e-5, float("nan"), float("inf"), -float("inf"), 1e39])
def test_layer_norm_refuses_a_bad_eps(eps):
    m = Model.__new__(Model)        # the check runs before the product is called
    m.h = None
    with pytest.raises(ValueError):
        m.layer_norm(0, eps=eps)


def test_entry_points_are_declared():
    names = ("roc_layernorm_fwd", "roc_layernorm_bwd", "roc_layernorm_workspace_bytes", "roc_host_layer_norm")
    for name in names:
        assert name in _lib.PROTOTYPES
        assert getattr(_lib.lib, name) is not None
    with open(os.path.join(ROOT, "include", "roc_b200.h")) as f:
        text = f.read()
    for name in names[:2]:
        assert re.search(r"\bint %s\(" % name, text)
    assert re.search(r"\bsize_t roc_layernorm_workspace_bytes\(", text)
    with open(os.path.join(ROOT, "include", "roc_host.h")) as f:
        assert re.search(r"\bint roc_host_layer_norm\(", f.read())
    assert len(_lib.HOST_OPS) == 17     # reported as batch_norm: no new op kind


def test_new_kernels_use_no_local_memory():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            found[name] = line
            name = None
    ln = [f for f in found if re.search(r"k_ln_", f)]
    # (S, J) shapes: S in {1, 2, 4, 8, 16, 32} at J = 1, and S = 32 at J = 2..7: 12.  Forward x relu 2, backward x
    # relu x accumulate 4, each also as the wide path; and the finalize.
    assert len(ln) == 12 * 2 + 12 * 4 + 2 + 4 + 1, len(ln)
    for f in ln:
        assert re.search(r"STACK:0\b", found[f]) and re.search(r"LOCAL:0\b", found[f]), (f, found[f])
