"""GATv2's dynamic attention without a GPU: the fp64 witness of tests/gatv2_witness.py against a per-edge restatement
of the formulas (loops over rows and heads, torch autograd for the gradients), shared and separate inputs; build_gatv2's
op graph on a recorder and its ValueErrors; and a check that the new kernels of sg.cu compiled without local memory or
a stack frame."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from gatv2_witness import kernel_witness
from opgraph import Recorder
from roc_b200 import _lib
from roc_b200.model import build_gatv2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _loop_gatv2(row_end, col, xl, xr, a, heads, slope):
    """the formulas of include/roc_b200.h, one row and one head at a time"""
    n, h = xr.shape
    f = h // heads
    rows = []
    for v in range(n):
        s, t = (int(row_end[v - 1]) if v else 0), int(row_end[v])
        out = []
        for k in range(heads):
            sl = slice(k * f, (k + 1) * f)
            if s == t:
                out.append(torch.zeros(f, dtype=torch.float64))
                continue
            es = []
            for e in range(s, t):
                z = xl[int(col[e]), sl] + xr[v, sl]
                es.append((a[k] * torch.where(z > 0, z, slope * z)).sum())
            p = torch.softmax(torch.stack(es), 0)
            out.append(sum(p[i] * xl[int(col[s + i]), sl] for i in range(t - s)))
        rows.append(torch.cat(out))
    return torch.stack(rows)


def _graph(n, edges, seed):
    rng = np.random.RandomState(seed)
    pairs = sorted([(i, i) for i in range(n)] + [tuple(rng.randint(0, n, 2)) for _ in range(edges)] + [(1, 2)] * 2)
    dst = np.array([p[0] for p in pairs])
    col = np.array([p[1] for p in pairs], dtype=np.uint32)
    return np.cumsum(np.bincount(dst, minlength=n)).astype(np.uint64), col


@pytest.mark.parametrize("h,heads,shared", [(1, 1, False), (6, 3, False), (8, 2, True), (5, 5, False)])
def test_witness_matches_the_per_edge_formulas(h, heads, shared):
    row_end, col = _graph(9, 25, seed=h + heads)
    rng = np.random.RandomState(1)
    xl = rng.standard_normal((9, h))
    xr = xl if shared else rng.standard_normal((9, h))
    a = rng.uniform(-1, 1, (heads, h // heads))
    gy = rng.standard_normal((9, h))
    w = kernel_witness(row_end, col, xl, xr, a, gy, heads, 0.2)
    tl = torch.tensor(xl, requires_grad=True)
    tr = tl if shared else torch.tensor(xr, requires_grad=True)
    ta = torch.tensor(a, requires_grad=True)
    y = _loop_gatv2(row_end, col, tl, tr, ta, heads, 0.2)
    (y * torch.from_numpy(gy)).sum().backward()
    np.testing.assert_allclose(w["out"], y.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(w["dxl"], tl.grad.numpy(), rtol=1e-10, atol=1e-12)
    if not shared:
        np.testing.assert_allclose(w["dxr"], tr.grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(w["da"], ta.grad.numpy(), rtol=1e-10, atol=1e-12)


class V2Recorder(Recorder):
    """Recorder with Model.dynamic_attention_gather, recorded as the attention_gather it reports as"""

    def dynamic_attention_gather(self, xl, xr, heads=1, negative_slope=0.2):
        self.params += 1
        return self._node("attention_gather", [xl, xr], self._call("dynamic_attention_gather", xl, xr, heads,
                                                                   negative_slope),
                          width=self.width[xl], heads=int(heads), slope=float(np.float32(negative_slope)),
                          dynamic=True, param=self.params - 1)


@pytest.mark.parametrize("share", [False, True])
def test_build_gatv2_op_graph(share):
    ir = V2Recorder(None)
    h = build_gatv2(ir, [12, 16, 6], 0.5, heads=4, share_weights=share, norm="batch", activation="elu")
    kinds = [n["kind"] for n in ir.nodes]
    lin = ["linear"] if share else ["linear", "linear"]
    assert kinds == (["dropout"] + lin + ["attention_gather", "batch_norm", "elu"] + ["dropout"] + lin +
                     ["attention_gather", "softmax_cross_entropy"])
    attn = [n for n in ir.nodes if n["kind"] == "attention_gather"]
    assert [n["attrs"]["heads"] for n in attn] == [4, 1]
    for n, (xl, xr) in zip(attn, h["attn_ins"]):
        assert n["ins"] == [xl, xr] and (xl == xr) == share
    assert h["attn"] == [n["out"] for n in attn] and len(h["relu_outs"]) == 1


@pytest.mark.parametrize("kw", [dict(activation="tanh"), dict(norm="layer"), dict(heads=0), dict(heads=9),
                                dict(heads=3), dict(heads=2.0), dict(heads=[2, 2]), dict(heads=True)])
def test_build_gatv2_refusals(kw):
    with pytest.raises(ValueError):
        build_gatv2(V2Recorder(None), [12, 16, 6], 0.5, **kw)


def test_entry_points_are_declared():
    for name in ("roc_sg_attn_v2_forward_planned", "roc_sg_attn_v2_backward_planned", "roc_sg_attn_v2_backward_exact",
                 "roc_host_dynamic_attention_gather"):
        assert name in _lib.PROTOTYPES
    assert len(_lib.HOST_OPS) == 17 and _lib.SG_LAUNCH_KINDS[-1] == "colsum"


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
    v2 = [f for f in found if re.search(r"sg_v2_", f)]
    assert len(v2) == 8 * 4 + 8 + 2, len(v2)
    for f in v2:
        assert re.search(r"STACK:0\b", found[f]) and re.search(r"LOCAL:0\b", found[f]), (f, found[f])
