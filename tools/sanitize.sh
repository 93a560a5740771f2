#!/bin/bash
# compute-sanitizer over the tiny configuration (SURVEY §5): memcheck, then racecheck, on
#   (a) __graft_entry__.smoke()  — one GCN training step through the Model API (SG, wgmma GEMMs, softmax, Adam)
#   (b) the ScatterGather sum with the fused epilogue on a small R-MAT graph at 41, 64, 100, 200 and 602 floats, each
#       followed by one max-aggregation forward and backward; then the attention forward and backward at 41 and 64
#       floats with one head and at 64 and 256 floats with eight, on float4 rows, and at 256 floats with two heads on
#       rows of 257 floats (the scalar path); then the edge-weighted forward, its transposed backward and the edge
#       dot (overwriting, then accumulating) at 41, 64, 200 and 602 floats; then the exact sum (with norm and relu)
#       and min backwards over the transpose at the same widths, and the exact attention backward at 41 floats with
#       one head and 64 with eight;
#   (c) the warp-specialised dW kernel at 602 x 64 with the dropout mask and at 64 x 41, on rows that wrap its ring
#       and end in a partial block.
# Usage: tools/sanitize.sh [logdir]   (needs a GPU; `make sanitize`)
set -u
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
LOG="${1:-$ROOT/sanitize_logs}"
mkdir -p "$LOG"
cd "$ROOT"
cat > "$LOG/sg.py" <<'PY'
import os, sys
import numpy as np, torch
sys.path.insert(0, os.getcwd())
from roc_b200 import kernels as K, datasets
re, col = datasets.rmat_graph(10, 6000, seed=3)
n = re.shape[0]
plan = K.SgPlan(0, n - 1, 0, re.cuda(), col.cuda())
for h in (41, 64, 100, 200, 602):
    x = K.padded(n, h, "cuda", fill=torch.rand((n, h), device="cuda"))
    plan.forward(x, epilogue=3)
    mx, arg = plan.minmax_forward(x, 1)                 # max aggregation and its backward
    g = plan.minmax_backward(x, arg)
    torch.cuda.synchronize()
for h, heads in ((41, 1), (64, 1), (64, 8), (256, 8)):
    x = K.padded(n, h, "cuda", fill=torch.rand((n, h), device="cuda"))
    sc = torch.randn((n, 2 * heads), device="cuda")
    out, stats = plan.attn_forward(x, sc, heads)
    plan.attn_backward(x, sc, out, stats, x, heads)
    torch.cuda.synchronize()
xs = torch.rand((n, 257), device="cuda")[:, :256]            # ld = 257: the scalar path
sc = torch.randn((n, 4), device="cuda")
out = torch.zeros((n, 257), device="cuda")[:, :256]
out, stats = plan.attn_forward(xs, sc, 2, out=out)
plan.attn_backward(xs, sc, out, stats, xs, 2, in_grad=torch.zeros((n, 257), device="cuda")[:, :256])
torch.cuda.synchronize()
tr = K.SgTranspose(re.cuda(), col.cuda())
w = torch.rand(col.shape[0], device="cuda")
for h in (41, 64, 200, 602):
    x = K.padded(n, h, "cuda", fill=torch.rand((n, h), device="cuda"))
    y = plan.weighted_forward(x, w)
    tr.backward(y, w)
    dw = plan.edge_dot(y, x)
    plan.edge_dot(y, x, dw=dw, accumulate=True)
    torch.cuda.synchronize()
for h in (41, 64, 200, 602):                                 # the exact backwards over the same transpose
    x = K.padded(n, h, "cuda", fill=torch.rand((n, h), device="cuda"))
    tr.sum_backward(x, epilogue=3, row_end=re.cuda())
    mx, arg = plan.minmax_forward(x, 2)
    tr.minmax_backward(x, arg)
    torch.cuda.synchronize()
for h, heads in ((41, 1), (64, 8)):
    x = K.padded(n, h, "cuda", fill=torch.rand((n, h), device="cuda"))
    sc = torch.randn((n, 2 * heads), device="cuda")
    out, stats = plan.attn_forward(x, sc, heads)
    tr.attn_backward(plan, x, sc, out, stats, x, heads)
    torch.cuda.synchronize()
tr.close()
print("sg ok")
PY
cat > "$LOG/dw.py" <<'PY'
import os, sys
import torch
sys.path.insert(0, os.getcwd())
from roc_b200 import _lib, kernels as K
rows = 20000 - 5
for inn, out, masked in ((602, 64, True), (64, 41, False), (64, 41, True)):
    x = K.padded(rows, inn, "cuda", fill=torch.rand((rows, inn), device="cuda"))
    dy = K.padded(rows, out, "cuda", fill=torch.rand((rows, out), device="cuda"))
    mask = K.dropout_mask(rows, inn, 0, 0.5, 7, 1) if masked else None
    w = torch.zeros((out, inn), device="cuda")
    dw = torch.zeros((out, inn), device="cuda")
    K.linear_bwd_fused(x, w, None, dy, dw, None, mask=mask, rate=0.5 if masked else 0.0, parts=_lib.LINEAR_BWD_ONLY_DW)
    assert _lib.last_gemm_info(_lib.GEMM_DW)["epi"] == 1
    torch.cuda.synchronize()
print("dw ok")
PY
rc=0
for tool in memcheck racecheck; do
  compute-sanitizer --tool $tool --error-exitcode 9 python -c "import __graft_entry__ as g; g.smoke()" > "$LOG/${tool}_smoke.log" 2>&1 || rc=1
  compute-sanitizer --tool $tool --error-exitcode 9 python "$LOG/sg.py" > "$LOG/${tool}_sg.log" 2>&1 || rc=1
  compute-sanitizer --tool $tool --error-exitcode 9 python "$LOG/dw.py" > "$LOG/${tool}_dw.log" 2>&1 || rc=1
  tail -2 "$LOG/${tool}_smoke.log" "$LOG/${tool}_sg.log" "$LOG/${tool}_dw.log"
done
exit $rc
