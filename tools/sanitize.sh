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
#       and end in a partial block;
#   (d) the elementwise kernels: each of the four softmax cross-entropy kernels (C = 7, 41, 100, 300) with metrics,
#       plain and with the fused norm, on 8 SMs so that every grid loops; dropout on the float4 and scalar paths; and
#       roc_push_rows into local slabs on both paths and both lane counts.
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
cat > "$LOG/ew.py" <<'PY'
import ctypes as C, os, sys
import torch
sys.path.insert(0, os.getcwd())
from roc_b200 import _lib, kernels as K
lib = _lib.lib
prev = lib.roc_set_sm_reserve(torch.cuda.get_device_properties(0).multi_processor_count - 8)
n = 3001
mask = torch.randint(0, 4, (n,), dtype=torch.int32, device="cuda")
row_end = torch.cumsum(torch.randint(0, 9, (n,), device="cuda"), 0)
for c in (7, 41, 100, 300):                                  # LR = 8, 16, 32 and the warp-per-row kernel
    z = K.padded(n, c, "cuda", fill=torch.randn((n, c), device="cuda"))
    lab = torch.randint(0, c, (n,), dtype=torch.int32, device="cuda")
    K.softmax_xent_bwd(z, lab, mask, compact=True)
    K.softmax_xent_bwd_norm(z, lab, mask, row_end, 0, compact=True, with_perf=True)
    torch.cuda.synchronize()
for h in (41, 64):
    x = torch.randn((n, h), device="cuda")
    K.dropout_fwd(K.padded(n, h, "cuda", fill=x), 5, 0.5, 7, 1)     # float4 path
    K.dropout_fwd(x, 5, 0.5, 7, 1)                                 # scalar path when h % 4
    torch.cuda.synchronize()
lib.roc_set_sm_reserve(prev)
src = torch.randn((2000, 264), device="cuda")
for h in (41, 200):                                          # LR = 16 / 32 on the float4 path
    rows = torch.randint(0, 2000, (n,), dtype=torch.int32, device="cuda")
    peer = torch.randint(0, 2, (n,), dtype=torch.uint8, device="cuda")
    dst = torch.randperm(n, device="cuda").to(torch.int32)
    slabs = [torch.zeros((n, 264), device="cuda") for _ in range(2)]
    for off in (0, 1):                                       # 1: a base 4 bytes off alignment takes the scalar path
        bases = (C.c_void_p * 2)(*[s.data_ptr() + 4 * off for s in slabs])
        assert lib.roc_push_rows(n, h, rows.data_ptr(), peer.data_ptr(), dst.data_ptr(), src.data_ptr(), 264,
                                 C.cast(bases, C.c_void_p), 2, 264, 1, None) == 0
    torch.cuda.synchronize()
print("ew ok")
PY
rc=0
for tool in memcheck racecheck; do
  compute-sanitizer --tool $tool --error-exitcode 9 python -c "import __graft_entry__ as g; g.smoke()" > "$LOG/${tool}_smoke.log" 2>&1 || rc=1
  compute-sanitizer --tool $tool --error-exitcode 9 python "$LOG/sg.py" > "$LOG/${tool}_sg.log" 2>&1 || rc=1
  compute-sanitizer --tool $tool --error-exitcode 9 python "$LOG/dw.py" > "$LOG/${tool}_dw.log" 2>&1 || rc=1
  compute-sanitizer --tool $tool --error-exitcode 9 python "$LOG/ew.py" > "$LOG/${tool}_ew.log" 2>&1 || rc=1
  tail -2 "$LOG/${tool}_smoke.log" "$LOG/${tool}_sg.log" "$LOG/${tool}_dw.log" "$LOG/${tool}_ew.log"
done
exit $rc
