#!/bin/bash
# compute-sanitizer over the tiny configuration (SURVEY §5): memcheck, then racecheck, on
#   (a) __graft_entry__.smoke()  — one GCN training step through the Model API (SG, wgmma GEMMs, softmax, Adam)
#   (b) the ScatterGather sum with the fused epilogue on a small R-MAT graph at 41, 64, 100, 200 and 602 floats, each
#       followed by one max-aggregation forward and backward.
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
print("sg ok")
PY
rc=0
for tool in memcheck racecheck; do
  compute-sanitizer --tool $tool --error-exitcode 9 python -c "import __graft_entry__ as g; g.smoke()" > "$LOG/${tool}_smoke.log" 2>&1 || rc=1
  compute-sanitizer --tool $tool --error-exitcode 9 python "$LOG/sg.py" > "$LOG/${tool}_sg.log" 2>&1 || rc=1
  tail -2 "$LOG/${tool}_smoke.log" "$LOG/${tool}_sg.log"
done
exit $rc
