#!/bin/bash
# compute-sanitizer over the tiny configuration (SURVEY §5): memcheck, then racecheck, on
#   (a) __graft_entry__.smoke()  — one GCN training step through the Model API (SG, wgmma GEMMs, softmax, Adam)
#   (b) every ScatterGather variant (registers / cp.async / TMA bulk-copy rings / producer-consumer ring) on the
#       ragged test graph, then one max-aggregation forward and backward.
# Usage: tools/sanitize.sh [logdir]   (needs a GPU; `make sanitize`)
set -u
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
LOG="${1:-$ROOT/sanitize_logs}"
mkdir -p "$LOG"
cd "$ROOT"
cat > "$LOG/sg_variants.py" <<'PY'
import os, sys
import numpy as np, torch
sys.path.insert(0, os.getcwd())
from roc_b200 import kernels as K, datasets
re, col = datasets.rmat_graph(10, 6000, seed=3)
n = re.shape[0]
plan = K.SgPlan(0, n - 1, 0, re.cuda(), col.cuda())
for h in (41, 64, 200):
    x = K.padded(n, h, "cuda", fill=torch.rand((n, h), device="cuda"))
    outs = []
    for v in ("a", "c", "t", "b", "r"):
        os.environ["ROC_SG_VARIANT"] = v
        outs.append(plan.forward(x, epilogue=3).clone())
    torch.cuda.synchronize()
    assert all(torch.equal(o.view(torch.int32), outs[0].view(torch.int32)) for o in outs), h
    os.environ.pop("ROC_SG_VARIANT")
    mx, arg = plan.minmax_forward(x, 1)                 # max aggregation and its backward (kernel A + fix-ups)
    g = plan.minmax_backward(x, arg)
    torch.cuda.synchronize()
print("sg variants ok")
PY
rc=0
for tool in memcheck racecheck; do
  compute-sanitizer --tool $tool --error-exitcode 9 python -c "import __graft_entry__ as g; g.smoke()" > "$LOG/${tool}_smoke.log" 2>&1 || rc=1
  compute-sanitizer --tool $tool --error-exitcode 9 python "$LOG/sg_variants.py" > "$LOG/${tool}_sg.log" 2>&1 || rc=1
  tail -2 "$LOG/${tool}_smoke.log" "$LOG/${tool}_sg.log"
done
exit $rc
