"""GPU suite: the training step bench.py times, at full size, against an fp64 reference.

For each of bench.py's configs 1-5 the workload is built as bench.py builds it (make_graph, build_model, the node data
of bench.run_ours uploaded through set_tensor_from_host_ptr / set_labels) with the Model wrapped in a Recorder.  Two
steps run: train_mode / zero_gradients / forward / backward / update, then train_epoch().  After each, the host keeps
the logits, every dW, the ReLU outputs, the metrics, the weights and the Adam moments.  Then the product is closed and
tests/scale_witness.py runs each step on the whole card, from the product's own weights before that step (W0, then W1),
so errors do not compound.  Bars (conftest.rel_close, DESIGN.md section 4):

    logits, ReLU outputs      1e-4 relative + 1e-5 * max|want|
    dW                        2e-4 relative + 1e-5 * max|want| + the dW GEMM's own bound (see below)
    layer 1's dL/dY           1e-4 relative + 1e-5 * max|want|
    trainLoss                 2e-4 relative
    trainAll / valAll / testAll   exact
    the three correct-counts  equal, but for rows whose fp64 top-two probabilities lie within 1e-6
    Adam                      W1 from W0 and the product's dW1 by an fp64 restatement of roc_adam_update at t = 1,
                              and W2 from W1, dW2 and the product's moments at t = 2: W, m and v at
                              1e-5 relative + 1e-6 * max|want|

The dW bar.  DESIGN.md section 4's 2e-4 + 1e-5 * max covers an error carried in from 1e-4-accurate operands, not
the dW GEMM's own rounding, which grows with the rows it sums: tests/tf32_bound.py models it (the 3xTF32 split, and
accumulation that truncates, so that a split-K range of L rows loses about L / 8 * 2^-23 of its partial sums).  At
1000 rows that is nothing; at 4 M rows it is 4.5e-4 * max|dW| on layer 1 of config 2.  So each dW is held to the sum
of the parity bar and tf32_bound.RefAccumulator's bound on the witness's own operands (dY and the dropped X, fp64),
over the dW kernel's split-K ranges.  The ranges are restated from the kernel's plan (dw_split_rows) and pinned to the
v_per_split that roc_last_gemm_info reports for the step's last dW launch.  The dW operand that comes from the
backward pass, layer 1's dL/dY, is compared with the product's too, so that the excess is not an upstream error.

Two smaller checks: set_tensor / set_tensor_from_host_ptr / get_tensor round trips across the 64 M-float staging
chunks (2 * chunkRows + 13 rows, after a narrow tensor that leaves the staging buffer small), exact; and config 2 with
bf16 features against its fp32 twin on the bf16-rounded features, byte for byte over two steps.

Each test prints the worst error-to-bar ratio per quantity, the device memory of each side and the wall time.
Measured on one H100 80GB HBM3 (700 W): see MEASURED below.  Configs 2-5 carry full_size in their names: deselect them
with -k "not full_size"; each skips when the GPU has less free memory than it needs."""
import math
import time

import numpy as np
import pytest
import torch

from bench_inputs import bench_module, node_inputs
from opgraph import Recorder
from roc_b200 import _lib, bf16, datasets
from roc_b200.model import Host, Model, build_gcn
from scale_witness import scale_witness

pytestmark = pytest.mark.gpu
DEV = "cuda"
B = bench_module()
GB = 1 << 30
# free device memory each config needs: the larger of the product's device memory and the witness's peak, measured
# (MEASURED), plus about 1 GB.  Config 3's product holds 77.2 GB: two dozen [2.45 M x 256] fp32 tensors and their
# gradients, so it needs nearly the whole card.
NEED_GB = {1: 1, 2: 43, 3: 78, 4: 45, 5: 14}
MEASURED = """
Worst error / bar over both steps, on one H100 80GB HBM3 (700 W), 78.7 GB free at the start.  dW: the worst parameter
under its bar (parity bar + GEMM bound), and in brackets the same error against the parity bar alone.
config  logits  relu   dL/dY  dW             trainLoss  Adam W / m / v          witness peak  product  time
1       0.023   0.016  0.013  0.020 (0.024)  2.4e-4     0.005 / 0.009 / 0.011   0.1 GB        0.0 GB     2 s
2       0.16    0.21   0.33   0.18  (5.9)    2.5e-3     0.016 / 0.007 / 0.009   40.9 GB       17.4 GB    68 s
3       0.11    0.086  0.13   0.18  (2.3)    3.5e-3     0.015 / 0.011 / 0.015   46.6 GB       77.2 GB   176 s
4       0.19    0.22   0.39   0.21  (8.5)    3.6e-3     0.016 / 0.007 / 0.010   42.9 GB       21.6 GB   107 s
5       0.22    0.19   0.36   0.12  (2.2)    2.1e-3     0.022 / 0.032 / 0.017   12.3 GB       11.2 GB    29 s
dW split-K ranges (rows x ranges): 602 -> 64 / 128 161344 x 26; 64 / 128 -> 41 31776 x 132; config 3 18560 x 132
(100 wide) and 37120 x 66 (256 wide); config 5 8992 x 26 and 3552 x 66.
Correct-counts: product and fp64 differ by at most 1 row, always within the rows near a tie (up to 2277 of 4.19 M).
ReLU signs taken from the product at a tie: up to 357 elements per layer.  Config 2's bf16 twin: 77 s.  The data
paths: a few seconds.  The whole file: 8.3 minutes.
"""


def need(gb, what):
    free, _ = torch.cuda.mem_get_info()
    if free < gb * GB:
        pytest.skip("%s needs %d GB of free device memory, %.1f GB are free" % (what, gb, free / GB))


class Report:
    """worst error / bar per quantity; failures are collected so that every ratio is printed before the assert"""

    def __init__(self, title):
        self.title, self.worst, self.bad, self.notes = title, {}, [], []

    def ratio(self, what, got, want, rtol, atol_scale, extra=0.0):
        """extra: an absolute bound added element by element"""
        got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
        assert got.shape == want.shape, (what, got.shape, want.shape)
        bound = rtol * np.abs(want) + atol_scale * (np.abs(want).max() if want.size else 0.0) + extra + 1e-30
        err = np.abs(got - want)
        r = float((err / bound).max()) if want.size else 0.0
        self.worst[what] = max(self.worst.get(what, 0.0), r)
        if not r <= 1.0:
            self.bad.append("%s: error %.3g x the bar" % (what, r))

    def exact(self, what, ok, detail):
        if not ok:
            self.bad.append("%s: %s" % (what, detail))

    def note(self, s):
        self.notes.append(s)

    def finish(self):
        print("\n[%s]" % self.title)
        for k in sorted(self.worst):
            print("  %-28s worst error / bar %.3g" % (k, self.worst[k]))
        for s in self.notes:
            print("  " + s)
        assert not self.bad, "%s: %s" % (self.title, "; ".join(self.bad))


def snapshot(m, hnd, ir):
    """what the step left on the device: logits, dW, W, Adam's m and v, the ReLU outputs, the metrics"""
    P = m.num_parameters()
    return dict(logits=m.get_tensor(hnd["logits"]),
                dW=[m.get_parameter(p, "grad") for p in range(P)], W=[m.get_parameter(p) for p in range(P)],
                M=[m.get_parameter(p, "m") for p in range(P)], V=[m.get_parameter(p, "v") for p in range(P)],
                relu={n["layer"]: m.get_tensor(n["out"]) for n in ir.nodes if n["kind"] == "relu"}
                if ir is not None else {},
                dy0=m.get_tensor(linear_out(ir, 0), grad=True) if ir is not None else None,
                dw_info=_lib.last_gemm_info(_lib.GEMM_DW), metrics=m.metrics())


def linear_out(ir, p):
    return next(n["out"] for n in ir.nodes if n["kind"] == "linear" and n["attrs"]["param"] == p)


def dw_split_rows(rows, in_dim, out_dim):
    """(splits, rows per split-K range) of the tensor-core dW GEMM, restated from tc_dw_plan and tc_linear_dw
    (linear_tc_dw.cu): one range per SM over the CTAs per range (a CTA takes 128 X columns), at most one per 64 rows,
    rounded up to the kernel's 32-row stage"""
    splits = max(1, torch.cuda.get_device_properties(0).multi_processor_count // -(-in_dim // 128))
    splits = min(splits, (rows + 63) // 64)
    return splits, -(-(-(-rows // splits)) // 32) * 32


def run_product(cfg, graph, feats, labels, mask, features="float32", weights=None):
    """bench.py's model of config cfg for two training steps.  features="bfloat16": build_gcn with bf16 input
    features (no Recorder: it records fp32 leaves only).  Returns (ir, W0, [step 1, step 2], device bytes held)."""
    re_h, col_h = graph
    free0 = torch.cuda.mem_get_info()[0]
    host = Host(0, 0, 1)
    host.graph_from_arrays(re_h, col_h)
    info = host.graph_info()
    assert (info["rowLeft"], info["rowRight"]) == (0, re_h.shape[0] - 1)
    m = Model(host, seed=1)
    if features == "float32":
        ir = Recorder(m)
        hnd = B.build_model(ir, cfg)
    else:
        c = B.CONFIGS[cfg]
        assert c["kind"] == "gcn"
        ir = None
        hnd = build_gcn(m, c["layers"], B.DROPOUT, lr=B.LR, weight_decay=B.WD, features=features)
    for p, w in enumerate(weights or []):
        m.set_parameter(p, w)
    m.set_tensor_from_host_ptr(hnd["input"], feats.data_ptr())
    m.set_labels(hnd["label"], labels.numpy())
    m.set_tensor_from_host_ptr(hnd["mask"], mask.data_ptr())
    w0 = [m.get_parameter(p) for p in range(m.num_parameters())]
    m.train_mode(); m.zero_gradients(); m.forward(); m.backward(); m.update()
    s1 = snapshot(m, hnd, ir)
    m.train_epoch()
    s2 = snapshot(m, hnd, ir)
    host.synchronize()
    held = free0 - torch.cuda.mem_get_info()[0]
    host.close()
    torch.cuda.empty_cache()
    return ir, w0, [s1, s2], held


def adam_ref(w, g, m, v, t):
    """roc_adam_update in fp64 (oracle.adam_update's semantics: coupled L2, eps outside the sqrt) with the host's
    bias-corrected alpha_t (AdamOptimizer::next: beta1 = 0.9f, beta2 = 0.999f, accumulated in double) at step t"""
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
    alpha_t = float(np.float32(B.LR * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)))
    wd, eps = float(np.float32(B.WD)), float(np.float32(1e-8))
    w, g, m, v = (np.asarray(a, dtype=np.float64) for a in (w, g, m, v))
    gt = g + wd * w
    m = b1 * m + (1 - b1) * gt
    v = b2 * v + (1 - b2) * gt * gt
    return w - alpha_t * m / (np.sqrt(v) + eps), m, v


def check_config(cfg):
    need(NEED_GB[cfg], "config %d" % cfg)
    rep = Report("config %d: %s" % (cfg, B.CONFIGS[cfg]["desc"]))
    compare_config(cfg, rep)
    rep.finish()          # here, so that a failure's traceback holds none of the full-size arrays


def compare_config(cfg, rep):
    c = B.CONFIGS[cfg]
    t0 = time.time()
    graph = B.make_graph(datasets, cfg, 1, DEV)[:2]
    n, e = graph[0].shape[0], graph[1].shape[0]
    feats, labels, mask = node_inputs(n, c["layers"], DEV)
    ir, w0, steps, held = run_product(cfg, graph, feats, labels, mask)
    t1 = time.time()
    rep.note("graph N=%d E=%d; product: %.1f GB held on the device, %.0f s with the graph build and the uploads"
             % (n, e, held / GB, t1 - t0))
    lab, mk = labels.numpy(), mask.numpy()
    w_in = w0
    shapes = [w.shape for w in w0]                      # [out][in]
    split = {p: dw_split_rows(n, i, o)[1] for p, (o, i) in enumerate(shapes)}
    for s in steps:     # the step's last dW launch is parameter 0's (backward runs in reverse creation order)
        info = s["dw_info"]
        assert info["path"] == 1 and (info["splits"], info["v_per_split"]) == dw_split_rows(n, shapes[0][1], shapes[0][0]), info
    rep.note("dW split-K: " + ", ".join("dW[%d] %d rows x %d" % (p, split[p], dw_split_rows(n, i, o)[0])
                                        for p, (o, i) in enumerate(shapes)))
    for step, s in enumerate(steps, 1):
        torch.cuda.reset_peak_memory_stats()
        t2 = time.time()
        wit = scale_witness(ir, graph, feats, lab, mk, w_in, step=step, device=DEV, dw_split=split, keep_dy=(0,),
                            relu_masks={layer: r > 0 for layer, r in s["relu"].items()})
        rep.note("step %d witness: peak %.1f GB allocated, %.0f s" %
                 (step, torch.cuda.max_memory_allocated() / GB, time.time() - t2))
        torch.cuda.empty_cache()
        # the ReLU outputs first, in layer order: the first one out of bounds locates a fault
        for layer in sorted(s["relu"]):
            rep.ratio("relu (layer %d)" % layer, s["relu"][layer], np.maximum(wit["pre"][layer], 0.0), 1e-4, 1e-5)
            flips = int(((wit["pre"][layer] > 0) != (s["relu"][layer] > 0)).sum())
            if flips:
                rep.note("step %d relu layer %d: %d signs taken from the product at a tie" % (step, layer, flips))
        rep.ratio("logits", s["logits"], wit["logits"], 1e-4, 1e-5)
        rep.ratio("layer 1 dL/dY", s["dy0"], wit["dy"][0], 1e-4, 1e-5)
        for p, (a, b) in enumerate(zip(s["dW"], wit["dW"])):
            rep.ratio("dW[%d]" % p, a, b, 2e-4, 1e-5, extra=wit["dW_bound"][p])
            # reported, not asserted: the same error against the parity bar alone
            r = float((np.abs(np.asarray(a, np.float64) - b) / (2e-4 * np.abs(b) + 1e-5 * np.abs(b).max() + 1e-30)).max())
            key = "dW[%d], parity bar only" % p
            rep.worst[key] = max(rep.worst.get(key, 0.0), r)
        pm, wm = s["metrics"], wit["metrics"]
        rep.ratio("trainLoss", pm["trainLoss"], wm["trainLoss"], 2e-4, 0.0)
        for k in ("trainAll", "valAll", "testAll"):
            rep.exact("step %d %s" % (step, k), pm[k] == wm[k], "%d, fp64 %d" % (pm[k], wm[k]))
        for k in ("trainCorrect", "valCorrect", "testCorrect"):
            ties = wm["near_ties"][k]
            rep.exact("step %d %s" % (step, k), abs(pm[k] - wm[k]) <= ties,
                      "%d, fp64 %d, %d rows near a tie" % (pm[k], wm[k], ties))
            rep.note("step %d %s: product %d, fp64 %d, %d rows within 1e-6 of a tie" % (step, k, pm[k], wm[k], ties))
        # Adam at t = step, from the product's own inputs to the update
        prev_m = [np.zeros_like(w) for w in w_in] if step == 1 else steps[0]["M"]
        prev_v = [np.zeros_like(w) for w in w_in] if step == 1 else steps[0]["V"]
        for p in range(len(w_in)):
            wr, mr, vr = adam_ref(w_in[p], s["dW"][p], prev_m[p], prev_v[p], step)
            rep.ratio("Adam W", s["W"][p], wr, 1e-5, 1e-6)
            rep.ratio("Adam m", s["M"][p], mr, 1e-5, 1e-6)
            rep.ratio("Adam v", s["V"][p], vr, 1e-5, 1e-6)
        w_in = s["W"]
        del wit
    rep.note("total %.0f s" % (time.time() - t0))


def test_config1_bench_step():
    check_config(1)


def test_config2_full_size_bench_step():
    check_config(2)


def test_config3_full_size_bench_step():
    check_config(3)


def test_config4_full_size_bench_step():
    check_config(4)


def test_config5_full_size_bench_step():
    check_config(5)


# ------------------------------------------------------------------------------------------------- data paths ---
def chunk_rows(h):
    """rows per staging chunk of Model::set_tensor / get_tensor: 64 M floats"""
    return max(1, (64 << 20) // h)


def same_bytes(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("kind,h", [("f32", 602), ("f32", 64), ("int", 64), ("bf16", 602)],
                         ids=["f32_padded_602", "f32_dense_64", "int_64", "bf16_602"])
def test_data_paths_across_staging_chunks(kind, h):
    """A node tensor of 2 * chunkRows + 13 rows (two whole staging chunks and a partial one) round-trips exactly
    through set_tensor and set_tensor_from_host_ptr (pinned rows, as bench.py uploads) and get_tensor.  A narrow
    padded tensor is written first, so that the staging buffer is small and must grow for the wide one; it must
    still read back intact at the end.  fp32 at H = 602 is re-pitched through staging, at H = 64 it is one copy; a
    bf16 tensor is rounded on the device from fp32 rows (and widened back through staging), or copied as raw bits."""
    n = 2 * chunk_rows(h) + 13
    need(4 if kind != "f32" or h != 64 else 2, "the data paths")
    host = Host(0, 0, 1)
    host.graph_from_arrays(np.arange(1, n + 1, dtype=np.uint64), np.arange(n, dtype=np.uint32))
    m = Model(host, seed=1)
    rng = np.random.default_rng(h)
    small = m.create_node_tensor(3)
    assert m.tensor_shape(small) == (n, 3, 4)
    s = rng.standard_normal((n, 3), dtype=np.float32)
    m.set_tensor(small, s)
    assert same_bytes(m.get_tensor(small), s)
    if kind == "int":
        t = m.create_node_tensor(h, is_int=True)
        a = rng.integers(-2 ** 31, 2 ** 31 - 1, size=(n, h), dtype=np.int32)
        b = torch.from_numpy(rng.integers(-2 ** 31, 2 ** 31 - 1, size=(n, h), dtype=np.int32)).pin_memory()
        m.set_tensor(t, a)
        assert same_bytes(m.get_tensor(t, dtype=np.int32), a), "set_tensor"
        m.set_tensor_from_host_ptr(t, b.data_ptr())
        assert same_bytes(m.get_tensor(t, dtype=np.int32), b.numpy()), "set_tensor_from_host_ptr"
    elif kind == "f32":
        t = m.create_node_tensor(h)
        assert m.tensor_shape(t)[2] == (h if h % 4 == 0 else (h + 3) // 4 * 4)
        a = rng.standard_normal((n, h), dtype=np.float32)
        b = torch.from_numpy(rng.standard_normal((n, h), dtype=np.float32)).pin_memory()
        m.set_tensor(t, a)
        assert same_bytes(m.get_tensor(t), a), "set_tensor"
        m.set_tensor_from_host_ptr(t, b.data_ptr())
        assert same_bytes(m.get_tensor(t), b.numpy()), "set_tensor_from_host_ptr"
    else:
        t = m.create_node_tensor(h, dtype="bfloat16")
        a = rng.standard_normal((n, h), dtype=np.float32) * 100
        b = torch.from_numpy(rng.standard_normal((n, h), dtype=np.float32)).pin_memory()
        m.set_tensor(t, a)                                      # fp32 rows, rounded on the device
        assert np.array_equal(m.get_tensor(t, raw=True), bf16.to_bits(a)), "set_tensor from fp32"
        assert same_bytes(m.get_tensor(t), bf16.round_f32(a)), "get_tensor widened"
        m.set_tensor_from_host_ptr(t, b.data_ptr())
        assert np.array_equal(m.get_tensor(t, raw=True), bf16.to_bits(b.numpy())), "set_tensor_from_host_ptr"
        raw = torch.from_numpy(-a).to(torch.bfloat16)          # raw bits
        m.set_tensor(t, raw)
        assert np.array_equal(m.get_tensor(t, raw=True), raw.view(torch.int16).numpy().view(np.uint16)), "raw bits"
        assert same_bytes(m.get_tensor(t), raw.float().numpy()), "raw bits widened"
    assert same_bytes(m.get_tensor(small), s), "the narrow tensor changed"
    host.close()


def test_config2_bf16_twin_full_size():
    """Config 2 with bf16 features (build_gcn(..., features="bfloat16") uploading the raw fp32 features, rounded on
    the device) against the fp32 build on the bf16-rounded features, from the same W0: logits, every dW, the weights
    after each update and the six counts byte-identical over two steps (README.md: the bf16 kernels widen X exactly).
    trainLoss is left out: its fp32 atomics are not ordered."""
    need(NEED_GB[2], "config 2 with bf16 features")
    c = B.CONFIGS[2]
    t0 = time.time()
    graph = B.make_graph(datasets, 2, 1, DEV)[:2]
    n = graph[0].shape[0]
    feats, labels, mask = node_inputs(n, c["layers"], DEV)
    rounded = torch.empty(feats.shape, dtype=torch.float32, pin_memory=True)
    for r0 in range(0, n, 1 << 18):
        rounded[r0:r0 + (1 << 18)] = torch.from_numpy(bf16.round_f32(feats[r0:r0 + (1 << 18)].numpy()))
    _, w0, got, held_b = run_product(2, graph, feats, labels, mask, features="bfloat16")
    del feats
    _, _, want, held_f = run_product(2, graph, rounded, labels, mask, weights=w0)
    for step, (g, w) in enumerate(zip(got, want), 1):
        assert same_bytes(g["logits"], w["logits"]), "step %d: logits differ" % step
        for p in range(len(w0)):
            assert same_bytes(g["dW"][p], w["dW"][p]), "step %d: dW[%d] differs" % (step, p)
            assert same_bytes(g["W"][p], w["W"][p]), "step %d: W[%d] after Adam differs" % (step, p)
        counts = [k for k in g["metrics"] if k != "trainLoss"]
        assert [g["metrics"][k] for k in counts] == [w["metrics"][k] for k in counts], (step, g["metrics"], w["metrics"])
    print("\n[config 2 bf16 twin] N=%d: device %.1f GB (bf16) / %.1f GB (fp32), %.0f s" %
          (n, held_b / GB, held_f / GB, time.time() - t0))
