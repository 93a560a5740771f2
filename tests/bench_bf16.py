"""bench_bf16.py — the layer-1 Linear launches of bench.py configs 2, 4 and 5 on fp32 and on bf16 input features,
each alone (not a pytest file).

    python tests/bench_bf16.py [--rows 4194304] [--rounds 3] [--iters 10]

Per config, the forward 602 -> outDim (config 2 / 4: dropout mask on the input and the indegree-norm epilogue; config 5:
norm epilogue) and the dW (mask as the forward), CUDA-event timed on HBM-resident operands, fp32 X and bf16 X
alternating within each round.  Bytes are what a launch must move at the padded leading dimensions (X, Y or dY, mask
words, row ends, each once).  Also the device bytes of X in each form, and the upload of X from pinned host memory:
fp32 rows copied as they are against bf16 rows copied as they are, and fp32 rows converted on the device through 64 MB
staging chunks.  Prints the card (name, power limit, max SM clock), then one JSON line per measurement.
"""
import argparse
import importlib.util
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from roc_b200 import _lib  # noqa: E402
from roc_b200 import kernels as K  # noqa: E402

_spec = importlib.util.spec_from_file_location("bench_linear_cfg2", os.path.join(HERE, "bench_linear_cfg2.py"))
_b2 = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_b2)
timeit, card, PEAK_GBS = _b2.timeit, _b2.card, _b2.PEAK_GBS

CONFIGS = {2: (602, 64, True), 4: (602, 128, True), 5: (602, 256, False)}   # inDim, outDim, input dropout


def pad(h, m):
    return (h + m - 1) // m * m


def upload_ms(host, dev_out, iters):
    """ms per upload of a pinned host tensor"""
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_out.copy_(host, non_blocking=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        dev_out.copy_(host, non_blocking=True)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 22)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    dev, n = "cuda", a.rows
    print(json.dumps({"card": card(), "peak_GBps": PEAK_GBS,
                      "peak_source": "H100 SXM data sheet (3.35 TB/s HBM3)"}), flush=True)
    g = torch.Generator(device=dev).manual_seed(3)
    re = torch.cumsum(torch.randint(1, 30, (n,), device=dev, generator=g), 0)
    inn = 602
    xw = K.padded(n, inn, dev)
    xb = K.bf16_padded(n, inn, dev)
    step = 1 << 18
    for r0 in range(0, n, step):
        K.f32_to_bf16(torch.rand((min(step, n - r0), inn), device=dev, generator=g) * 2 - 1, out=xb[r0:r0 + step])
    K.bf16_to_f32(xb, out=xw)
    mask = K.dropout_mask(n, inn, 0, 0.5, 5, 1, dev)
    print(json.dumps({"x_bytes": {"float32": n * xw.stride(0) * 4, "bfloat16": n * xb.stride(0) * 2}}), flush=True)
    for cfg, (i, o, masked) in CONFIGS.items():
        m, rate = (mask, 0.5) if masked else (None, 0.0)
        w = (torch.rand(o, i, device=dev, generator=g) - 0.5) * 0.2
        y = K.padded(n, o, dev)
        dy = K.padded(n, o, dev)
        dy[:, :o] = torch.rand(n, o, device=dev, generator=g) - 0.5
        dw = torch.zeros(o, i, device=dev)
        mw = m.stride(0) * 4 if m is not None else 0
        launches = {
            ("fwd", "float32"): (n * (pad(i, 4) * 4 + o * 4 + mw + 8),
                                 lambda: K.linear_fwd_dropout(xw, w, m, rate, norm_row_end=re, out=y), _lib.GEMM_FWD),
            ("fwd", "bfloat16"): (n * (pad(i, 8) * 2 + o * 4 + mw + 8),
                                  lambda: K.linear_fwd_bf16(xb, w, m, rate, norm_row_end=re, out=y), _lib.GEMM_FWD),
            ("dW", "float32"): (n * (pad(i, 4) * 4 + pad(o, 4) * 4 + mw),
                                lambda: K.linear_bwd_dropout(xw, w, None, dy, dw, m, rate), _lib.GEMM_DW),
            ("dW", "bfloat16"): (n * (pad(i, 8) * 2 + pad(o, 4) * 4 + mw),
                                 lambda: K.linear_dw_bf16(xb, dy, dw, m, rate), _lib.GEMM_DW),
        }
        for rnd in range(a.rounds):
            for (kind, dt), (byt, fn, which) in launches.items():
                ms = timeit(fn, a.iters)
                gbs = byt / ms / 1e6
                print(json.dumps({"config": cfg, "launch": "%s %d->%d" % (kind, i, o), "x": dt, "round": rnd,
                                  "rows": n, "ms": round(ms, 4), "GB": round(byt / 1e9, 3), "GBps": round(gbs, 1),
                                  "bound_ms": round(byt / PEAK_GBS / 1e6, 4), "info": _lib.last_gemm_info(which)}),
                      flush=True)
        del launches, y, dy
        torch.cuda.empty_cache()
    print(json.dumps({"peak_allocated_bytes": torch.cuda.max_memory_allocated()}), flush=True)

    # uploads from pinned host memory
    rows = min(n, 1 << 20)
    h32 = torch.empty((rows, xw.stride(0)), dtype=torch.float32, pin_memory=True)
    hb = torch.empty((rows, xb.stride(0)), dtype=torch.bfloat16, pin_memory=True)
    h32[:, :inn].copy_(xw[:rows].cpu())
    hb[:, :inn].copy_(xb[:rows].cpu())
    d32 = torch.empty_like(h32, device=dev)
    db = torch.empty_like(hb, device=dev)
    chunk_rows = (64 << 20) // (xw.stride(0) * 4)
    stage = torch.empty((chunk_rows, xw.stride(0)), device=dev)

    def convert_upload():
        for r0 in range(0, rows, chunk_rows):
            r1 = min(rows, r0 + chunk_rows)
            stage[:r1 - r0].copy_(h32[r0:r1], non_blocking=True)
            K.f32_to_bf16(stage[:r1 - r0, :inn], out=db[r0:r1, :inn])

    for rnd in range(a.rounds):
        t32 = upload_ms(h32, d32, 5)
        tb = upload_ms(hb, db, 5)
        tc = timeit(convert_upload, 5)
        print(json.dumps({"upload_rows": rows, "round": rnd, "float32_ms": round(t32, 3), "bfloat16_ms": round(tb, 3),
                          "float32_converted_ms": round(tc, 3), "float32_bytes": h32.numel() * 4,
                          "bfloat16_bytes": hb.numel() * 2}), flush=True)


if __name__ == "__main__":
    main()
