"""An fp64 interpreter of the op-graph IR that tests/opgraph.py's Recorder records, built to run bench.py's models at
full size on one GPU.  It runs the same on the CPU, where tests/test_scale_witness_cpu.py pins it to opgraph.witness.

It covers the ops the benchmarked models use (SUPPORTED; scatter_gather(t, AGGR_AVG) records as the sum and two
norms) and refuses any other by name.  Torch autograd derives the gradients, as in opgraph.witness.  The one
hand-written piece is the aggregation (Aggregate): forward A @ x, backward A^T @ g, both as index_add over chunks of
the edge list.  The backward does not assume that A is symmetric.  Nothing is shared with the product's kernels.

Memory, so that the witness fits on the card once the product is closed:
  * the aggregation runs over `edge_chunk` edges at a time (2 M edges at H = 256 gather 4 GB in fp64) and saves
    nothing for its backward but the edge lists;
  * dropout is torch.where(bool keep, x * scale, 0) with the keep mask built `mask_rows` rows at a time by
    oracle.dropout_mask, so autograd saves a bool mask.  A dropout whose input needs no gradient (the features) is
    computed outside autograd, row chunk by row chunk, straight from the host tensor;
  * ReLU is opgraph._relu_with_mask, which saves a bool mask;
  * each tensor is dropped once its last reader has run, and the ReLU pre-activations are kept on the host."""
import numpy as np
import torch

import tf32_bound as tb
from oracle import oracle
from opgraph import _relu_with_mask
from roc_b200 import _lib

SUPPORTED = ("dropout", "linear", "indegree_norm", "scatter_gather", "relu", "add", "softmax_cross_entropy")
TIE = 1e-6      # rows whose two largest fp64 probabilities lie this close: the argmax may go either way in fp32


def check_ops(ir):
    for node in ir.nodes:
        if node["kind"] not in SUPPORTED:
            raise ValueError("scale_witness: layer %d: op %s is not supported" % (node["layer"], node["kind"]))


def _chunks(total, size):
    return [(a, min(total, a + size)) for a in range(0, total, size)]


def _spmm(x, rows, cols, chunk, log):
    """y[rows[e]] += x[cols[e]] over every edge e, `chunk` edges at a time"""
    y = torch.zeros_like(x)
    parts = _chunks(rows.shape[0], chunk)
    for a, b in parts:
        y.index_add_(0, rows[a:b], x[cols[a:b]])
    log.append(("aggregate", len(parts), parts[-1][1] - parts[-1][0] if parts else 0, chunk))
    return y


class Aggregate(torch.autograd.Function):
    """y = A x for A[dst][src] = the edge count: y[v] = sum over v's in-edges (u -> v) of x[u].  dL/dx = A^T g:
    dx[u] = sum over u's out-edges (u -> v) of g[v].  The edges ride on ctx; nothing of x is saved."""

    @staticmethod
    def forward(ctx, x, dst, src, chunk, log):
        ctx.edges = (dst, src, chunk, log)
        return _spmm(x, dst, src, chunk, log)

    @staticmethod
    def backward(ctx, g):
        dst, src, chunk, log = ctx.edges
        return _spmm(g.contiguous(), src, dst, chunk, log), None, None, None, None


def metrics(logits, labels, mask, tie=TIE):
    """The loss metrics of roc_oracle_softmax_xent_bwd (oracle/roc_oracle.c) from fp64 logits: P = softmax per row;
    trainLoss = the sum over train rows (mask 0) of 1 - P[true] (not the cross-entropy); the predicted class is the
    first maximum of P (a strict >); the six counts per mask 0 / 1 / 2 (train / val / test).  near_ties: per mask
    value, the rows whose two largest P lie within `tie`.  logits: [N][C] tensor; labels, mask: [N] tensors."""
    with torch.no_grad():
        p = torch.softmax(logits, dim=1)
        top = p.max(dim=1, keepdim=True).values
        idx = torch.arange(p.shape[1], device=p.device)
        pred = torch.where(p == top, idx, p.shape[1]).min(dim=1).values      # the first maximum
        second = torch.where(idx == pred[:, None], -1.0, p).max(dim=1).values if p.shape[1] > 1 else top[:, 0] - 1
        near = (top[:, 0] - second) <= tie
        lab = labels.to(torch.int64)
        hit = pred == lab
        out = {"trainLoss": float((1.0 - p.gather(1, lab[:, None])[:, 0])[mask == 0].sum())}
        names = {0: ("trainAll", "trainCorrect"), 1: ("valAll", "valCorrect"), 2: ("testAll", "testCorrect")}
        ties = {}
        for k, (all_, correct) in names.items():
            sel = mask == k
            out[all_] = int(sel.sum())
            out[correct] = int((hit & sel).sum())
            ties[correct] = int((near & sel).sum())
        out["near_ties"] = ties
    return out


def scale_witness(ir, graph, feats, labels, mask, weights, step=1, relu_masks=None, device="cpu",
                  edge_chunk=1 << 21, mask_rows=1 << 18, dw_split=None, keep_dy=()):
    """The recorded graph (a Recorder) in torch fp64 with autograd on `device`, for one training step.

    graph: (row_end, col), one partition covering the graph.  feats: {leaf id: [N][H] host array or tensor} (one
    array: the first leaf), read `mask_rows` rows at a time.  labels: [N] class indices.  mask: [N] MASK_*.
    weights: W_mem[o][i] per parameter.  step: the product's train-step counter during this step's forward (the first
    step is 1).  relu_masks: {layer: the product's relu output > 0}, taken where fp32 and fp64 tie at 0.
    dw_split: {parameter: rows per split-K range of the product's dW GEMM}: for each, the error bound of that GEMM on
    these operands (tf32_bound.RefAccumulator: the 3xTF32 split and the truncating accumulation, range by range).
    keep_dy: parameters whose dL/dY (the gradient of the Linear's output, the dW GEMM's other operand) is returned.

    Returns dict(logits [N][C], dW (zeros for a Linear off the loss's path), pre {layer: the ReLU pre-activation},
    metrics (see metrics()), chunks [(what, chunks, rows or edges in the last chunk, chunk size)], dW_bound
    {parameter: [out][in]}, dy {parameter: [N][out]}), fp64 numpy on the host."""
    check_ops(ir)
    dev = torch.device(device)
    row_end = np.asarray(graph[0]).astype(np.int64)
    n = row_end.shape[0]
    deg = np.diff(np.concatenate([[0], row_end]))
    dst = torch.from_numpy(np.repeat(np.arange(n, dtype=np.int64), deg)).to(dev)
    src = torch.from_numpy(np.asarray(graph[1]).astype(np.int64)).to(dev)
    dinv = torch.from_numpy(1.0 / np.sqrt(deg.astype(np.float64))).to(dev).unsqueeze(1)
    relu_masks = relu_masks or {}
    if not isinstance(feats, dict):
        feats = {ir.leaves[0]: feats}
    val = {t: torch.as_tensor(a) for t, a in feats.items()}
    ws = [torch.tensor(np.asarray(w), dtype=torch.float64, device=dev).requires_grad_(True) for w in weights]
    last = {}
    for i, node in enumerate(ir.nodes):
        for t in node["ins"]:
            last[t] = i
    log, pre, logits, loss = [], {}, None, None
    dw_split, dw_bound, dy = dw_split or {}, {}, {}

    def rows(x):
        """a host or fp32 tensor as a device fp64 one, `mask_rows` rows at a time"""
        if x.device == dev and x.dtype == torch.float64:
            return x
        y = torch.empty(x.shape, dtype=torch.float64, device=dev)
        for a, b in _chunks(x.shape[0], mask_rows):
            y[a:b] = x[a:b].to(dev).double()
        return y

    def keep_chunks(h, a):
        parts = _chunks(n, mask_rows)
        log.append(("dropout mask", len(parts), parts[-1][1] - parts[-1][0], mask_rows))
        for r0, r1 in parts:
            k = oracle.dropout_mask(r0, r1 - r0, h, a["rate"], a["key"], step)
            yield r0, r1, torch.from_numpy(k).to(dev).bool()

    def relu(x, layer, what):
        pre[layer] = x.detach().cpu().numpy()
        pm = relu_masks.get(layer)
        return _relu_with_mask(x, pm if pm is not None else x.detach() > 0, what)

    for i, node in enumerate(ir.nodes):
        k, a, ins, what = node["kind"], node["attrs"], node["ins"], "layer %d (%s)" % (node["layer"], node["kind"])
        x = val[ins[0]] if ins[0] in val else None
        if k == "linear":
            xin, p = rows(x), a["param"]
            y = xin @ ws[p].T
            if y.requires_grad and (p in dw_split or p in keep_dy):
                y.register_hook(lambda g, xin=xin, p=p: _dw_hook(g, xin, p, dw_split, dw_bound, keep_dy, dy))
            if a["activation"] == _lib.AC_MODE_RELU:
                y = relu(y, node["layer"], what)
        elif k == "indegree_norm":
            y = rows(x) * dinv
        elif k == "scatter_gather":
            y = Aggregate.apply(rows(x), dst, src, edge_chunk, log)
        elif k == "relu":
            y = relu(rows(x), node["layer"], what)
        elif k == "add":
            y = rows(x) + rows(val[ins[1]])
        elif k == "dropout":
            scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(a["rate"])))
            if a["rate"] <= 0:
                y = rows(x)
            elif x.requires_grad:
                keep = torch.empty(x.shape, dtype=torch.bool, device=dev)
                for r0, r1, kc in keep_chunks(x.shape[1], a):
                    keep[r0:r1] = kc
                y = torch.where(keep, x * scale, 0.0)
            else:                        # outside autograd: nothing to save
                y = torch.empty(x.shape, dtype=torch.float64, device=dev)
                for r0, r1, kc in keep_chunks(x.shape[1], a):
                    y[r0:r1] = torch.where(kc, x[r0:r1].to(dev).double() * scale, 0.0)
        elif k == "softmax_cross_entropy":
            logits = rows(x)
            lab = torch.as_tensor(np.asarray(labels).astype(np.int64)).to(dev)
            mk = torch.as_tensor(np.asarray(mask).astype(np.int64)).to(dev)
            train = mk == 0
            # the gradient is that of the summed cross-entropy over the train rows (witness_gat.train_loss)
            loss = torch.nn.functional.cross_entropy(logits[train], lab[train], reduction="sum")
            perf = metrics(logits.detach(), lab, mk)
            y = None
        if node["out"] is not None:
            val[node["out"]] = y
        for t in ins:
            if last[t] == i:
                val.pop(t, None)
    del val
    if loss.requires_grad:               # else no parameter reaches the loss
        loss.backward()
    return dict(logits=logits.detach().cpu().numpy(),
                dW=[w.grad.cpu().numpy() if w.grad is not None else np.zeros(tuple(w.shape)) for w in ws],
                pre=pre, metrics=perf, chunks=log, dW_bound=dw_bound, dy=dy)


def _dw_hook(g, x, p, dw_split, dw_bound, keep_dy, dy, chunk=1 << 17):
    """dL/dY of parameter p's Linear arrives: keep it, and bound the error of dW = dY^T X as the product's dW GEMM
    computes it, over its split-K ranges (chunk: rows per step, a multiple of 8)"""
    if p in keep_dy:
        dy[p] = g.detach().cpu().numpy()
    if p in dw_split:
        acc = tb.RefAccumulator(split=dw_split[p])
        with torch.no_grad():
            for a, b in _chunks(g.shape[0], chunk):
                acc.add(g[a:b].T, x[a:b].T)
            dw_bound[p] = acc.result()[1].cpu().numpy()
