"""Kernel-level entry points (include/roc_b200.h) on torch CUDA tensors.

torch is used here only as the owner of device memory and streams: every
function passes raw device pointers + the current CUDA stream to the C ABI.
2-D tensors may be row-padded views (stride(0) = ld >= shape[1], stride(1) = 1).
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from ._lib import check, lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _ld(t):
    assert t.dim() == 2 and t.stride(1) == 1, "need a row-major 2-D tensor"
    return t.stride(0)


def padded(rows, h, device="cuda", dtype=torch.float32, fill=None):
    """[rows][h] view of a [rows][round_up(h,4)] allocation (the host's node-tensor layout)."""
    ld = (h + 3) // 4 * 4
    buf = torch.zeros((rows, ld), device=device, dtype=dtype)
    v = buf[:, :h]
    if fill is not None:
        v.copy_(fill)
    return v


def _v2_a(a):
    """GATv2's attention vectors [heads][F] in the kernels' layout: a[k][f] at f * heads + k (a Model parameter's)."""
    assert a.dim() == 2 and a.dtype == torch.float32
    return a.t().contiguous()


def _smx_t(t, device):
    """The softmax aggregation's temperature as one fp32 float in device memory: a float, or a 1-element fp32 tensor on
    the device, used as is (a learned t is read where Adam updates it)."""
    if isinstance(t, torch.Tensor):
        assert t.numel() == 1 and t.dtype == torch.float32 and t.is_cuda
        return t
    return torch.full((1,), float(t), device=device, dtype=torch.float32)


def _dot_scale(q, heads, scale):
    """The dot-product attention's scale: as given, or 1 / sqrt(F), F = H / heads, computed in double and rounded to
    fp32 once."""
    if scale is None:
        return float(np.float32(1.0 / math.sqrt(q.shape[1] // int(heads))))
    return float(scale)


class SgPlan:
    """roc_sg_plan for one partition's CSR (rowEnd u64 END offsets, colSrc u32)."""

    def __init__(self, row_left, row_right, col_left, row_end, col_src):
        _lib.require_device()
        assert row_end.dtype == torch.int64 or row_end.dtype == torch.uint64
        assert col_src.dtype in (torch.int32, torch.uint32)
        self.row_left, self.row_right, self.col_left = int(row_left), int(row_right), int(col_left)
        self.row_end, self.col_src = row_end, col_src   # keep alive
        self.nloc = self.row_right - self.row_left + 1
        h = C.c_void_p()
        check(lib.roc_sg_plan_create(self.row_left, self.row_right, self.col_left, _ptr(row_end), _ptr(col_src),
                                     _stream(), C.byref(h)), "roc_sg_plan_create")
        self.handle = h

    def info(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib.roc_sg_plan_info(self.handle, C.byref(a), C.byref(b), C.byref(c)))
        return {"chunks": a.value, "carries": b.value, "heavy_rows": c.value}

    def _rows(self, like, dtype=torch.float32):
        """A new [Nloc][H] output for an input `like` of width H: padded to float4 rows when like's rows are, else
        dense."""
        h = like.shape[1]
        if _ld(like) % 4 == 0:
            return padded(self.nloc, h, like.device, dtype=dtype)
        return torch.empty((self.nloc, h), device=like.device, dtype=dtype)

    def reserve(self, max_h):
        check(lib.roc_sg_plan_reserve(self.handle, int(max_h)), "roc_sg_plan_reserve")

    def forward(self, x, out=None, epilogue=0):
        h = x.shape[1]
        if out is None:
            out = self._rows(x)
        check(lib.roc_sg_forward_planned(self.handle, h, _ptr(x), _ld(x), _ptr(out), _ld(out), int(epilogue),
                                         _stream()), "roc_sg_forward_planned")
        return out

    def forward_bf16(self, x, out=None, epilogue=0):
        """roc_sg_forward_planned_bf16: forward() over bf16 rows (16-byte aligned, ld a multiple of 8, as bf16_padded
        makes them), accumulated in fp32 into an fp32 `out`."""
        assert x.dtype == torch.bfloat16
        if out is None:
            out = padded(self.nloc, x.shape[1], x.device)
        check(lib.roc_sg_forward_planned_bf16(self.handle, x.shape[1], _ptr(x), _ld(x), _ptr(out), _ld(out),
                                              int(epilogue), _stream()), "roc_sg_forward_planned_bf16")
        return out

    def teleport_forward(self, x, t, alpha, beta, epilogue=0, out=None):
        """roc_sg_forward_teleport_planned: post(fmaf(alpha, pre(sum of x over each row's in-edges), beta * t)), pre /
        post the divide by sqrt(in-degree) of SG_EPI_NORM / SG_EPI_NORM_OUT in `epilogue`.  t has one row per plan row,
        any pitch."""
        if out is None:
            out = self._rows(x)
        check(lib.roc_sg_forward_teleport_planned(self.handle, x.shape[1], _ptr(x), _ld(x), float(alpha), _ptr(t),
                                                  _ld(t), float(beta), _ptr(out), _ld(out), int(epilogue), _stream()),
              "roc_sg_forward_teleport_planned")
        return out

    def forward_dropout(self, x, keep, rate, out=None, epilogue=0):
        """roc_sg_forward_dropout_planned: forward() with edge dropout, each kept edge's row added as fmaf(s, x, acc),
        s = 1 / (1 - rate) in fp32, and a dropped edge's row never read.  keep: bit 0 of attn_keep_mask()'s bytes
        (row_is_source=False for the forward, True for the backward over the same CSR); keep=None or rate=0 is
        forward()."""
        out = self._rows(x) if out is None else out
        check(lib.roc_sg_forward_dropout_planned(self.handle, x.shape[1], _ptr(x), _ld(x), _ptr(out), _ld(out),
                                                 int(epilogue), _ptr(keep), float(rate), _stream()),
              "roc_sg_forward_dropout_planned")
        return out

    def teleport_forward_dropout(self, x, t, alpha, beta, keep, rate, epilogue=0, out=None):
        """roc_sg_forward_teleport_dropout_planned: teleport_forward() over forward_dropout()'s sum."""
        out = self._rows(x) if out is None else out
        check(lib.roc_sg_forward_teleport_dropout_planned(self.handle, x.shape[1], _ptr(x), _ld(x), float(alpha),
                                                          _ptr(t), _ld(t), float(beta), _ptr(out), _ld(out),
                                                          int(epilogue), _ptr(keep), float(rate), _stream()),
              "roc_sg_forward_teleport_dropout_planned")
        return out

    def rows_sorted(self):
        """True if every row's sources are strictly increasing (no duplicate edges)."""
        ok = C.c_int()
        check(lib.roc_sg_plan_rows_sorted(self.handle, C.byref(ok), _stream()), "roc_sg_plan_rows_sorted")
        return bool(ok.value)

    def minmax_forward(self, x, aggr, out=None, arg=None):
        """Max (aggr = AGGR_MAX) or min (AGGR_MIN) aggregation -> (out [Nloc][H] fp32, arg [Nloc][H]): arg holds the
        source id of the first edge in CSR order with the extreme value (uint32 bits in int32 storage; SG_NOARG,
        i.e. -1, for a row with no edge)."""
        h = x.shape[1]
        if out is None:
            out = self._rows(x)
        if arg is None:
            arg = self._rows(x, dtype=torch.int32)
        check(lib.roc_sg_minmax_forward_planned(self.handle, int(aggr), h, _ptr(x), _ld(x), _ptr(out), _ld(out),
                                                _ptr(arg), _ld(arg), _stream()), "roc_sg_minmax_forward_planned")
        return out, arg

    def minmax_forward_bf16(self, x, aggr, out=None, arg=None):
        """roc_sg_minmax_forward_planned_bf16: minmax_forward() over bf16 rows (16-byte aligned, ld a multiple of 8, as bf16_padded makes them)."""
        assert x.dtype == torch.bfloat16
        out = self._rows(x) if out is None else out
        arg = self._rows(x, dtype=torch.int32) if arg is None else arg
        check(lib.roc_sg_minmax_forward_planned_bf16(self.handle, int(aggr), x.shape[1], _ptr(x), _ld(x), _ptr(out),
                                                     _ld(out), _ptr(arg), _ld(arg), _stream()),
              "roc_sg_minmax_forward_planned_bf16")
        return out, arg

    def minmax_backward(self, gy, arg, self_base=0, out=None):
        """Gradient of minmax_forward's input: out[u] = sum over row u's edges e (v = col[e]) of gy[v] where
        arg[v] == self_base + u.  gy and arg are indexed like the forward's input."""
        h = gy.shape[1]
        if out is None:
            out = self._rows(gy)
        check(lib.roc_sg_minmax_backward_planned(self.handle, h, int(self_base), _ptr(gy), _ld(gy), _ptr(arg),
                                                 _ld(arg), _ptr(out), _ld(out), _stream()),
              "roc_sg_minmax_backward_planned")
        return out

    def attn_forward(self, x, scores, heads=1, slope=0.2, self_base=0, out=None, stats=None):
        """Attention aggregation (include/roc_b200.h) -> (out [Nloc][H], stats [Nloc][2*heads] = m | 1/Z per head).
        x and scores ([*][2*heads] = s_dst | s_src) are indexed like minmax_forward's input."""
        h = x.shape[1]
        if out is None:
            out = self._rows(x)
        if stats is None:
            stats = torch.empty((self.nloc, 2 * heads), device=x.device)
        check(lib.roc_sg_attn_forward_planned(self.handle, int(heads), h, float(slope), int(self_base), _ptr(x), _ld(x),
                                              _ptr(scores), _ld(scores), _ptr(out), _ld(out), _ptr(stats),
                                              _ld(stats), _stream()), "roc_sg_attn_forward_planned")
        return out, stats

    def attn_forward_bf16(self, x, scores, heads=1, slope=0.2, self_base=0, out=None, stats=None):
        """roc_sg_attn_forward_planned_bf16: attn_forward() over bf16 feature rows (16-byte aligned, ld a multiple of 8, as bf16_padded makes them)."""
        assert x.dtype == torch.bfloat16
        out = self._rows(x) if out is None else out
        stats = torch.empty((self.nloc, 2 * heads), device=x.device) if stats is None else stats
        check(lib.roc_sg_attn_forward_planned_bf16(self.handle, int(heads), x.shape[1], float(slope), int(self_base),
                                                   _ptr(x), _ld(x), _ptr(scores), _ld(scores), _ptr(out), _ld(out),
                                                   _ptr(stats), _ld(stats), _stream()),
              "roc_sg_attn_forward_planned_bf16")
        return out, stats

    def attn_backward(self, x, scores, out, stats, gy, heads=1, slope=0.2, self_base=0, in_grad=None,
                      score_grad=None):
        """Its backward -> (in_grad [Nloc][H], score_grad [Nloc][2*heads] = d s_dst | d s_src).  x, scores, out, stats
        and gy are indexed like the forward's input (for a whole graph: the forward's own outputs)."""
        h = x.shape[1]
        if in_grad is None:
            in_grad = self._rows(x)
        if score_grad is None:
            score_grad = torch.empty((self.nloc, 2 * heads), device=x.device)
        check(lib.roc_sg_attn_backward_planned(self.handle, int(heads), h, float(slope), int(self_base), _ptr(x),
                                               _ld(x), _ptr(scores), _ld(scores), _ptr(out), _ld(out), _ptr(stats),
                                               _ld(stats), _ptr(gy), _ld(gy), _ptr(in_grad), _ld(in_grad),
                                               _ptr(score_grad), _ld(score_grad), _stream()),
              "roc_sg_attn_backward_planned")
        return in_grad, score_grad

    def attn_backward_bf16(self, x, scores, out, stats, gy, heads=1, slope=0.2, self_base=0, in_grad=None,
                           score_grad=None):
        """roc_sg_attn_backward_planned_bf16: attn_backward() with bf16 feature rows x (16-byte aligned, ld a multiple of 8, as bf16_padded makes them)."""
        assert x.dtype == torch.bfloat16
        in_grad = self._rows(x) if in_grad is None else in_grad
        score_grad = torch.empty((self.nloc, 2 * heads), device=x.device) if score_grad is None else score_grad
        check(lib.roc_sg_attn_backward_planned_bf16(self.handle, int(heads), x.shape[1], float(slope), int(self_base),
                                                    _ptr(x), _ld(x), _ptr(scores), _ld(scores), _ptr(out), _ld(out),
                                                    _ptr(stats), _ld(stats), _ptr(gy), _ld(gy), _ptr(in_grad),
                                                    _ld(in_grad), _ptr(score_grad), _ld(score_grad), _stream()),
              "roc_sg_attn_backward_planned_bf16")
        return in_grad, score_grad

    def attn_v2_forward(self, xl, xr, a, heads=1, slope=0.2, out=None, stats=None):
        """GATv2's dynamic attention (roc_sg_attn_v2_forward_planned) -> (out [Nloc][H], stats [Nloc][2*heads] =
        m | 1/Z per head).  xl, xr: [Nloc][H] fp32 rows (the plan covers a whole graph); a: [heads][F] fp32."""
        out = self._rows(xl) if out is None else out
        stats = torch.empty((self.nloc, 2 * heads), device=xl.device) if stats is None else stats
        check(lib.roc_sg_attn_v2_forward_planned(self.handle, int(heads), xl.shape[1], float(slope), _ptr(xl), _ld(xl),
                                                 _ptr(xr), _ld(xr), _ptr(_v2_a(a)), _ptr(out), _ld(out),
                                                 _ptr(stats), _ld(stats), _stream()), "roc_sg_attn_v2_forward_planned")
        return out, stats

    def attn_v2_backward(self, xl, xr, a, out, stats, gy, heads=1, slope=0.2, dxl=None, dxr=None):
        """Its backward over the same CSR (exact on a symmetric graph) -> (dxl, dxr, da [heads][F]).  When xl and xr
        are one tensor its gradient is dxl + dxr."""
        dxl = self._rows(xl) if dxl is None else dxl
        dxr = self._rows(xr) if dxr is None else dxr
        da = torch.empty((a.shape[1], a.shape[0]), device=xl.device)
        check(lib.roc_sg_attn_v2_backward_planned(self.handle, int(heads), xl.shape[1], float(slope), _ptr(xl),
                                                  _ld(xl), _ptr(xr), _ld(xr), _ptr(_v2_a(a)), _ptr(out), _ld(out),
                                                  _ptr(stats), _ld(stats), _ptr(gy), _ld(gy), _ptr(dxl), _ld(dxl),
                                                  _ptr(dxr), _ld(dxr), _ptr(da), _stream()),
              "roc_sg_attn_v2_backward_planned")
        return dxl, dxr, da.t()

    def attn_dot_forward(self, q, k, v, heads=1, scale=None, out=None, stats=None, keep_stats=True):
        """Dot-product attention (roc_sg_attn_dot_forward_planned) -> (out [Nloc][H], stats [Nloc][2*heads] = m | 1/Z
        per head, or None with keep_stats=False, the inference form).  q, k, v: [Nloc][H] fp32 rows (the plan covers a
        whole graph; they may be one tensor or column blocks of one buffer); scale: None for 1 / sqrt(F)."""
        out = self._rows(q) if out is None else out
        if stats is None and keep_stats:
            stats = torch.empty((self.nloc, 2 * heads), device=q.device)
        check(lib.roc_sg_attn_dot_forward_planned(self.handle, int(heads), q.shape[1], _dot_scale(q, heads, scale),
                                                  _ptr(q), _ld(q), _ptr(k), _ld(k), _ptr(v), _ld(v), _ptr(out),
                                                  _ld(out), _ptr(stats), _ld(stats) if stats is not None else 0,
                                                  _stream()), "roc_sg_attn_dot_forward_planned")
        return out, stats

    def attn_dot_backward(self, q, k, v, out, stats, gy, heads=1, scale=None, dq=None, dk=None, dv=None):
        """Its backward over the same CSR (exact on a symmetric graph) -> (dq, dk, dv).  When q, k and v are one
        tensor its gradient is dq + dk + dv."""
        dq = self._rows(q) if dq is None else dq
        dk = self._rows(k) if dk is None else dk
        dv = self._rows(v) if dv is None else dv
        check(lib.roc_sg_attn_dot_backward_planned(self.handle, int(heads), q.shape[1], _dot_scale(q, heads, scale),
                                                   _ptr(q), _ld(q), _ptr(k), _ld(k), _ptr(v), _ld(v), _ptr(out),
                                                   _ld(out), _ptr(stats), _ld(stats), _ptr(gy), _ld(gy), _ptr(dq),
                                                   _ld(dq), _ptr(dk), _ld(dk), _ptr(dv), _ld(dv), _stream()),
              "roc_sg_attn_dot_backward_planned")
        return dq, dk, dv

    def softmax_forward(self, x, t, out=None, stats=None, keep_stats=True):
        """Softmax aggregation with temperature t (roc_sg_softmax_forward_planned) -> (out [Nloc][H], stats
        [Nloc][2H] = m | 1/Z per column, or None with keep_stats=False, the inference form).  x: [Nloc][H] fp32 rows
        (the plan covers a whole graph); t: a float or a 1-element fp32 device tensor."""
        out = self._rows(x) if out is None else out
        if stats is None and keep_stats:
            stats = torch.empty((self.nloc, 2 * x.shape[1]), device=x.device)
        tt = _smx_t(t, x.device)
        check(lib.roc_sg_softmax_forward_planned(self.handle, x.shape[1], _ptr(tt), _ptr(x), _ld(x), _ptr(out),
                                                 _ld(out), _ptr(stats), _ld(stats) if stats is not None else 0,
                                                 _stream()), "roc_sg_softmax_forward_planned")
        return out, stats

    def softmax_backward(self, x, t, out, stats, gy, dx=None, want_dt=True):
        """Its backward over the same CSR (exact on a symmetric graph) -> (dx, dt as a 1-element tensor, or None with
        want_dt=False)."""
        dx = self._rows(x) if dx is None else dx
        dt = torch.empty((1,), device=x.device) if want_dt else None
        tt = _smx_t(t, x.device)
        check(lib.roc_sg_softmax_backward_planned(self.handle, x.shape[1], _ptr(tt), _ptr(x), _ld(x), _ptr(out),
                                                  _ld(out), _ptr(stats), _ld(stats), _ptr(gy), _ld(gy), _ptr(dx),
                                                  _ld(dx), _ptr(dt), _stream()), "roc_sg_softmax_backward_planned")
        return dx, dt

    def attn_keep_mask(self, rate, seed, step, self_base=0, row_is_source=False, out=None):
        """roc_sg_attn_keep_mask: attention dropout's keep bytes of the plan's edges in its edge order, a uint8 [E]
        tensor (bit k keeps head k).  row_is_source=False: the pairs (self_base + r <- col[e]), the forward's and the
        d s_dst pass's; True: the reverse pairs (col[e] <- self_base + r), the planned input-gradient pass's."""
        if out is None:
            out = torch.empty(max(self.num_edges(), 1), dtype=torch.uint8, device="cuda")
        check(lib.roc_sg_attn_keep_mask(self.handle, int(self_base), int(bool(row_is_source)), float(rate), int(seed),
                                        int(step), _ptr(out), _stream()), "roc_sg_attn_keep_mask")
        return out

    def attn_forward_dropout(self, x, scores, keep, rate, heads=1, slope=0.2, self_base=0, out=None, stats=None):
        """roc_sg_attn_forward_dropout_planned (its _bf16 form for a bf16 x): attn_forward() with attention dropout,
        keep from attn_keep_mask(row_is_source=False); keep=None or rate=0 is attn_forward()."""
        out = self._rows(x) if out is None else out
        stats = torch.empty((self.nloc, 2 * heads), device=x.device) if stats is None else stats
        name = "roc_sg_attn_forward_dropout_planned" + ("_bf16" if x.dtype == torch.bfloat16 else "")
        check(getattr(lib, name)(self.handle, int(heads), x.shape[1], float(slope), int(self_base), _ptr(x), _ld(x),
                                 _ptr(scores), _ld(scores), _ptr(out), _ld(out), _ptr(stats), _ld(stats), _ptr(keep),
                                 float(rate), _stream()), name)
        return out, stats

    def attn_backward_dropout(self, x, scores, out, stats, gy, keep, keep_rev, rate, heads=1, slope=0.2, self_base=0,
                              in_grad=None, score_grad=None):
        """roc_sg_attn_backward_dropout_planned (its _bf16 form for a bf16 x): attn_backward() with attention dropout;
        keep as the forward's, keep_rev from attn_keep_mask(row_is_source=True), out the dropped forward output."""
        in_grad = self._rows(x) if in_grad is None else in_grad
        score_grad = torch.empty((self.nloc, 2 * heads), device=x.device) if score_grad is None else score_grad
        name = "roc_sg_attn_backward_dropout_planned" + ("_bf16" if x.dtype == torch.bfloat16 else "")
        check(getattr(lib, name)(self.handle, int(heads), x.shape[1], float(slope), int(self_base), _ptr(x), _ld(x),
                                 _ptr(scores), _ld(scores), _ptr(out), _ld(out), _ptr(stats), _ld(stats), _ptr(gy),
                                 _ld(gy), _ptr(in_grad), _ld(in_grad), _ptr(score_grad), _ld(score_grad), _ptr(keep),
                                 _ptr(keep_rev), float(rate), _stream()), name)
        return in_grad, score_grad

    def weighted_forward(self, x, w, out=None):
        """Edge-weighted sum: out[r] = sum over row r's edges e of w[e - col_left] * x[col[e]]; w is a flat fp32 array in
        the plan's edge order, x is indexed like forward's input."""
        h = x.shape[1]
        if out is None:
            out = self._rows(x)
        check(lib.roc_sg_weighted_forward_planned(self.handle, h, _ptr(x), _ld(x), _ptr(w), _ptr(out), _ld(out),
                                                  _stream()), "roc_sg_weighted_forward_planned")
        return out

    def weighted_forward_bf16(self, x, w, out=None):
        """roc_sg_weighted_forward_planned_bf16: weighted_forward() over bf16 rows (16-byte aligned, ld a multiple of 8, as bf16_padded makes them)."""
        assert x.dtype == torch.bfloat16
        out = self._rows(x) if out is None else out
        check(lib.roc_sg_weighted_forward_planned_bf16(self.handle, x.shape[1], _ptr(x), _ld(x), _ptr(w), _ptr(out),
                                                       _ld(out), _stream()), "roc_sg_weighted_forward_planned_bf16")
        return out

    def edge_dot(self, gy, x, dw=None, accumulate=False):
        """Gradient of weighted_forward's weights: dw[e - col_left] (+)= gy[r] . x[col[e]] for every edge e of row r;
        gy has the plan's rows, x is indexed like the forward's input."""
        if dw is None:
            dw = torch.empty(max(self.num_edges(), 1), device=gy.device)
        check(lib.roc_sg_edge_dot_planned(self.handle, gy.shape[1], _ptr(gy), _ld(gy), _ptr(x), _ld(x), _ptr(dw),
                                          int(bool(accumulate)), _stream()), "roc_sg_edge_dot_planned")
        return dw

    def edge_dot_bf16(self, gy, x, dw=None, accumulate=False):
        """roc_sg_edge_dot_planned_bf16: edge_dot() with bf16 rows x (16-byte aligned, ld a multiple of 8, as bf16_padded makes them)."""
        assert x.dtype == torch.bfloat16
        dw = torch.empty(max(self.num_edges(), 1), device=gy.device) if dw is None else dw
        check(lib.roc_sg_edge_dot_planned_bf16(self.handle, gy.shape[1], _ptr(gy), _ld(gy), _ptr(x), _ld(x), _ptr(dw),
                                               int(bool(accumulate)), _stream()), "roc_sg_edge_dot_planned_bf16")
        return dw

    def num_edges(self):
        return int(self.row_end[-1].item()) - self.col_left if self.nloc else 0

    def close(self):
        if self.handle:
            lib.roc_sg_plan_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _DeviceArray:
    """A borrowed device array, for torch.as_tensor through __cuda_array_interface__."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr or 0, False), "version": 2}


class SgTranspose:
    """roc_sg_transpose of a whole graph's CSR (row_end: N END offsets, col: E sources, every id < N): the exact input
    gradients of the edge-weighted sum, the sum, max / min and attention on any graph."""

    def __init__(self, row_end, col):
        _lib.require_device()
        assert row_end.dtype in (torch.int64, torch.uint64) and col.dtype in (torch.int32, torch.uint32)
        self.row_end, self.col = row_end, col
        self.n = row_end.shape[0]
        self.num_edges = int(row_end[-1].item()) if self.n else 0
        h = C.c_void_p()
        check(lib.roc_sg_transpose_create(self.n, _ptr(row_end), _ptr(col), _stream(), C.byref(h)),
              "roc_sg_transpose_create")
        self.handle = h

    def backward(self, gy, w, out=None):
        """in_grad[j] = sum over the edges e with col[e] = j of w[e] * gy[dst(e)]; gy and in_grad have N rows."""
        h = gy.shape[1]
        if out is None:
            out = padded(self.n, h, gy.device) if _ld(gy) % 4 == 0 else torch.empty((self.n, h), device=gy.device)
        check(lib.roc_sg_weighted_backward_planned(self.handle, h, _ptr(gy), _ld(gy), _ptr(w), _ptr(out), _ld(out),
                                                   _stream()), "roc_sg_weighted_backward_planned")
        return out

    def _rows(self, like):
        """A new [N][H] output for an input `like`: padded to float4 rows when like's rows are, else dense."""
        h = like.shape[1]
        return padded(self.n, h, like.device) if _ld(like) % 4 == 0 else torch.empty((self.n, h), device=like.device)

    def sum_backward(self, gy, epilogue=0, row_end=None, out=None):
        """The sum's exact input gradient: out[j] = epi(sum over the edges e with col[e] = j of gy[dst(e)]).  With
        SG_EPI_NORM, row_end (the graph's, u64 END offsets) is required: NORM divides by j's in-degree in it."""
        h = gy.shape[1]
        if out is None:
            out = self._rows(gy)
        check(lib.roc_sg_transpose_sum_backward(self.handle, h, _ptr(gy), _ld(gy), _ptr(out), _ld(out), int(epilogue),
                                                _ptr(row_end), _stream()), "roc_sg_transpose_sum_backward")
        return out

    def sum_backward_dropout(self, gy, keep, rate, epilogue=0, row_end=None, out=None):
        """roc_sg_transpose_sum_backward_dropout: sum_backward() over the kept edges, each added as fmaf(s, gy, acc);
        keep in the transposed plan's edge order (attn_keep_mask()).  keep=None or rate=0 is sum_backward()."""
        out = self._rows(gy) if out is None else out
        check(lib.roc_sg_transpose_sum_backward_dropout(self.handle, gy.shape[1], _ptr(gy), _ld(gy), _ptr(out),
                                                        _ld(out), int(epilogue), _ptr(row_end), _ptr(keep),
                                                        float(rate), _stream()),
              "roc_sg_transpose_sum_backward_dropout")
        return out

    def minmax_backward(self, gy, arg, out=None):
        """Max / min's exact input gradient for arg from SgPlan.minmax_forward: out[j] = sum over the distinct
        destinations i of j's out-edges of gy[i] where arg[i] == j (a duplicate edge counts once)."""
        h = gy.shape[1]
        if out is None:
            out = self._rows(gy)
        check(lib.roc_sg_transpose_minmax_backward(self.handle, h, _ptr(gy), _ld(gy), _ptr(arg), _ld(arg), _ptr(out),
                                                   _ld(out), _stream()), "roc_sg_transpose_minmax_backward")
        return out

    def attn_backward(self, plan, x, scores, out, stats, gy, heads=1, slope=0.2, in_grad=None, score_grad=None):
        """Attention's exact backward -> (in_grad [N][H], score_grad [N][2*heads] = d s_dst | d s_src), with `plan` the
        whole graph's SgPlan and the other arguments as SgPlan.attn_backward's."""
        h = x.shape[1]
        if in_grad is None:
            in_grad = self._rows(x)
        if score_grad is None:
            score_grad = torch.empty((self.n, 2 * heads), device=x.device)
        check(lib.roc_sg_attn_backward_exact(plan.handle, self.handle, int(heads), h, float(slope), _ptr(x), _ld(x),
                                             _ptr(scores), _ld(scores), _ptr(out), _ld(out), _ptr(stats), _ld(stats),
                                             _ptr(gy), _ld(gy), _ptr(in_grad), _ld(in_grad), _ptr(score_grad),
                                             _ld(score_grad), _stream()), "roc_sg_attn_backward_exact")
        return in_grad, score_grad

    def attn_backward_bf16(self, plan, x, scores, out, stats, gy, heads=1, slope=0.2, in_grad=None, score_grad=None):
        """roc_sg_attn_backward_exact_bf16: attn_backward() with bf16 feature rows x (16-byte aligned, ld a multiple of 8, as bf16_padded makes them)."""
        assert x.dtype == torch.bfloat16
        in_grad = self._rows(x) if in_grad is None else in_grad
        score_grad = torch.empty((self.n, 2 * heads), device=x.device) if score_grad is None else score_grad
        check(lib.roc_sg_attn_backward_exact_bf16(plan.handle, self.handle, int(heads), x.shape[1], float(slope),
                                                  _ptr(x), _ld(x), _ptr(scores), _ld(scores), _ptr(out), _ld(out),
                                                  _ptr(stats), _ld(stats), _ptr(gy), _ld(gy), _ptr(in_grad),
                                                  _ld(in_grad), _ptr(score_grad), _ld(score_grad), _stream()),
              "roc_sg_attn_backward_exact_bf16")
        return in_grad, score_grad

    def attn_v2_backward(self, plan, xl, xr, a, out, stats, gy, heads=1, slope=0.2, dxl=None, dxr=None):
        """roc_sg_attn_v2_backward_exact: SgPlan.attn_v2_backward with the source pass over this transpose, exact on
        any graph.  plan is the forward's plan of the same graph."""
        dxl = plan._rows(xl) if dxl is None else dxl
        dxr = plan._rows(xr) if dxr is None else dxr
        da = torch.empty((a.shape[1], a.shape[0]), device=xl.device)
        check(lib.roc_sg_attn_v2_backward_exact(plan.handle, self.handle, int(heads), xl.shape[1], float(slope),
                                                _ptr(xl), _ld(xl), _ptr(xr), _ld(xr), _ptr(_v2_a(a)), _ptr(out),
                                                _ld(out), _ptr(stats), _ld(stats), _ptr(gy), _ld(gy), _ptr(dxl),
                                                _ld(dxl), _ptr(dxr), _ld(dxr), _ptr(da), _stream()),
              "roc_sg_attn_v2_backward_exact")
        return dxl, dxr, da.t()

    def attn_dot_backward(self, plan, q, k, v, out, stats, gy, heads=1, scale=None, dq=None, dk=None, dv=None):
        """roc_sg_attn_dot_backward_exact: SgPlan.attn_dot_backward with the source pass over this transpose, exact on
        any graph.  plan is the forward's plan of the same graph."""
        dq = plan._rows(q) if dq is None else dq
        dk = plan._rows(k) if dk is None else dk
        dv = plan._rows(v) if dv is None else dv
        check(lib.roc_sg_attn_dot_backward_exact(plan.handle, self.handle, int(heads), q.shape[1],
                                                 _dot_scale(q, heads, scale), _ptr(q), _ld(q), _ptr(k), _ld(k), _ptr(v),
                                                 _ld(v), _ptr(out), _ld(out), _ptr(stats), _ld(stats), _ptr(gy),
                                                 _ld(gy), _ptr(dq), _ld(dq), _ptr(dk), _ld(dk), _ptr(dv), _ld(dv),
                                                 _stream()), "roc_sg_attn_dot_backward_exact")
        return dq, dk, dv

    def softmax_backward(self, plan, x, t, out, stats, gy, dx=None, want_dt=True):
        """roc_sg_softmax_backward_exact: SgPlan.softmax_backward with the source pass over this transpose, exact on
        any graph.  plan is the forward's plan of the same graph."""
        dx = plan._rows(x) if dx is None else dx
        dt = torch.empty((1,), device=x.device) if want_dt else None
        tt = _smx_t(t, x.device)
        check(lib.roc_sg_softmax_backward_exact(plan.handle, self.handle, x.shape[1], _ptr(tt), _ptr(x), _ld(x),
                                                _ptr(out), _ld(out), _ptr(stats), _ld(stats), _ptr(gy), _ld(gy),
                                                _ptr(dx), _ld(dx), _ptr(dt), _stream()),
              "roc_sg_softmax_backward_exact")
        return dx, dt

    def attn_keep_mask(self, rate, seed, step, out=None):
        """roc_sg_attn_keep_mask over the transposed plan (selfBase 0, the row the source): the keep bytes the exact
        backward's input-gradient pass reads, a uint8 [E] tensor in the transposed edge order."""
        plan_t = C.c_void_p()
        check(lib.roc_sg_transpose_info(self.handle, None, None, None, C.byref(plan_t)), "roc_sg_transpose_info")
        if out is None:
            out = torch.empty(max(self.num_edges, 1), dtype=torch.uint8, device="cuda")
        check(lib.roc_sg_attn_keep_mask(plan_t, 0, 1, float(rate), int(seed), int(step), _ptr(out), _stream()),
              "roc_sg_attn_keep_mask")
        return out

    def attn_backward_dropout(self, plan, x, scores, out, stats, gy, keep, keep_t, rate, heads=1, slope=0.2,
                              in_grad=None, score_grad=None):
        """roc_sg_attn_backward_dropout_exact (its _bf16 form for a bf16 x): attn_backward() with attention dropout;
        keep from plan.attn_keep_mask(), keep_t from attn_keep_mask()."""
        in_grad = self._rows(x) if in_grad is None else in_grad
        score_grad = torch.empty((self.n, 2 * heads), device=x.device) if score_grad is None else score_grad
        name = "roc_sg_attn_backward_dropout_exact" + ("_bf16" if x.dtype == torch.bfloat16 else "")
        check(getattr(lib, name)(plan.handle, self.handle, int(heads), x.shape[1], float(slope), _ptr(x), _ld(x),
                                 _ptr(scores), _ld(scores), _ptr(out), _ld(out), _ptr(stats), _ld(stats), _ptr(gy),
                                 _ld(gy), _ptr(in_grad), _ld(in_grad), _ptr(score_grad), _ld(score_grad), _ptr(keep),
                                 _ptr(keep_t), float(rate), _stream()), name)
        return in_grad, score_grad

    def info(self):
        """Copies of the transposed CSR: {"row_end": int64 [N], "col": int32 [E], "perm": int32 [E]} (the uint32 /
        uint64 bits in signed storage) on the device."""
        re_, col, perm = C.c_void_p(), C.c_void_p(), C.c_void_p()
        check(lib.roc_sg_transpose_info(self.handle, C.byref(re_), C.byref(col), C.byref(perm), None),
              "roc_sg_transpose_info")
        torch.cuda.current_stream().synchronize()

        def copy(p, n, typestr):
            if n == 0:
                return torch.empty(0, dtype=torch.int64 if typestr == "<i8" else torch.int32, device="cuda")
            return torch.as_tensor(_DeviceArray(p.value, n, typestr), device="cuda").clone()
        return {"row_end": copy(re_, self.n, "<i8"), "col": copy(col, self.num_edges, "<i4"),
                "perm": copy(perm, self.num_edges, "<i4")}

    def close(self):
        if self.handle:
            lib.roc_sg_transpose_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def sg_launches():
    """The kernel launches of this thread's last planned ScatterGather call (roc_sg_last_call_info): a list of dicts
    kind ("main", "ring", "fixup", ...), red, vec, lanes, nch, grid."""
    return _lib.sg_last_call_info()


def sg_forward(row_left, row_right, col_left, row_end, col_src, x):
    """Plan-less form with the reference kernel's argument list; dense [N][H] in, [Nloc][H] out."""
    assert x.is_contiguous()
    out = torch.empty((row_right - row_left + 1, x.shape[1]), device=x.device, dtype=torch.float32)
    check(lib.roc_sg_forward(row_left, row_right, col_left, x.shape[1], _ptr(row_end), _ptr(col_src), _ptr(x),
                             _ptr(out), _stream()), "roc_sg_forward")
    return out


def sg_backward(row_left, row_right, col_left, row_end, col_src, gy):
    assert gy.is_contiguous()
    out = torch.empty((row_right - row_left + 1, gy.shape[1]), device=gy.device, dtype=torch.float32)
    check(lib.roc_sg_backward(row_left, row_right, col_left, gy.shape[1], _ptr(row_end), _ptr(col_src), _ptr(gy),
                              _ptr(out), _stream()), "roc_sg_backward")
    return out


def build_csr(row_left, row_right, col_left, raw_rows, raw_cols, want_edge_structs=True):
    nloc = row_right - row_left + 1
    eloc = raw_cols.shape[0]
    rp = torch.empty(nloc, dtype=torch.int64, device=raw_rows.device)
    es = torch.empty((max(eloc, 1), 2), dtype=torch.int32, device=raw_rows.device) if want_edge_structs else None
    cs = torch.empty(max(eloc, 1), dtype=torch.int32, device=raw_rows.device)
    check(lib.roc_build_csr(row_left, row_right, col_left, _ptr(raw_rows), _ptr(raw_cols), _ptr(rp), _ptr(es),
                            _ptr(cs), _stream()), "roc_build_csr")
    return rp, (es[:eloc] if es is not None else None), cs[:eloc]


def indegree_norm(row_left, row_right, col_left, row_end, x, out=None, relu_mask_of=None):
    if out is None:
        out = torch.empty_like(x) if x.is_contiguous() else padded(x.shape[0], x.shape[1], x.device)
    check(lib.roc_indegree_norm(row_left, row_right, col_left, x.shape[1], _ptr(row_end), _ptr(x), _ld(x), _ptr(out),
                                _ld(out), _ptr(relu_mask_of), _stream()), "roc_indegree_norm")
    return out


def activation_fwd(x, mode):
    y = torch.empty_like(x)
    check(lib.roc_activation_fwd(x.shape[0], x.shape[1], mode, _ptr(x), _ld(x), _ptr(y), _ld(y), _stream()))
    return y


def activation_bwd(y, dy, mode, dx=None):
    acc = dx is not None
    if dx is None:
        dx = torch.empty_like(y)
    check(lib.roc_activation_bwd(y.shape[0], y.shape[1], mode, _ptr(y), _ld(y), _ptr(dy), _ld(dy), _ptr(dx), _ld(dx),
                                 int(acc), _stream()))
    return dx


def activation_fwd_y_bf16(x, mode=_lib.AC_MODE_RELU, out=None):
    """roc_activation_fwd_y_bf16: relu of fp32 x stored as bf16 (bf16_padded rows unless `out` is given)."""
    if out is None:
        out = bf16_padded(x.shape[0], x.shape[1], x.device)
    check(lib.roc_activation_fwd_y_bf16(x.shape[0], x.shape[1], int(mode), _ptr(x), _ld(x), _ptr(out), _ld(out),
                                        _stream()), "roc_activation_fwd_y_bf16")
    return out


def activation_bwd_y_bf16(y, dy, mode=_lib.AC_MODE_RELU, dx=None):
    """roc_activation_bwd_y_bf16: activation_bwd() with the relu mask read from a bf16 y."""
    acc = dx is not None
    if dx is None:
        dx = torch.empty_like(dy)
    check(lib.roc_activation_bwd_y_bf16(y.shape[0], y.shape[1], int(mode), _ptr(y), _ld(y), _ptr(dy), _ld(dy),
                                        _ptr(dx), _ld(dx), int(acc), _stream()), "roc_activation_bwd_y_bf16")
    return dx


def add_fwd(a, b):
    y = torch.empty_like(a)
    check(lib.roc_add_fwd(a.shape[0], a.shape[1], _ptr(a), _ld(a), _ptr(b), _ld(b), _ptr(y), _ld(y), _stream()))
    return y


def add_bwd(dy, da, acc_a, db, acc_b):
    check(lib.roc_add_bwd(dy.shape[0], dy.shape[1], _ptr(dy), _ld(dy), _ptr(da), _ld(da) if da is not None else 0,
                          int(acc_a), _ptr(db), _ld(db) if db is not None else 0, int(acc_b), _stream()))


def scaled_add_fwd(a, b, alpha, beta, out=None):
    """roc_scaled_add_fwd: fmaf(alpha, a, beta * b), beta * b rounded first."""
    if out is None:
        out = torch.empty_like(a) if a.is_contiguous() else padded(a.shape[0], a.shape[1], a.device)
    check(lib.roc_scaled_add_fwd(a.shape[0], a.shape[1], float(alpha), _ptr(a), _ld(a), float(beta), _ptr(b), _ld(b),
                                 _ptr(out), _ld(out), _stream()), "roc_scaled_add_fwd")
    return out


def scaled_add_bwd(dy, alpha, da, acc_a, beta, db, acc_b):
    """roc_scaled_add_bwd: da (+)= alpha * dy, db (+)= beta * dy (accumulating with fmaf); da or db may be None."""
    check(lib.roc_scaled_add_bwd(dy.shape[0], dy.shape[1], _ptr(dy), _ld(dy), float(alpha), _ptr(da),
                                 _ld(da) if da is not None else 0, int(acc_a), float(beta), _ptr(db),
                                 _ld(db) if db is not None else 0, int(acc_b), _stream()), "roc_scaled_add_bwd")


def dropout_fwd(x, first_row, rate, seed, step, out=None):
    if out is None:
        out = torch.empty_like(x) if x.is_contiguous() else padded(x.shape[0], x.shape[1], x.device)
    check(lib.roc_dropout_fwd(x.shape[0], x.shape[1], first_row, rate, seed, step, _ptr(x), _ld(x), _ptr(out),
                              _ld(out), _stream()), "roc_dropout_fwd")
    return out


def dropout_mask(rows, h, first_row, rate, seed, step, device="cuda"):
    """Packed keep-mask [rows][round_up(ceil(h/32), 4)] uint32 (as int32 storage) of roc_dropout_fwd's mask."""
    ldm = ((h + 31) // 32 + 3) // 4 * 4
    m = torch.empty((rows, ldm), dtype=torch.int32, device=device)
    check(lib.roc_dropout_mask(rows, h, first_row, rate, seed, step, _ptr(m), ldm, _stream()), "roc_dropout_mask")
    return m


def softmax_xent_bwd(logits, labels, mask, compact=False):
    """labels: one-hot fp32 [N][C] (reference format) or, with compact=True, int32 class ids [N]."""
    g = torch.empty_like(logits)
    perf = torch.zeros(7, dtype=torch.int32, device=logits.device)
    if compact:
        check(lib.roc_softmax_xent_bwd_idx(logits.shape[0], logits.shape[1], _ptr(logits), _ld(logits), _ptr(labels),
                                           _ptr(mask), _ptr(g), _ld(g), _ptr(perf), _stream()))
    else:
        check(lib.roc_softmax_xent_bwd(logits.shape[0], logits.shape[1], _ptr(logits), _ld(logits), _ptr(labels),
                                       _ld(labels), _ptr(mask), _ptr(g), _ld(g), _ptr(perf), _stream()))
    return g, _perf_dict(perf)


def _linear_out(x, w, out, y_bf16):
    """The output of a forward Linear and its flags beyond the norm: fp32 rows padded to 4, or with y_bf16 bf16 rows
    padded to 8 (ROC_LINEAR_Y_BF16)."""
    if out is None:
        out = bf16_padded(x.shape[0], w.shape[0], x.device) if y_bf16 else padded(x.shape[0], w.shape[0], x.device)
    assert (out.dtype == torch.bfloat16) == bool(y_bf16)
    return out, (_lib.LINEAR_Y_BF16 if y_bf16 else 0)


def linear_fwd(x, w, activation=0, norm_row_end=None, col_left=0, out=None, y_bf16=False):
    """x [N][in] (ld-padded ok), w [out][in] contiguous (= W_mem[o*in + i]) -> [N][out]; with y_bf16 the result is
    stored in bf16 (round to nearest even)."""
    assert w.is_contiguous()
    out, yflag = _linear_out(x, w, out, y_bf16)
    flags = (_lib.LINEAR_NORM_EPILOGUE if norm_row_end is not None else 0) | yflag
    check(lib.roc_linear_fwd(x.shape[0], x.shape[1], w.shape[0], _ptr(x), _ld(x), _ptr(w), _ptr(out), _ld(out),
                             activation, flags, _ptr(norm_row_end), col_left, _stream()), "roc_linear_fwd")
    return out


def linear_fwd_dropout(x, w, mask, rate, activation=0, norm_row_end=None, col_left=0, out=None, y_bf16=False):
    """linear_fwd(dropout(x)) with the dropout applied while loading x (mask from dropout_mask)."""
    assert w.is_contiguous()
    out, yflag = _linear_out(x, w, out, y_bf16)
    flags = (_lib.LINEAR_NORM_EPILOGUE if norm_row_end is not None else 0) | yflag
    check(lib.roc_linear_fwd_dropout(x.shape[0], x.shape[1], w.shape[0], _ptr(x), _ld(x), _ptr(w), _ptr(out),
                                     _ld(out), activation, flags, _ptr(norm_row_end), col_left, _ptr(mask),
                                     mask.stride(0) if mask is not None else 0, rate, _stream()),
          "roc_linear_fwd_dropout")
    return out


def bf16_padded(rows, h, device="cuda"):
    """[rows][h] view of a zeroed bf16 [rows][round_up(h, 8)] allocation (the bf16 node-tensor layout)."""
    ld = (h + 7) // 8 * 8
    return torch.zeros((rows, ld), device=device, dtype=torch.bfloat16)[:, :h]


def f32_to_bf16(x, out=None):
    """roc_f32_to_bf16: fp32 [rows][h] -> bf16 (round to nearest even); the pad columns of `out`'s rows are zeroed."""
    if out is None:
        out = bf16_padded(x.shape[0], x.shape[1], x.device)
    assert out.dtype == torch.bfloat16
    check(lib.roc_f32_to_bf16(x.shape[0], x.shape[1], _ptr(x), _ld(x), _ptr(out), _ld(out), _stream()),
          "roc_f32_to_bf16")
    return out


def bf16_to_f32(x, out=None):
    """roc_bf16_to_f32: bf16 [rows][h] -> fp32, exactly."""
    assert x.dtype == torch.bfloat16
    if out is None:
        out = padded(x.shape[0], x.shape[1], x.device)
    check(lib.roc_bf16_to_f32(x.shape[0], x.shape[1], _ptr(x), _ld(x), _ptr(out), _ld(out), _stream()),
          "roc_bf16_to_f32")
    return out


def dropout_fwd_bf16(x, first_row, rate, seed, step, out=None):
    """roc_dropout_fwd_bf16: dropout of a bf16 x into fp32."""
    assert x.dtype == torch.bfloat16
    if out is None:
        out = padded(x.shape[0], x.shape[1], x.device)
    check(lib.roc_dropout_fwd_bf16(x.shape[0], x.shape[1], first_row, rate, seed, step, _ptr(x), _ld(x), _ptr(out),
                                   _ld(out), _stream()), "roc_dropout_fwd_bf16")
    return out


def linear_fwd_bf16(x, w, mask=None, rate=0.0, activation=0, norm_row_end=None, col_left=0, out=None, y_bf16=False):
    """roc_linear_fwd_bf16: linear_fwd_dropout with a bf16 x."""
    assert x.dtype == torch.bfloat16 and w.is_contiguous()
    out, yflag = _linear_out(x, w, out, y_bf16)
    flags = (_lib.LINEAR_NORM_EPILOGUE if norm_row_end is not None else 0) | yflag
    check(lib.roc_linear_fwd_bf16(x.shape[0], x.shape[1], w.shape[0], _ptr(x), _ld(x), _ptr(w), _ptr(out), _ld(out),
                                  activation, flags, _ptr(norm_row_end), col_left, _ptr(mask),
                                  mask.stride(0) if mask is not None else 0, rate, _stream()), "roc_linear_fwd_bf16")
    return out


def linear_dw_bf16(x, dy, dw, mask=None, rate=0.0, y=None, activation=0):
    """roc_linear_dw_bf16: dW += dY^T dropout(x) for a bf16 x (with the in-place relu backward of dy first when
    activation is RELU)."""
    assert x.dtype == torch.bfloat16
    ws_bytes = lib.roc_linear_bwd_workspace_bytes(x.shape[0], x.shape[1], dy.shape[1])
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x.device)
    check(lib.roc_linear_dw_bf16(x.shape[0], x.shape[1], dy.shape[1], _ptr(x), _ld(x), _ptr(y),
                                 _ld(y) if y is not None else 0, _ptr(dy), _ld(dy), _ptr(dw), activation, _ptr(ws),
                                 ws_bytes, _ptr(mask), mask.stride(0) if mask is not None else 0, rate, _stream()),
          "roc_linear_dw_bf16")
    return dw


def linear_bwd_dropout(x, w, y, dy, dw, mask, rate, dx=None, activation=0, accumulate_dx=False):
    """linear_bwd where the forward input was dropout(x); dx is the gradient of x (pre-dropout)."""
    ws_bytes = lib.roc_linear_bwd_workspace_bytes(x.shape[0], x.shape[1], w.shape[0])
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x.device)
    check(lib.roc_linear_bwd_dropout(x.shape[0], x.shape[1], w.shape[0], _ptr(x), _ld(x), _ptr(w), _ptr(y),
                                     _ld(y) if y is not None else 0, _ptr(dy), _ld(dy), _ptr(dw), _ptr(dx),
                                     _ld(dx) if dx is not None else 0, activation, int(accumulate_dx), _ptr(ws),
                                     ws_bytes, _ptr(mask), mask.stride(0) if mask is not None else 0, rate,
                                     _stream()), "roc_linear_bwd_dropout")
    return dw, dx


def linear_bwd_fused(x, w, y, dy, dw, dx, activation=0, mask=None, rate=0.0, relu_of=None, norm_row_end=None,
                     col_left=0, accumulate_dx=False, parts=0):
    """roc_linear_bwd_fused: dX epilogue = dropout backward -> relu mask (relu_of > 0) -> / sqrt(deg) [-> += dx].
    parts = 1 / 2 computes only dX / only dW (ROC_LINEAR_BWD_ONLY_DX / _ONLY_DW); dx may be None without dX."""
    ws_bytes = lib.roc_linear_bwd_workspace_bytes(x.shape[0], x.shape[1], w.shape[0])
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x.device)
    a = _lib.LinearBwdArgs()
    a.rows, a.inDim, a.outDim = x.shape[0], x.shape[1], w.shape[0]
    a.X, a.ldX, a.W = x.data_ptr(), _ld(x), w.data_ptr()
    a.Y, a.ldY = (y.data_ptr(), _ld(y)) if y is not None else (None, 0)
    a.dY, a.ldDY, a.dW = dy.data_ptr(), _ld(dy), dw.data_ptr()
    a.dX, a.ldDX = (dx.data_ptr(), _ld(dx)) if dx is not None else (None, 0)
    a.activation, a.accumulate_dX = activation, int(accumulate_dx)
    a.parts = parts
    a.workspace, a.workspaceBytes = ws.data_ptr(), ws_bytes
    if mask is not None:
        a.dropMask, a.ldMask = mask.data_ptr(), mask.stride(0)
    a.dropRate = rate
    if relu_of is not None:
        a.dxReluOf, a.ldReluOf = relu_of.data_ptr(), _ld(relu_of)
    if norm_row_end is not None:
        a.dxNormRowEnd, a.colLeft = norm_row_end.data_ptr(), col_left
    check(lib.roc_linear_bwd_fused(C.byref(a), _stream()), "roc_linear_bwd_fused")
    return dw, dx


def _perf_dict(perf):
    p = perf.cpu()
    return {"trainLoss": float(p[:1].view(torch.float32)[0]), "trainAll": int(p[1]), "testAll": int(p[2]),
            "valAll": int(p[3]), "trainCorrect": int(p[4]), "testCorrect": int(p[5]), "valCorrect": int(p[6])}


def softmax_xent_bwd_norm(logits, labels, mask, row_end, col_left=0, compact=False, with_perf=False):
    """softmax_xent_bwd with the logits' InDegreeNorm backward fused: grad rows divided by sqrt(deg).  Returns the
    gradient, or (gradient, metrics dict as softmax_xent_bwd's) with with_perf=True."""
    g = torch.empty_like(logits)
    perf = torch.zeros(7, dtype=torch.int32, device=logits.device)
    check(lib.roc_softmax_xent_bwd_norm(logits.shape[0], logits.shape[1], _ptr(logits), _ld(logits),
                                        None if compact else _ptr(labels), 0 if compact else _ld(labels),
                                        _ptr(labels) if compact else None, _ptr(mask), _ptr(g), _ld(g),
                                        _ptr(row_end), col_left, _ptr(perf), _stream()), "roc_softmax_xent_bwd_norm")
    return (g, _perf_dict(perf)) if with_perf else g


def sigmoid_xent_bwd(logits, labels_bits, mask, row_end=None, col_left=0, with_metrics=False, out=None):
    """roc_sigmoid_xent_bwd: the multi-label sigmoid cross-entropy's gradient (sigmoid(z) - y on train rows, 0 on the
    rest), divided by sqrt(deg) when row_end is given (the logits' InDegreeNorm backward).  labels_bits: int32 or
    uint32-valued [N][W >= ceil(C / 32)] bit-packed labels (model.pack_multilabels).  Returns the gradient, or
    (gradient, metrics dict as _lib.MultilabelMetrics.as_dict()) with with_metrics=True.  out: the gradient's
    [N][C] (ld-padded ok) buffer."""
    g = torch.empty_like(logits) if out is None else out
    metrics = torch.zeros(18, dtype=torch.float64, device=logits.device) if with_metrics else None
    check(lib.roc_sigmoid_xent_bwd(logits.shape[0], logits.shape[1], _ptr(logits), _ld(logits), _ptr(labels_bits),
                                   _ld(labels_bits), _ptr(mask), _ptr(g), _ld(g), _ptr(row_end), col_left,
                                   _ptr(metrics), _stream()), "roc_sigmoid_xent_bwd")
    if not with_metrics:
        return g
    raw = metrics.cpu().numpy()
    m = _lib.MultilabelMetrics.from_buffer_copy(raw.tobytes())
    return g, m.as_dict()


class BatchNormState:
    """What a training batchnorm_fwd keeps for batchnorm_bwd: a, b (fp32), mean, invstd (fp64), H values each; and the
    workspace (roc_batchnorm_workspace_bytes)."""

    def __init__(self, rows, h, device="cuda"):
        self.a = torch.zeros(h, device=device)
        self.b = torch.zeros(h, device=device)
        self.mean = torch.zeros(h, device=device, dtype=torch.float64)
        self.invstd = torch.zeros(h, device=device, dtype=torch.float64)
        self.ws_bytes = lib.roc_batchnorm_workspace_bytes(rows, h)
        self.ws = torch.empty(max(self.ws_bytes, 16), device=device, dtype=torch.uint8)


def batchnorm_fwd(x, gamma, beta, run_mean, run_var, training=True, relu=False, eps=1e-5, momentum=0.1, state=None,
                  out=None):
    """roc_batchnorm_fwd on a [rows][H] tensor whose rows are padded to float4 (padded()): y = relu?(x a + b) per
    column, with a, b from the batch statistics (training: run_mean / run_var updated in place, `state` filled) or from
    the running statistics.  Returns (y, state)."""
    rows, h = x.shape
    if state is None:
        state = BatchNormState(rows, h, x.device)
    if out is None:
        out = padded(rows, h, x.device)
    check(lib.roc_batchnorm_fwd(rows, h, _ptr(x), _ld(x), _ptr(gamma), _ptr(beta), float(eps), float(momentum),
                                _ptr(run_mean), _ptr(run_var), int(bool(training)), int(bool(relu)), _ptr(out),
                                _ld(out), _ptr(state.a), _ptr(state.b), _ptr(state.mean), _ptr(state.invstd),
                                _ptr(state.ws), state.ws_bytes, _stream()), "roc_batchnorm_fwd")
    return out, state


def batchnorm_bwd(x, dy, gamma, state, relu=False, dx=None, accumulate=False, need_dx=True):
    """roc_batchnorm_bwd after a training batchnorm_fwd that filled `state`: returns (dx, dgamma, dbeta).  dx is
    written into (or with accumulate=True added to) `dx` when given; need_dx=False skips it (dx is then None)."""
    rows, h = x.shape
    dgamma = torch.empty(h, device=x.device)
    dbeta = torch.empty(h, device=x.device)
    if need_dx and dx is None:
        dx = padded(rows, h, x.device)
    if not need_dx:
        dx = None
    check(lib.roc_batchnorm_bwd(rows, h, _ptr(x), _ld(x), _ptr(dy), _ld(dy), int(bool(relu)), _ptr(gamma),
                                _ptr(state.a), _ptr(state.b), _ptr(state.mean), _ptr(state.invstd), _ptr(dgamma),
                                _ptr(dbeta), _ptr(dx), _ld(dx) if dx is not None else 0, int(bool(accumulate)),
                                _ptr(state.ws), state.ws_bytes, _stream()), "roc_batchnorm_bwd")
    return dx, dgamma, dbeta


def layernorm_fwd(x, gamma, beta, relu=False, eps=1e-5, out=None):
    """roc_layernorm_fwd on a [rows][H] tensor whose rows are padded to float4 (padded()): per row,
    y = relu?((x - mean) / sqrt(var + eps) * gamma + beta).  Returns y (padded rows unless `out` is given)."""
    rows, h = x.shape
    if out is None:
        out = padded(rows, h, x.device)
    check(lib.roc_layernorm_fwd(rows, h, _ptr(x), _ld(x), _ptr(gamma), _ptr(beta), float(eps), int(bool(relu)),
                                _ptr(out), _ld(out), _stream()), "roc_layernorm_fwd")
    return out


def layernorm_bwd(x, dy, gamma, beta, relu=False, eps=1e-5, dx=None, accumulate=False, need_dx=True):
    """roc_layernorm_bwd on the inputs of a layernorm_fwd: returns (dx, dgamma, dbeta).  dx is written into (or with
    accumulate=True added to) `dx` when given; need_dx=False skips it (dx is then None)."""
    rows, h = x.shape
    dgamma = torch.empty(h, device=x.device)
    dbeta = torch.empty(h, device=x.device)
    if need_dx and dx is None:
        dx = padded(rows, h, x.device)
    if not need_dx:
        dx = None
    ws_bytes = lib.roc_layernorm_workspace_bytes(rows, h)
    ws = torch.empty(max(ws_bytes, 16), device=x.device, dtype=torch.uint8)
    check(lib.roc_layernorm_bwd(rows, h, _ptr(x), _ld(x), _ptr(dy), _ld(dy), int(bool(relu)), _ptr(gamma), _ptr(beta),
                                float(eps), _ptr(dgamma), _ptr(dbeta), _ptr(dx), _ld(dx) if dx is not None else 0,
                                int(bool(accumulate)), _ptr(ws), ws_bytes, _stream()), "roc_layernorm_bwd")
    return dx, dgamma, dbeta


def _check_a(a, h, heads):
    """the C ABI reads A as a dense [2 * heads][F] fp32 array"""
    assert a.dtype == torch.float32 and a.is_contiguous() and tuple(a.shape) == (2 * int(heads), h // int(heads)), \
        "a must be a contiguous fp32 [2 * heads][F] tensor"


def attn_scores_fwd(x, a, heads, out=None):
    """roc_attn_scores_fwd on fp32 x [rows][H] (H = heads * F) and a [2 * heads][F]: returns s [rows][2 * heads] =
    [s_dst | s_src] (padded rows unless `out` is given)."""
    rows, h = x.shape
    _check_a(a, h, heads)
    if out is None:
        out = padded(rows, 2 * heads, x.device)
    check(lib.roc_attn_scores_fwd(rows, h, int(heads), _ptr(x), _ld(x), _ptr(a), _ptr(out), _ld(out), _stream()),
          "roc_attn_scores_fwd")
    return out


def attn_scores_fwd_bf16(x, a, heads, out=None):
    """roc_attn_scores_fwd_bf16: attn_scores_fwd() on bf16 rows (the bytes of the fp32 call on x.float())."""
    assert x.dtype == torch.bfloat16
    rows, h = x.shape
    _check_a(a, h, heads)
    if out is None:
        out = padded(rows, 2 * heads, x.device)
    check(lib.roc_attn_scores_fwd_bf16(rows, h, int(heads), _ptr(x), _ld(x), _ptr(a), _ptr(out), _ld(out),
                                       _stream()), "roc_attn_scores_fwd_bf16")
    return out


def _attn_scores_bwd(fn, x, a, ds, heads, dx, accumulate, need_dx):
    rows, h = x.shape
    _check_a(a, h, heads)
    if need_dx and dx is None:
        dx = padded(rows, h, x.device)
    if not need_dx:
        dx = None
    da = torch.empty(a.shape, device=x.device)
    ws_bytes = lib.roc_attn_scores_workspace_bytes(rows, h, int(heads))
    ws = torch.empty(max(ws_bytes, 16), device=x.device, dtype=torch.uint8)
    check(getattr(lib, fn)(rows, h, int(heads), _ptr(x), _ld(x), _ptr(a), _ptr(ds), _ld(ds), _ptr(dx),
                           _ld(dx) if dx is not None else 0, int(bool(accumulate)), _ptr(da), _ptr(ws), ws_bytes,
                           _stream()), fn)
    return dx, da


def attn_scores_bwd(x, a, ds, heads, dx=None, accumulate=False, need_dx=True):
    """roc_attn_scores_bwd: returns (dx, da).  dx is written into (accumulate=True: added to) `dx` when given;
    need_dx=False computes da only (dx is then None)."""
    return _attn_scores_bwd("roc_attn_scores_bwd", x, a, ds, heads, dx, accumulate, need_dx)


def attn_scores_bwd_bf16(x, a, ds, heads, dx=None, accumulate=False, need_dx=True):
    """roc_attn_scores_bwd_bf16: attn_scores_bwd() on bf16 rows of x; dx stays fp32."""
    assert x.dtype == torch.bfloat16
    return _attn_scores_bwd("roc_attn_scores_bwd_bf16", x, a, ds, heads, dx, accumulate, need_dx)


def linear_bwd(x, w, y, dy, dw, dx=None, activation=0, accumulate_dx=False):
    ws_bytes = lib.roc_linear_bwd_workspace_bytes(x.shape[0], x.shape[1], w.shape[0])
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x.device)
    check(lib.roc_linear_bwd(x.shape[0], x.shape[1], w.shape[0], _ptr(x), _ld(x), _ptr(w), _ptr(y),
                             _ld(y) if y is not None else 0, _ptr(dy), _ld(dy), _ptr(dw), _ptr(dx),
                             _ld(dx) if dx is not None else 0, activation, int(accumulate_dx), _ptr(ws), ws_bytes,
                             _stream()), "roc_linear_bwd")
    return dw, dx


def adam_update(w, g, m, v, alpha_t, beta1, beta2, wd, eps):
    check(lib.roc_adam_update(w.numel(), alpha_t, beta1, beta2, wd, eps, _ptr(g), _ptr(m), _ptr(v), _ptr(w),
                              _stream()))


def launch_count():
    return lib.roc_launch_count()
