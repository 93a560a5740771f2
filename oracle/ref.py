"""ref.py — ctypes front end of oracle/_ref/libroc_ref.so: the REFERENCE's own CUDA
kernels (cut from the reference sources by oracle/Makefile) launched with the
reference's grid shapes on torch CUDA tensors.  TEST INFRASTRUCTURE ONLY: the
second parity witness and the "reference kernel on the same H100" timing column.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(_HERE, "_ref", "libroc_ref.so")
_LIB = None


def available():
    return os.path.exists(PATH)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(PATH)
    return _LIB


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _ok(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed: %d" % (what, rc))


def node_structs(row_end):
    """NodeStruct[] = u64 END offsets (types.h:9-11)."""
    return row_end.to(torch.int64).contiguous()


def edge_structs(col_src, row_end_local, row_left, col_left):
    """EdgeStruct[] {src,dst} built by the reference's own init_graph_kernel (load_task.cu:271-294)."""
    nloc = row_end_local.shape[0]
    eloc = col_src.shape[0]
    rp = torch.empty(nloc, dtype=torch.int64, device=col_src.device)
    es = torch.empty((max(eloc, 1), 2), dtype=torch.int32, device=col_src.device)
    _ok(lib().roc_ref_init_graph(C.c_uint32(row_left), C.c_uint32(row_left + nloc - 1), C.c_uint64(col_left), _p(rp),
                                 _p(es), _p(row_end_local.to(torch.int64).contiguous()),
                                 _p(col_src.to(torch.int32).contiguous())), "init_graph_kernel")
    torch.cuda.synchronize()
    return rp, es[:eloc]


def scatter_gather(row_left, row_right, col_left, row_ptrs, edge_structs_, x, out=None):
    """aggre_coop_kernel with the launch of scattergather_kernel.cu:141-143. x: dense [N][H]."""
    h = x.shape[1]
    assert x.is_contiguous() and h <= 512
    if out is None:
        out = torch.empty((row_right - row_left + 1, h), device=x.device, dtype=torch.float32)
    _ok(lib().roc_ref_scatter_gather(C.c_uint32(row_left), C.c_uint32(row_right), C.c_uint64(col_left), C.c_int(h),
                                     _p(row_ptrs), _p(edge_structs_), _p(x), _p(out)), "aggre_coop_kernel")
    return out


def indegree_norm(row_left, row_right, col_left, row_ptrs, x):
    out = torch.empty_like(x)
    _ok(lib().roc_ref_indegree_norm(C.c_uint32(row_left), C.c_uint32(row_right), C.c_uint64(col_left),
                                    C.c_int(x.shape[1]), _p(row_ptrs), _p(x), _p(out)), "norm_coop_kernel")
    return out


def linear_fwd(x, w, relu=False):
    y = torch.empty((x.shape[0], w.shape[0]), device=x.device, dtype=torch.float32)
    _ok(lib().roc_ref_linear_fwd(C.c_int(x.shape[0]), C.c_int(x.shape[1]), C.c_int(w.shape[0]), _p(w), _p(x), _p(y),
                                 C.c_int(int(relu))), "linear fwd")
    return y


def linear_bwd(x, w, y, dy, dw, dx, relu=False):
    _ok(lib().roc_ref_linear_bwd(C.c_int(x.shape[0]), C.c_int(x.shape[1]), C.c_int(w.shape[0]), _p(w), _p(x), _p(y),
                                 _p(dy), _p(dw), _p(dx), C.c_int(int(relu))), "linear bwd")


def activation_fwd(x, mode):
    y = torch.empty_like(x)
    _ok(lib().roc_ref_activation(C.c_int(x.shape[0]), C.c_int(x.shape[1]), C.c_int(mode), C.c_int(0), _p(x), None,
                                 None, _p(y)), "activation fwd")
    return y


def activation_bwd(x, y, dy, dx, mode):
    """dx += f'(.) * dy  (beta = 1, activation_kernel.cu:128-132)."""
    _ok(lib().roc_ref_activation(C.c_int(y.shape[0]), C.c_int(y.shape[1]), C.c_int(mode), C.c_int(1), _p(y), _p(dy),
                                 _p(x), _p(dx)), "activation bwd")
    return dx


class Perf(C.Structure):
    _fields_ = [("trainLoss", C.c_float), ("trainAll", C.c_int), ("testAll", C.c_int), ("valAll", C.c_int),
                ("trainCorrect", C.c_int), ("testCorrect", C.c_int), ("valCorrect", C.c_int)]


def softmax_xent_bwd(logits, onehot, mask):
    g = torch.empty_like(logits)
    perf = Perf()
    _ok(lib().roc_ref_softmax_xent_bwd(C.c_int(logits.shape[0]), C.c_int(logits.shape[1]), _p(logits), _p(onehot),
                                       _p(mask), _p(g), C.byref(perf)), "softmax")
    torch.cuda.synchronize()
    return g, {k: getattr(perf, k) for k, _ in Perf._fields_}


def adam_update(w, wgrad_replicas, m, v, alpha_t, beta1, beta2, wd, eps):
    count = w.numel()
    reps = wgrad_replicas.numel() // count
    _ok(lib().roc_ref_adam_update(C.c_int(count), C.c_int(reps), C.c_float(alpha_t), C.c_float(beta1),
                                  C.c_float(beta2), C.c_float(wd), C.c_float(eps), _p(wgrad_replicas), _p(m), _p(v),
                                  _p(w)), "adam")


def add_fwd(a, b):
    y = torch.empty_like(a)
    _ok(lib().roc_ref_add_fwd(C.c_longlong(a.numel()), _p(a), _p(b), _p(y)), "op_kernel")
    return y


def glorot(in_dim, out_dim, seed, device="cuda"):
    w = torch.empty((out_dim, in_dim), device=device, dtype=torch.float32)
    _ok(lib().roc_ref_glorot(C.c_int(in_dim), C.c_int(out_dim), C.c_int(seed), _p(w)), "glorot")
    return w


def sync():
    _ok(lib().roc_ref_sync(), "sync")
