"""ctypes front end of tests/minmax_oracle.c: the CPU definition of max / min ScatterGather and its backward.

TEST INFRASTRUCTURE ONLY.  The reference has no max aggregation, so these routines define the semantics
(include/roc_b200.h, roc_sg_minmax_forward_planned) rather than restate the reference.  The library is compiled on
first use into a per-user temporary directory (keyed by the source's hash), so the repository tree stays untouched.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

AGGR_MAX, AGGR_MIN = 1, 2
NOARG = 0xFFFFFFFF

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "minmax_oracle.c")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "roc_minmax_oracle_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, "libminmax_oracle_%s.so" % tag)
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-shared", "-std=gnu11",
                                   "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, path)          # atomic: concurrent test processes never load a half-written file
        _LIB = C.CDLL(path)
    return _LIB


def _p(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def forward(row_left, row_right, col_left, row_end, col_src, x, aggr):
    """x: [N][H] whole matrix indexed by source id -> (out [Nloc][H] fp32, arg [Nloc][H] uint32)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    h = x.shape[1]
    nloc = row_right - row_left + 1
    out = np.empty((nloc, h), dtype=np.float32)
    arg = np.empty((nloc, h), dtype=np.uint32)
    lib().minmax_oracle_forward(C.c_uint32(row_left), C.c_uint32(row_right), C.c_uint64(col_left), C.c_int(h),
                                _p(np.ascontiguousarray(row_end, dtype=np.uint64)),
                                _p(np.ascontiguousarray(col_src, dtype=np.uint32)), _p(x), C.c_int(aggr), _p(out),
                                _p(arg))
    return out, arg


def backward(row_left, row_right, col_left, row_end, col_src, gy, arg, self_base=0, acc64=True):
    """gy, arg: [N][H] indexed by source id -> the input's gradient [Nloc][H]."""
    gy = np.ascontiguousarray(gy, dtype=np.float32)
    arg = np.ascontiguousarray(arg, dtype=np.uint32)
    h = gy.shape[1]
    nloc = row_right - row_left + 1
    out = np.empty((nloc, h), dtype=np.float32)
    lib().minmax_oracle_backward(C.c_uint32(row_left), C.c_uint32(row_right), C.c_uint64(col_left), C.c_int(h),
                                 _p(np.ascontiguousarray(row_end, dtype=np.uint64)),
                                 _p(np.ascontiguousarray(col_src, dtype=np.uint32)), _p(gy), _p(arg),
                                 C.c_uint32(self_base), _p(out), C.c_int(1 if acc64 else 0))
    return out
