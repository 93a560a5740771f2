"""CPU suite, part 2: the C-ABI library loads without a GPU, exports every symbol
the headers declare, its host-side pieces (partitioner, CLI parser) agree with the
oracle bit for bit, and compute entry points refuse to run without a device
instead of falling back to anything."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import oracle
from roc_b200 import _lib, datasets


def declared(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(roc_[a-z0-9_]+)\s*\(", src)))


@pytest.mark.parametrize("header", ["roc_b200.h", "roc_host.h"])
def test_every_declared_symbol_is_exported_and_bound(header):
    names = declared(header)
    assert len(names) > 10
    for n in names:
        assert hasattr(_lib.lib, n), "%s declared in %s but not exported" % (n, header)
        assert n in _lib.PROTOTYPES, "%s has no ctypes prototype" % n


def test_no_undeclared_prototypes():
    names = set(declared("roc_b200.h")) | set(declared("roc_host.h"))
    assert set(_lib.PROTOTYPES) <= names


def test_struct_layouts_match_the_header(tmp_path):
    """The ctypes mirrors of the C structs (roc_linear_bwd_args, roc_gemm_info, roc_sg_launch, roc_sg_call_info,
    roc_host_op_info, roc_perf_metrics) have the C layout: a tiny C program compiled against include/roc_host.h prints
    sizeof / offsetof of every field."""
    structs = [("roc_linear_bwd_args", _lib.LinearBwdArgs), ("roc_gemm_info", _lib.GemmInfo),
               ("roc_sg_launch", _lib.SgLaunch), ("roc_sg_call_info", _lib.SgCallInfo),
               ("struct roc_host_op_info", _lib.HostOpInfo)]
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "roc_host.h"', 'int main(void) {']
    for cname, py in structs:
        prog += ['  printf("%%zu\\n", sizeof(%s));' % cname]
        prog += ['  printf("%%zu\\n", offsetof(%s, %s));' % (cname, f) for f, _ in py._fields_]
    prog += ['  printf("%zu\\n", sizeof(roc_perf_metrics));', '  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    pos = 0
    for cname, py in structs:
        assert out[pos] == C.sizeof(py), cname
        for f, _ in py._fields_:
            pos += 1
            assert getattr(py, f).offset == out[pos], (cname, f)
        pos += 1
    assert pos == len(out) - 1
    assert out[-1] == C.sizeof(_lib.PerfMetrics)


def test_host_op_kinds_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "roc_host.h")).read()
    for i, kind in enumerate(_lib.HOST_OPS):
        assert re.search(r"#define ROC_HOST_OP_%s %d\b" % (kind.upper(), i), hdr), kind
    assert len(re.findall(r"#define ROC_HOST_OP_", hdr)) == len(_lib.HOST_OPS)


def test_gemm_info_hook_without_a_gemm():
    """roc_last_gemm_info rejects a bad kind and reports "none yet" on a thread that has run no Linear."""
    info = _lib.GemmInfo()
    assert _lib.lib.roc_last_gemm_info(3, C.byref(info)) == _lib.ROC_ERR_INVALID
    assert _lib.lib.roc_last_gemm_info(0, None) == _lib.ROC_ERR_INVALID
    import threading
    got = []
    t = threading.Thread(target=lambda: got.append(_lib.last_gemm_info(1)))
    t.start()
    t.join()
    assert got == [{k: 0 for k, _ in _lib.GemmInfo._fields_}]
    assert _lib.lib.roc_last_gemm_path(1) in (0, 1, 2) and _lib.lib.roc_last_gemm_path(7) == 0


def test_sg_call_info_hook_without_a_call():
    """roc_sg_last_call_info rejects a NULL info, reports no launches on a thread that has made no ScatterGather call,
    and its constants match the header's."""
    assert _lib.lib.roc_sg_last_call_info(None) == _lib.ROC_ERR_INVALID
    import threading
    got = []
    t = threading.Thread(target=lambda: got.append(_lib.sg_last_call_info()))
    t.start()
    t.join()
    assert got == [[]]
    hdr = open(os.path.join(ROOT, "include", "roc_b200.h")).read()
    assert int(re.search(r"#define ROC_SG_MAX_LAUNCHES (\d+)", hdr).group(1)) == _lib.SG_MAX_LAUNCHES
    for i, kind in enumerate(_lib.SG_LAUNCH_KINDS):
        assert re.search(r"#define ROC_SG_LAUNCH_%s %d\b" % (kind.upper(), i), hdr), kind


def test_library_is_sm90a_only():
    out = subprocess.run(["cuobjdump", "--list-elf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_partition_matches_oracle_bit_for_bit():
    rng = np.random.RandomState(0)
    cases = []
    for n, pairs, seed in ((50, 100, 1), (300, 1200, 2), (1000, 4500, 3)):
        re_, _ = datasets.uniform_graph(n, pairs, seed=seed)
        cases.append(re_.numpy().astype(np.uint64))
    re_, _ = datasets.rmat_graph(10, 6000, seed=4)
    cases.append(re_.numpy().astype(np.uint64))
    cases.append(np.cumsum(rng.randint(0, 4, size=777)).astype(np.uint64) + 1)   # empty rows allowed
    for row_end in cases:
        n, e = row_end.shape[0], int(row_end[-1])
        for parts in (1, 2, 3, 4, 8):
            k, vb, eb = oracle.partition(row_end, parts)
            gvb = np.zeros((parts, 2), dtype=np.uint32)
            geb = np.zeros((parts, 2), dtype=np.uint64)
            nr = C.c_int(0)
            rc = _lib.lib.roc_partition(n, e, parts, row_end.ctypes.data, gvb.ctypes.data, geb.ctypes.data,
                                        C.cast(C.byref(nr), C.c_void_p))
            assert nr.value == k
            assert (rc == 0) == (k == parts)
            m = min(k, parts)
            assert np.array_equal(gvb[:m], vb[:m]) and np.array_equal(geb[:m], eb[:m])


def test_partition_rejects_bad_arguments():
    vb = np.zeros((2, 2), dtype=np.uint32)
    assert _lib.lib.roc_partition(0, 0, 2, None, vb.ctypes.data, None, None) == _lib.ROC_ERR_INVALID


def test_compute_refuses_without_a_device():
    if _lib.device_count() > 0:
        pytest.skip("a GPU is present")
    h = C.c_void_p()
    rc = _lib.lib.roc_sg_plan_create(0, 9, 0, C.c_void_p(16), C.c_void_p(16), None, C.byref(h))
    assert rc == _lib.ROC_ERR_NO_DEVICE
    with pytest.raises(_lib.RocError):
        _lib.require_device()
    from roc_b200 import model
    with pytest.raises(_lib.RocError):
        model.Host(0, 0, 1)


def test_product_never_touches_the_oracle():
    """The oracle is test infrastructure: nothing shipped may import, link or call it."""
    bad = []
    for base, _, files in os.walk(os.path.join(ROOT, "roc_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cc", ".h")):
                txt = open(os.path.join(base, f)).read()
                if re.search(r"\boracle\b", txt) and f != "__init__.py":
                    bad.append(os.path.join(base, f))
    assert not bad, bad
    ldd = subprocess.run(["ldd", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle" not in ldd and "roc_ref" not in ldd


def test_driver_cli_usage():
    exe = os.path.join(ROOT, "roc_b200", "bin", "roc_gnn")
    assert os.path.exists(exe)
    p = subprocess.run([exe], capture_output=True, text=True)
    assert p.returncode == 2 and "usage" in p.stderr
