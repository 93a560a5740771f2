"""GPU suite: the sum ScatterGather over bf16 rows (roc_sg_forward_planned_bf16) against the fp32 call on the widened
rows, bit for bit.  Both run on the same long-lived plans of sg_matrix.graphs() (empty rows, carries, heavy rows, a
row of 32 carries and one of 33, a slice with global ids and 64-bit edge offsets), at every scalar-path width of
sg_matrix.SCALAR and every rung of the row-shape table on float4 rows, with no epilogue, NORM and NORM | RELU, into
Guarded outputs whose sentinels must survive.  The bf16 rows carry NaN in their pad columns, which the ring's 16-byte
copies read past an odd number of T-columns and never add.  Each call's launch list is the sum's with reduction 12 on
its main kernel or ring and the sum's fix-ups; both kernels must have run.  Then R-MAT scale 22 (config 2's graph) at
H = 64 and 41."""
import numpy as np
import pytest
import torch

import sg_matrix as sm
from roc_b200 import _lib, datasets
from roc_b200 import kernels as K

pytestmark = pytest.mark.gpu
BSUM = _lib.SG_RED_BSUM
EPIS = (0, sm.NORM, sm.NORM | sm.RELU)
VEC_WIDTHS = [4 * qc for qc, _, _ in sm.RUNGS]          # one float4 width per rung: 16 .. 1024 floats
SEEN = set()


def bf16_rows(rng, rows, h, pad=8):
    """bf16 [rows][h] (finite values of both signs and many magnitudes) in rows of round_up(h, 8) + pad elements whose
    pad columns hold NaN."""
    ld = (h + 7) // 8 * 8 + pad
    buf = torch.full((rows, ld), float("nan"), dtype=torch.bfloat16, device=sm.DEV)
    v = rng.standard_normal((rows, h)) * np.exp2(rng.randint(-6, 7, size=(rows, h)))
    buf[:, :h] = torch.from_numpy(v.astype(np.float32)).to(sm.DEV).to(torch.bfloat16)
    return buf[:, :h]


def widened(x):
    """fp32 copy of bf16 rows, in 16-byte aligned rows of round_up(h, 4) + 4 floats"""
    h = x.shape[1]
    out = torch.full((x.shape[0], sm.r4(h) + 4), float("nan"), device=sm.DEV)[:, :h]
    return K.bf16_to_f32(x, out=out)


def bf16_launches(s, vec, h):
    """The fp32 sum's launch list with the main kernel / ring reporting the sum over bf16 rows."""
    return [(k, BSUM if k in ("main", "ring") else r, v, ln, nch, g) for k, r, v, ln, nch, g in sm.planned(s, sm.SUM, vec, h)]


def compare(g, x, h, vec, epi, what):
    xw = widened(x)
    want, got = sm.guarded(g.nloc, h, vec), sm.guarded(g.nloc, h, vec)
    g.plan.forward(xw, out=want.view, epilogue=epi)
    g.plan.forward_bf16(x, out=got.view, epilogue=epi)
    sm.launches(what, bf16_launches(g.sched, vec, h), SEEN)
    torch.cuda.synchronize()
    got.check_guards(what)
    assert np.array_equal(got.bits(), want.bits()), "%s: bits differ from the fp32 call on the widened rows" % what


@pytest.mark.parametrize("name", ["empty", "single", "tiny", "aligned", "straddle", "carry32", "ragged", "slice"])
def test_bf16_sum_matches_fp32_on_widened_rows(name):
    g = sm.graphs()[name]
    rng = np.random.RandomState(sum(map(ord, name)))
    for vec, widths in ((True, VEC_WIDTHS), (False, sm.SCALAR)):
        for h in widths:
            x = bf16_rows(rng, g.n, h)
            for epi in EPIS:
                compare(g, x, h, vec, epi, "%s H=%d %s epi=%d" % (name, h, "float4" if vec else "scalar", epi))


def test_bf16_sum_ran_every_kernel():
    """After the matrix: the ring (float4 rows of 17..64 T-columns) and the register kernel at every rung on both
    paths, all instantiated for the sum over bf16 rows."""
    if not SEEN:
        pytest.skip("run with the matrix")
    want = {x for x in sm.every_instantiation([sm.SUM]) if x[0] in ("main", "ring")}
    want = {(k, BSUM, v, ln, nch) for k, _, v, ln, nch in want}
    assert want <= SEEN, sorted(want - SEEN)
    assert ("ring", BSUM, 4, 32, 1) in SEEN and ("ring", BSUM, 4, 32, 2) in SEEN


def test_bf16_sum_refuses_bad_layouts():
    g = sm.graphs()["tiny"]
    x = bf16_rows(np.random.RandomState(1), g.n, 12)
    out = K.padded(g.nloc, 12)
    bad_ld = torch.zeros((g.n, 20), dtype=torch.bfloat16, device=sm.DEV)[:, :12]     # ld % 8 != 0
    with pytest.raises(_lib.RocError):
        g.plan.forward_bf16(bad_ld, out=out)
    shifted = torch.zeros((g.n * 16 + 4,), dtype=torch.bfloat16, device=sm.DEV)[4:].view(g.n, 16)[:, :12]
    with pytest.raises(_lib.RocError):                                                # base not 16-byte aligned
        g.plan.forward_bf16(shifted, out=out)
    g.plan.forward_bf16(x, out=out)


@pytest.mark.parametrize("h", [64, 41])
def test_bf16_sum_rmat22(h):
    """Config 2's graph (R-MAT scale 22, 4.2 M rows, 69 M edges) at its two aggregation widths."""
    row_end, col = datasets.rmat_graph(22, 1 << 25, seed=1, device=sm.DEV)
    torch.cuda.synchronize()
    n = row_end.shape[0]
    plan = K.SgPlan(0, n - 1, 0, row_end, col)
    g = torch.Generator(device=sm.DEV)
    g.manual_seed(h)
    x = torch.randn((n, (h + 7) // 8 * 8), device=sm.DEV, generator=g).to(torch.bfloat16)[:, :h]
    for epi in EPIS:
        want = plan.forward(widened(x), epilogue=epi)
        got = plan.forward_bf16(x, epilogue=epi)
        kinds = {l["kind"] for l in K.sg_launches()}
        assert kinds & {"main", "ring"}
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), "R-MAT-22 H=%d epi=%d" % (h, epi)
    plan.close()
