"""Every ScatterGather instantiation against an exact or fp64 reference, on graphs built to hit the plan's edge cases.

Each case here is one reduction family on one path at one width, chosen at both ends of a rung of the row-shape
table (sg_matrix.py) and past the widest, where the call is cut into column blocks, and loops over every graph of
sg_matrix.graphs().  roc_sg_last_call_info reports what each call launched; every case asserts the whole launch list
(kind, reduction, VEC, L, NCH, grid), and test_matrix_covered checks at the end that every main kernel and fix-up
instantiation the table can produce was reached.

Features are multiples of 1/16 with |x| <= 8, so every fp32 partial sum on these graphs is exact in any order: the
sum, its norm / relu epilogue, max / min (values and indices) and the max / min backward are compared bit for bit.
A dropped, doubled or misrouted edge, carry or column is then off by a whole term.  Attention keeps the fp64 oracle
and the error bound of test_attn_gpu.py (sg_matrix.close_terms).  Input pad columns hold NaN; outputs sit in
buffers with a guard row above and below and at least 4 guard columns, filled with a sentinel that must survive
(vector path: the pad columns up to round_up(H, 4) may be written, nothing past them).  Each call is repeated and
must give the same bits.

test_one_plan_for_every_call runs one plan, reserved small, on a side stream through growing and shrinking widths,
both paths, every reduction and changing head counts and selfBase; each call must match a fresh plan bit for bit."""
import numpy as np
import pytest
import torch

import attn_oracle as ao
import minmax_oracle as mmo
from conftest import rel_close
from oracle import oracle
from roc_b200 import _lib
from sg_matrix import (ADST, ASRC, ASTAT, ATTN, MASK, MAX, MIN, NORM, RELU, SCALAR, SLOPE, SUM, Guarded, attn_backward,
                       attn_forward, check_bits, close_terms, dev_in, every_instantiation, exact, graphs, guarded,
                       launches, no_new_nan, planned, same_bits, scores_dev, valid_heads)

pytestmark = pytest.mark.gpu
RAN, SEEN = set(), set()
REDUCTIONS = (SUM, MAX, MIN, MASK, ASTAT, ATTN, ADST, ASRC)


# ---------------------------------------------------------------------------------------------------- the matrix ---
# widths at both ends of every rung, and column blocks whose remainders land on different rungs
SUM_V = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 1024, 1025, 1324, 2051]
MM_V = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 700]
ATTN_V = [1, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512]
ATTN_S = [1, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256]
CASES = ([("sum", True, h) for h in SUM_V] + [("sum", False, h) for h in SCALAR] +
         [("minmax", True, h) for h in MM_V] + [("minmax", False, h) for h in SCALAR] +
         [("attn", True, h) for h in ATTN_V] + [("attn", False, h) for h in ATTN_S])


def case_id(c):
    return "%s-%s-%d" % (c[0], "vec" if c[1] else "scalar", c[2])


def repeat_same(first, again, what):
    for a, b in zip(first, again):
        same_bits(a, b, what)


@pytest.mark.parametrize("h", SUM_V, ids=str)
@pytest.mark.parametrize("vec", [True], ids=["vec"])
def test_sum_vector(vec, h):
    run_sum(vec, h)


@pytest.mark.parametrize("h", SCALAR, ids=str)
@pytest.mark.parametrize("vec", [False], ids=["scalar"])
def test_sum_scalar(vec, h):
    run_sum(vec, h)


def run_sum(vec, h):
    for g in graphs().values():
        rng = np.random.RandomState(h * 7 + g.nloc)
        x = exact(rng, g.n, h)
        xd = dev_in(x, vec)
        want = oracle.scatter_gather(g.row_left, g.row_right, g.col_left, g.row_end, g.col, x)
        with np.errstate(divide="ignore", invalid="ignore"):
            normed = want / np.sqrt(g.deg.astype(np.float32))[:, None]          # degree 0: 0 / 0 = NaN (quirk Q5)
        for epi, ref in ((0, want), (NORM, normed), (NORM | RELU, np.maximum(normed, np.float32(0)))):
            what = "%s sum H=%d %s epi=%d" % (g.name, h, "vec" if vec else "scalar", epi)
            outs = []
            for _ in range(2):
                o = guarded(g.nloc, h, vec)
                g.plan.forward(xd, out=o.view, epilogue=epi)
                launches(what, planned(g.sched, SUM, vec, h), SEEN)
                outs.append(o)
            assert ref.dtype == np.float32
            check_bits(outs[0].host(), ref, what)
            outs[0].check_guards(what)
            repeat_same(outs[:1], outs[1:], what)
    RAN.add(case_id(("sum", vec, h)))


def minmax_call(plan, xd, aggr, rows, h, vec):
    o, a = guarded(rows, h, vec), guarded(rows, h, vec, index=True)
    plan.minmax_forward(xd, aggr, out=o.view, arg=a.view)
    return o, a


@pytest.mark.parametrize("h", MM_V, ids=str)
@pytest.mark.parametrize("vec", [True], ids=["vec"])
def test_minmax_vector(vec, h):
    run_minmax(vec, h)


@pytest.mark.parametrize("h", SCALAR, ids=str)
@pytest.mark.parametrize("vec", [False], ids=["scalar"])
def test_minmax_scalar(vec, h):
    run_minmax(vec, h)


def run_minmax(vec, h):
    """Max and min (values and indices bit-exact, ties resolved to the first edge) and their backward (exact)."""
    for g in graphs().values():
        rng = np.random.RandomState(h * 11 + g.nloc)
        x, gy = exact(rng, g.n, h), exact(rng, g.n, h)
        xd, gd = dev_in(x, vec), dev_in(gy, vec)
        for aggr, red in ((_lib.AGGR_MAX, MAX), (_lib.AGGR_MIN, MIN)):
            what = "%s %s H=%d %s" % (g.name, "max" if red == MAX else "min", h, "vec" if vec else "scalar")
            want, warg = mmo.forward(g.row_left, g.row_right, g.col_left, g.row_end, g.col, x, aggr)
            runs = []
            for _ in range(2):
                runs.append(minmax_call(g.plan, xd, aggr, g.nloc, h, vec))
                launches(what, planned(g.sched, red, vec, h), SEEN)
            o, a = runs[0]
            assert np.array_equal(o.host().view(np.int32), want.view(np.int32)), "%s: values differ" % what
            assert np.array_equal(a.host().view(np.uint32), warg), "%s: indices differ" % what
            o.check_guards(what)
            a.check_guards(what + " arg")
            repeat_same(runs[0], runs[1], what)
            # the backward gathers the indices of every id: the forward's own for a whole graph, else the whole graph's
            if g.full is None:
                arg_all, warg_all = a.view, warg
            else:
                _, warg_all = mmo.forward(0, g.full.n - 1, 0, g.full.row_end, g.full.col, x, aggr)
                arg_all = minmax_call(g.full.plan, xd, aggr, g.full.n, h, vec)[1].view
            wgrad = mmo.backward(g.row_left, g.row_right, g.col_left, g.row_end, g.col, gy, warg_all,
                                 self_base=g.self_base)
            what = what + " backward"
            grads = []
            for _ in range(2):
                o2 = guarded(g.nloc, h, vec)
                g.plan.minmax_backward(gd, arg_all, self_base=g.self_base, out=o2.view)
                launches(what, planned(g.sched, MASK, vec, h), SEEN)
                grads.append(o2)
            got = grads[0].host()
            bad = got != wgrad
            assert not bad.any(), "%s: %d/%d elements differ from the exact reference, first at %s" % (
                what, int(bad.sum()), bad.size, np.argwhere(bad)[0])
            grads[0].check_guards(what)
            repeat_same(grads[:1], grads[1:], what)
    RAN.add(case_id(("minmax", vec, h)))


def scores_dev(s):
    """score / stats inputs: [*][2 heads] with NaN in 3 pad columns."""
    return dev_in(s, False, ld=s.shape[1] + 3)


def attn_call(plan, xd, sd, heads, h, vec, rows, self_base):
    o, st = guarded(rows, h, vec), Guarded(rows, 2 * heads, 2 * heads + 4, 2 * heads)
    plan.attn_forward(xd, sd, heads, SLOPE, self_base=self_base, out=o.view, stats=st.view)
    return o, st


def attn_bwd_call(plan, xd, sd, o_all, st_all, gd, heads, h, vec, rows, self_base):
    ig, sg = guarded(rows, h, vec), Guarded(rows, 2 * heads, 2 * heads + 4, 2 * heads)
    plan.attn_backward(xd, sd, o_all, st_all, gd, heads, SLOPE, self_base=self_base, in_grad=ig.view,
                       score_grad=sg.view)
    return ig, sg


def attn_close(got, want, mag, what, eps):
    no_new_nan(got, want, what)
    close_terms(got, want, mag, what, eps)


@pytest.mark.parametrize("h", ATTN_V, ids=str)
@pytest.mark.parametrize("vec", [True], ids=["vec"])
def test_attn_vector(vec, h):
    run_attn(vec, h)


@pytest.mark.parametrize("h", ATTN_S, ids=str)
@pytest.mark.parametrize("vec", [False], ids=["scalar"])
def test_attn_scalar(vec, h):
    run_attn(vec, h)


def run_attn(vec, h):
    """Forward and backward at every valid head count, against the fp64 oracle (test_attn_gpu.check's bounds)."""
    for g in graphs().values():
        for heads in valid_heads(h):
            rng = np.random.RandomState(h * 13 + heads + g.nloc)
            x, gy = exact(rng, g.n, h), exact(rng, g.n, h)
            s = rng.randn(g.n, 2 * heads).astype(np.float32)
            xd, gd, sd = dev_in(x, vec), dev_in(gy, vec), scores_dev(s)
            what = "%s attention H=%d heads=%d %s" % (g.name, h, heads, "vec" if vec else "scalar")
            kw = dict(self_base=g.self_base, col_left=g.col_left)
            fw = []
            for _ in range(2):
                fw.append(attn_call(g.plan, xd, sd, heads, h, vec, g.nloc, g.self_base))
                launches(what + " forward", attn_forward(g.sched, vec, h, heads), SEEN)
            out, stats = fw[0]
            want, wstats = ao.forward(g.row_end, g.col, x, s, heads, SLOPE, **kw)
            mag = ao.forward(g.row_end, g.col, np.abs(x), s, heads, SLOPE, **kw)[0]
            attn_close(out.host(), want, mag, what + " forward", 0.0)
            no_new_nan(stats.host(), wstats, what + " stats")
            rel_close(stats.host(), wstats, rtol=1e-4, what=what + " stats")
            for b in (out, stats):
                b.check_guards(what + " forward")
            repeat_same(fw[0], fw[1], what + " forward")
            # the backward reads out / stats of every id: the forward's own for a whole graph, else the whole graph's
            if g.full is None:
                o_all, st_all = out.view, stats.view
            else:
                o_all, st_all = (b.view for b in attn_call(g.full.plan, xd, sd, heads, h, vec, g.full.n, 0))
            bw = []
            n = max(g.id_end, g.self_base + g.nloc)             # the ids the node records cover
            for _ in range(2):
                bw.append(attn_bwd_call(g.plan, xd, sd, o_all, st_all, gd, heads, h, vec, g.nloc, g.self_base))
                launches(what + " backward", attn_backward(g.sched, g.sched, vec, h, n), SEEN)
            ig, sg = bw[0]
            args = (g.row_end, g.col, x, s, o_all.cpu().numpy(), st_all.cpu().numpy())
            wig, wsg = ao.backward(*args, gy, heads, SLOPE, **kw)
            mig = ao.backward(*args, np.abs(gy), heads, SLOPE, **kw)[0]
            msg = ao.score_grad_magnitude(*args, gy, heads, SLOPE, **kw)
            attn_close(ig.host(), wig, mig, what + " input gradient", 0.0)
            sgh = sg.host()
            attn_close(sgh[:, :heads], wsg[:, :heads], msg[:, :heads], what + " d s_dst", 1e-6)
            attn_close(sgh[:, heads:], wsg[:, heads:], msg[:, heads:], what + " d s_src", 1e-6)
            for b in (ig, sg):
                b.check_guards(what + " backward")
            repeat_same(bw[0], bw[1], what + " backward")
    RAN.add(case_id(("attn", vec, h)))


# ----------------------------------------------------------------------------------------------- one long plan ---
def run_step(plan, g, step, inputs):
    """One call of the sequence below on `plan` -> its guarded outputs."""
    kind, vec, h = step[:3]
    x, gy, arg, s, o_all, st_all = (inputs[k] for k in ("x", "gy", "arg", "s", "o", "st"))
    xd, gd = x[(vec, h)], gy[(vec, h)]
    if kind == "sum":
        o = guarded(g.nloc, h, vec)
        plan.forward(xd, out=o.view, epilogue=step[3])
        return [o]
    if kind in ("max", "min"):
        return list(minmax_call(plan, xd, _lib.AGGR_MAX if kind == "max" else _lib.AGGR_MIN, g.nloc, h, vec))
    if kind == "mask":
        o = guarded(g.nloc, h, vec)
        plan.minmax_backward(gd, arg[(vec, h)], self_base=step[3], out=o.view)
        return [o]
    heads, self_base = step[3], step[4]
    sd = s[heads]
    fw = attn_call(plan, xd, sd, heads, h, vec, g.nloc, self_base)
    bw = attn_bwd_call(plan, xd, sd, o_all[(vec, h)], st_all[heads], gd, heads, h, vec, g.nloc, self_base)
    return list(fw) + list(bw)


def run_sequence(g, steps, rows, reserve):
    """Runs `steps` on one plan, on a side stream, after reserving it for width `reserve`, and each step on a fresh
    plan on the default stream; the outputs must agree bit for bit."""
    rng = np.random.RandomState(77)
    inputs = {k: {} for k in ("x", "gy", "arg", "s", "o", "st")}
    for step in steps:
        kind, vec, h = step[:3]
        key = (vec, h)
        if key not in inputs["x"]:
            inputs["x"][key] = dev_in(exact(rng, rows, h), vec)
            inputs["gy"][key] = dev_in(exact(rng, rows, h), vec)
            inputs["o"][key] = dev_in(exact(rng, rows, h), vec)
            a = guarded(rows, h, vec, index=True)
            ids = rng.randint(g.self_base, g.self_base + g.nloc, size=(rows, h))    # often a local row's own id
            a.view.copy_(torch.from_numpy(ids.astype(np.int32)))
            inputs["arg"][key] = a.view
        if kind == "attn" and step[3] not in inputs["s"]:
            heads = step[3]
            inputs["s"][heads] = scores_dev(rng.randn(rows, 2 * heads).astype(np.float32))
            st = np.concatenate([rng.randn(rows, heads), rng.uniform(0.05, 1.0, (rows, heads))], axis=1)
            inputs["st"][heads] = scores_dev(st.astype(np.float32))
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        plan = g.new_plan()
        plan.reserve(reserve)
    for i, step in enumerate(steps):
        with torch.cuda.stream(side):
            got = run_step(plan, g, step, inputs)
        side.synchronize()
        fresh = g.new_plan()
        want = run_step(fresh, g, step, inputs)
        torch.cuda.synchronize()
        fresh.close()
        for k, (a, b) in enumerate(zip(got, want)):
            assert np.array_equal(a.bits(), b.bits()), "%s step %d %s output %d: the long-lived plan differs from a " \
                                                       "fresh one" % (g.name, i, step, k)
    plan.close()


def test_one_plan_for_every_call():
    """Reserve-then-grow (the reserved carries are released on the stream), carries grown by attention and the
    index carries sized from them, shrinking widths, both paths, head counts 1 -> 8 -> 2, and selfBase moved past
    the ids the graph has (the attention record grows)."""
    g = graphs()["slice"]
    rl = g.self_base
    rows = g.n + g.nloc + 8                    # ids up to selfBase + nloc with selfBase = n
    steps = [("sum", True, 8, NORM), ("max", True, 100), ("mask", True, 100, rl), ("attn", False, 37, 1, rl),
             ("sum", False, 257, 0), ("attn", True, 512, 8, rl), ("min", True, 513), ("mask", True, 513, rl + 3),
             ("attn", True, 64, 2, g.n), ("mask", False, 33, rl + 5), ("sum", True, 4, NORM | RELU),
             ("max", False, 5), ("attn", False, 256, 8, rl), ("sum", True, 1025, 0), ("attn", True, 64, 2, rl)]
    run_sequence(g, steps, rows, 8)


def test_zero_carry_plan_through_attention():
    """A plan with no carries: every buffer the carries would need stays empty, through reserve and every pass."""
    g = graphs()["tiny"]
    assert g.sched.carries == 0
    steps = [("attn", True, 8, 1, 0), ("attn", True, 256, 8, 0), ("attn", False, 64, 2, 0), ("sum", True, 700, 0),
             ("max", False, 300), ("attn", False, 1, 1, 3)]
    run_sequence(g, steps, g.n + 8, 64)


# ---------------------------------------------------------------------------------------------------- coverage ---
def test_matrix_covered():
    """Every main-kernel and fix-up instantiation the row-shape table can produce was reached, and the matrix ran
    every case."""
    wanted = {case_id(c) for c in CASES}
    if not wanted <= RAN:
        pytest.skip("%d of the %d matrix cases did not run in this process" % (len(wanted - RAN), len(wanted)))
    want = every_instantiation(REDUCTIONS)
    missing = want - SEEN
    assert not missing, "never launched: %s" % sorted(missing)
    assert SEEN <= want, "launched outside the table: %s" % sorted(SEEN - want)
