"""Bit-exact pin of the tensor-core forward and dX GEMMs (k_tc_linear) where the persistent CTAs' tile counts differ:
streamed W at uneven and even tiles per CTA and at fewer tiles than CTAs, resident W at 1, 2 and 3 tiles per CTA with a
partial last tile, under every epilogue instantiation.  Each case runs at the whole chip and at two SM budgets set by
roc_set_sm_reserve, one odd and one of 8 SMs (the floor of sm_count()), and must give the digest in
tests/golden/fwd_tile_digests.npz, written by tests/golden/make_golden_tiles.py: forward and dX do not depend on the
SM count."""
import contextlib
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_tiles", os.path.join(HERE, "golden", "make_golden_tiles.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)
F = G.F
GOLDEN = dict(np.load(os.path.join(HERE, "golden", "fwd_tile_digests.npz")))
CASES = G.cases()
EPI = {"plain": 0, "norm": 8, "relu": -1, "mask-norm": 8, "omask": 2, "omask-reluof-norm": 14, "acc": -1}
BUDGETS = ("chip", "odd", "8")
TILES_PER_CTA = {"r1": 1, "r2": 2, "r3": 3}


def nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def budget_sms(budget):
    n = nsm()
    return {"chip": n, "odd": n - 1 if n % 2 == 0 else n - 2, "8": 8}[budget]


@contextlib.contextmanager
def sm_budget(sms):
    """sm_count() = sms for this thread's launches (the reserve is thread-local; the ctypes calls run on this thread)"""
    prev = F._lib.lib.roc_set_sm_reserve(nsm() - sms)
    try:
        yield
    finally:
        F._lib.lib.roc_set_sm_reserve(prev)


def test_budgets_differ():
    sms = [budget_sms(b) for b in BUDGETS]
    assert sms[1] % 2 == 1 and sms[2] == 8 and len(set(sms)) == 3, sms


@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("name", sorted(CASES))
def test_fwd_tiles(name, budget):
    kind, rows, inn, out, epi, streamed = CASES[name]
    sms = budget_sms(budget)
    with sm_budget(sms):
        got, info = F.run_case(kind, rows, inn, out, epi)
    n = out if kind == "fwd" else inn
    nc = 1 if n <= 32 else 2 if n <= 64 else 4
    tiles = -(-rows // 128)
    assert info["path"] == 1, info
    assert info["nc"] == nc and info["grid_y"] == -(-n // (32 * nc)), info
    assert info["epi"] == EPI[epi], info
    assert info["grid_x"] == min(max(sms // info["grid_y"], 1), tiles), (sms, info)
    assert info["w_resident"] == (0 if streamed else 1), info
    tag = name.split("-")[0]
    if budget == "chip" and tag in TILES_PER_CTA:
        assert rows % 128 and -(-tiles // info["grid_x"]) == TILES_PER_CTA[tag], info
    want = GOLDEN["sample_" + name]
    smp = got.reshape(-1)[F.sample_index(got.size)]
    assert F.digest(got) == str(GOLDEN["sha_" + name]), (
        "%s at %d SMs: output bits differ from the golden; sampled values differ by up to %.3e (max |out| %.3e)"
        % (name, sms, float(np.abs(smp.astype(np.float64) - want).max()), float(np.abs(got).max())))
