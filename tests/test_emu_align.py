"""fzb_align replayed on the emulated build: the bodies of the -m gpu tests of test_gpu_align.py at the sizes the CPU
emulator takes, in reverse and random thread order on grids of one and three SMs, and allocation failures in the
call's own buffers."""
import gc

import numpy as np
import pytest

import test_gpu_align as G
from fuzzysearch_b200 import _native as F
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)
from test_gpu_records import joined, rand
from test_host_align import align_anchored


def test_emu_align_classes_and_golden(emu_device):
    G.test_every_match_of_every_class(emu_device, b"ACGT", small=True)
    G.test_golden_fuzz_matches(emu_device, stride=5)
    G.test_wide_symbols_and_items(emu_device)


def test_emu_align_rows_edges_and_refusals(emu_device):
    G.test_align_in_each_rows(emu_device, small=True)
    G.test_rows_without_matches_and_empty_records(emu_device)
    G.test_generic_table_budget(emu_device)
    G.test_refusals_leave_the_handle_usable(emu_device)


def test_emu_align_edges(emu_device):
    G.test_edges(emu_device)


@pytest.mark.parametrize("sched,sms", [("reverse", "1"), ("reverse", "3"), ("random", "1"), ("random", "3")])
def test_emu_align_thread_order_and_grid_size(emu_device, monkeypatch, sched, sms):
    """The alignments depend neither on the order the threads run in nor on the number of CTAs."""
    monkeypatch.setenv("FZB_EMU_SCHED", sched)
    monkeypatch.setenv("FZB_EMU_SMS", sms)
    rng = np.random.default_rng(9)
    lims = [G.norm(l=3), G.norm(2, 0, 0), G.norm(2, 2, 1, 3), G.norm(l=0)]
    pats = [rand(rng, b"ACGT", m) for m in (40, 20, 33, 10)]
    recs = [rand(rng, b"ACGT", int(x)) for x in rng.integers(0, 90, size=60)]
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    items = []
    for r, t in enumerate(recs):
        for p, (P, lim) in enumerate(zip(pats, lims)):
            w = len(P) if p in (1, 3) else min(len(t), len(P) + int(rng.integers(-3, 4)))
            if 0 <= w <= len(t):
                s = int(rng.integers(0, len(t) - w + 1))
                items.append((p, int(off[r]) + s, int(off[r]) + s + w, t[s:s + w]))
    (start, cost, x, ins, dels), ops, oo, _ = hs.align(pats, *zip(*lims), [i[0] for i in items], [i[1] for i in items],
                                                       [i[2] for i in items], [3] * len(items))
    for k, (p, s, e, T) in enumerate(items):
        want = align_anchored(pats[p], T, lims[p], 3)
        n_ops = len(pats[p]) + int(ins[k])
        got = None if cost[k] < 0 else (int(cost[k]), bytes(ops[int(oo[k]):int(oo[k]) + n_ops]).decode())
        assert got == want, (sched, sms, k)
    hs.close()


def test_emu_align_allocation_failures(emu_device, monkeypatch):
    """FZB_EMU_FAIL_ALLOC=N: every buffer of the call can fail; the call raises CudaError, nothing leaks, and the same
    call on the same handle then answers."""
    P = b"GATTACA"
    recs = [b"xxGATTACAxx", b"TTGACCA", b"", b"GATACA"]
    buf, off = joined(recs)
    lev = G.norm(l=2)

    def call(hs):
        got = hs.align([P], [lev[0]], [lev[1]], [lev[2]], [lev[3]], [0, 0, 0], [2, -1, -1],
                       [9, int(off[2]) - 1, int(off[4]) - 1], [0, 2, 1])
        return [c.tolist() for c in got[0]], bytes(got[1][:int(got[2][-1])])

    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    good = call(hs)
    hs.close()
    gc.collect()
    raised = 0
    for nth in range(1, 7):
        live = F.lib().fzb_emu_live_allocations()
        hs = F.Haystack.from_host(buf)
        hs.set_records(off)
        monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", str(nth))
        try:
            assert call(hs)[0] == good[0], nth
        except F.CudaError:
            raised += 1
        monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", "")
        assert call(hs)[0] == good[0], nth
        assert hs.search_levenshtein(P, 1).triples()[0][:2] == (2, 9)
        hs.close()
        gc.collect()
        assert F.lib().fzb_emu_live_allocations() == live
    assert raised >= 5, raised
