"""The anchored nearest calls replayed on the emulated build: the bodies of the -m gpu tests of test_gpu_anchored.py
at the sizes the CPU emulator takes, in reverse and random thread order and on grids of one and three SMs, and
allocation failures in the calls' own buffer groups."""
import gc

import numpy as np
import pytest

import test_gpu_anchored as G
from fuzzysearch_b200 import _native as F
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)
from test_gpu_records import joined, rand


def test_emu_anchored_single_and_batch(emu_device):
    G.test_pattern_sizes_and_record_lengths(emu_device, small=True)
    G.test_lane_groups_and_cta_rows(emu_device, small=True)
    G.test_ties_extremes_separators_and_byte_values(emu_device)
    G.test_long_record_among_reads_and_mirror_identity(emu_device, small=True)


def test_emu_anchored_api_and_refusals(emu_device):
    G.test_anchored_against_unanchored(emu_device, small=True)
    G.test_public_api_and_align(emu_device, small=True)
    G.test_one_million_reads_96_barcodes(emu_device, small=True)
    G.test_searches_around_the_call_and_refusals(emu_device)


@pytest.mark.parametrize("sched,sms", [("reverse", "1"), ("reverse", "3"), ("", "1"), ("random", "3")])
def test_emu_anchored_thread_order_and_grid_size(emu_device, monkeypatch, sched, sms):
    """The answers depend neither on the order the threads run in nor on the number of CTAs."""
    monkeypatch.setenv("FZB_EMU_SCHED", sched)
    monkeypatch.setenv("FZB_EMU_SMS", sms)
    rng = np.random.default_rng(74)
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 120, size=700)]
    pats = G.mixed_patterns(rng, b"ACGT", 40, 1, 40) + [rand(rng, b"ACGT", 90)]
    for i, P in enumerate(pats):
        r = recs[3 * i]
        recs[3 * i] = P + r if i % 2 else r + P
    hs = F.Haystack.alloc(len(joined(recs)[0]) + 4096)
    for anchor, subs in G.BOTH:
        G.check_records(hs, pats[5], recs, anchor, subs, (sched, sms))
        G.check_records(hs, pats[-1], recs, anchor, subs, (sched, sms))
        G.check_batch(hs, pats[:3], recs, anchor, subs, (sched, sms))
        G.check_batch(hs, pats, recs, anchor, subs, (sched, sms))
    hs.close()


def test_emu_anchored_allocation_failures(emu_device, monkeypatch):
    """FZB_EMU_FAIL_ALLOC=N on a live handle: the calls' buffer groups are built whole or not at all, also when more
    patterns or a larger record set make them grow; the failed call raises CudaError, nothing leaks, the same call
    then answers."""
    few = [b"GATTACA", b"TTGA"]
    many = few * 20 + [b"GATTACA" * 12]  # more lanes, and a long pattern's record words
    small = [b"xxGATTACAxx", b"TTGACCA", b"", b"GATACA"]
    large = small * 3 + [b"GATTAC"]
    flags = (G.START, G.END | G.SUB)

    def run(hs, pats, recs):
        buf, off = joined(recs)
        hs.upload(buf)
        hs.set_records(off)
        if len(pats) == 1:
            return [[c.tolist() for c in hs.nearest_per_record(pats[0], f)[:2]] for f in flags]
        return [[c.tolist() for c in hs.nearest_best_per_record(pats, f)[0]] for f in flags]

    hs = F.Haystack.from_host(joined(large)[0])
    good = {(len(p), len(r)): run(hs, p, r) for p in ([few[0]], few, many) for r in (small, large)}
    hs.close()
    gc.collect()
    raised = 0
    for pats, grown in (([few[0]], False), ([few[0]], True), (few, False), (many, True)):
        for nth in range(1, 7):
            live = F.lib().fzb_emu_live_allocations()
            hs = F.Haystack.from_host(joined(large)[0])
            recs = large if grown else small
            if grown:  # the group exists: it has to grow
                pre = few if len(pats) > 2 else pats
                assert run(hs, pre, small) == good[len(pre), len(small)]
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", str(nth))
            try:
                assert run(hs, pats, recs) == good[len(pats), len(recs)], nth
            except F.CudaError:
                raised += 1
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", "")
            assert run(hs, pats, recs) == good[len(pats), len(recs)], nth
            hs.close()
            gc.collect()
            assert F.lib().fzb_emu_live_allocations() == live
    assert raised >= 4, raised
