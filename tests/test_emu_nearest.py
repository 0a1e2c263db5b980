"""fzb_nearest_distance / fzb_nearest_per_record replayed on the emulated build: the bodies of the -m gpu tests of
test_gpu_nearest.py at the sizes the CPU emulator takes, in reverse thread order and on grids of one and three SMs,
and allocation failures in the call's own buffer group."""
import gc

import numpy as np
import pytest

import test_gpu_nearest as G
from fuzzysearch_b200 import _native as F
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)
from test_gpu_records import joined, rand


def test_emu_nearest_sizes_lengths_and_seams(emu_device):
    G.test_pattern_sizes_and_short_texts(emu_device, small=True)
    G.test_lengths_around_segments_tiles_and_grid_passes(emu_device, small=True)
    G.test_best_occurrence_at_every_offset_around_the_seams(emu_device, small=True)


def test_emu_nearest_values_state_and_refusals(emu_device):
    G.test_ties_extremes_and_byte_values(emu_device)
    G.test_reupload_and_searches_around_the_call(emu_device)
    G.test_refusals_leave_the_handle_usable(emu_device)


def test_emu_nearest_records_and_public_api(emu_device):
    G.test_record_sets(emu_device, small=True)
    G.test_one_million_reads(emu_device, small=True)
    G.test_public_api(emu_device, small=True)


@pytest.mark.parametrize("sched,sms", [("reverse", "1"), ("reverse", "3"), ("", "1"), ("random", "3")])
def test_emu_nearest_thread_order_and_grid_size(emu_device, monkeypatch, sched, sms):
    """The answers depend neither on the order the threads run in nor on the number of CTAs."""
    monkeypatch.setenv("FZB_EMU_SCHED", sched)
    monkeypatch.setenv("FZB_EMU_SMS", sms)
    rng = np.random.default_rng(5)
    tile = G.THREADS * G.MIN_SEG
    S = bytearray(rand(rng, b"ACGT", 5 * tile + 77))
    for m in (20, 50, 100):
        P = rand(rng, b"ACGT", m)
        for at in (0, G.MIN_SEG - 3, tile - m // 2, 4 * tile + 5, len(S) - m):
            S[at:at + m] = P[:m // 2] + b"N" + P[m // 2 + 1:]
        hs = F.Haystack.from_host(bytes(S))
        G.check_handle(hs, P, bytes(S), (sched, sms))
        hs.close()
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 400, size=300)] + [bytes(S[:2 * tile + 9])]
    hs = F.Haystack.alloc(len(joined(recs)[0]))
    G.check_records(hs, rand(rng, b"ACGT", 21), recs, (sched, sms))
    hs.close()


def test_emu_nearest_allocation_failures(emu_device, monkeypatch):
    """FZB_EMU_FAIL_ALLOC=N on a live handle: the calls' buffer group is built whole or not at all, also when a
    larger record set makes it grow; the failed call raises CudaError, nothing leaks, the same call then answers."""
    P = b"GATTACA"
    small = [b"xxGATTACAxx", b"TTGACCA", b"", b"GATACA"]
    large = small * 3 + [b"GATTAC"]

    def per_record(hs, recs):
        buf, off = joined(recs)
        hs.upload(buf)
        hs.set_records(off)
        dist, end, _ = hs.nearest_per_record(P)
        return dist.tolist(), end.tolist()

    def whole(hs, recs):
        hs.upload(joined(recs)[0])
        return hs.nearest_distance(P)[:3]

    hs = F.Haystack.from_host(joined(large)[0])
    good = {(f, len(r)): f(hs, r) for f in (per_record, whole) for r in (small, large)}
    hs.close()
    gc.collect()
    raised = 0
    for first, grown in ((whole, False), (per_record, False), (per_record, True)):
        for nth in range(1, 6):
            live = F.lib().fzb_emu_live_allocations()
            hs = F.Haystack.from_host(joined(large)[0])
            recs = large if grown else small
            if grown:
                assert per_record(hs, small) == good[per_record, len(small)]  # the group exists: it has to grow
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", str(nth))
            try:
                assert first(hs, recs) == good[first, len(recs)], nth
            except F.CudaError:
                raised += 1
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", "")
            assert first(hs, recs) == good[first, len(recs)], nth
            assert whole(hs, small) == good[whole, len(small)], nth
            hs.close()
            gc.collect()
            assert F.lib().fzb_emu_live_allocations() == live
    assert raised >= 4, raised
