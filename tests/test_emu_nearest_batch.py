"""fzb_nearest_distance_batch / fzb_nearest_best_per_record replayed on the emulated build: the bodies of the -m gpu
tests of test_gpu_nearest_batch.py at the sizes the CPU emulator takes, in reverse and random thread order and on
grids of one and three SMs, and allocation failures in the calls' own buffer group."""
import gc

import numpy as np
import pytest

import test_gpu_nearest_batch as G
from fuzzysearch_b200 import _native as F
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)
from test_gpu_records import joined, rand


def test_emu_nearest_batch_geometry_ties_and_bytes(emu_device):
    G.test_group_geometry(emu_device, small=True)
    G.test_ties_empty_records_and_prefill(emu_device)
    G.test_byte_values(emu_device)


def test_emu_nearest_batch_records_api_and_refusals(emu_device):
    G.test_split_records_and_seams(emu_device, small=True)
    G.test_one_million_reads_96_barcodes(emu_device, small=True)
    G.test_public_api(emu_device, small=True)
    G.test_searches_around_the_call_and_refusals(emu_device)


@pytest.mark.parametrize("sched,sms", [("reverse", "1"), ("reverse", "3"), ("", "1"), ("random", "3")])
def test_emu_nearest_batch_thread_order_and_grid_size(emu_device, monkeypatch, sched, sms):
    """The answers depend neither on the order the threads run in nor on the number of CTAs."""
    monkeypatch.setenv("FZB_EMU_SCHED", sched)
    monkeypatch.setenv("FZB_EMU_SMS", sms)
    rng = np.random.default_rng(39)
    pats = G.mixed_patterns(rng, b"ACGT", 40) + [rand(rng, b"ACGT", 100)]
    S = bytearray(rand(rng, b"ACGT", 3 * 8 * G.MIN_SEG * int(sms) + 77))
    for k, at in enumerate((0, G.MIN_SEG - 3, 8 * G.MIN_SEG - 10, len(S) // 2, len(S) - 70)):
        P = pats[k * 7]
        S[at:at + len(P)] = P[:len(P) // 2] + b"N" + P[len(P) // 2 + 1:]
    hs = F.Haystack.from_host(bytes(S))
    G.check_whole(hs, pats, bytes(S), (sched, sms))
    hs.close()
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 300, size=60)] + [bytes(S[:3 * G.MIN_SEG + 9])]
    hs = F.Haystack.alloc(len(joined(recs)[0]))
    G.check_records(hs, pats, recs, G.expected_stacked(pats, recs, ord("x")), (sched, sms))
    hs.close()


def test_emu_nearest_batch_allocation_failures(emu_device, monkeypatch):
    """FZB_EMU_FAIL_ALLOC=N on a live handle: the calls' buffer group is built whole or not at all, also when more
    patterns or a larger record set make it grow; the failed call raises CudaError, nothing leaks, the same call then
    answers."""
    few = [b"GATTACA", b"TTGA"]
    many = few * 20 + [b"GATTACA" * 12]  # more lanes, and a long pattern's record words
    small = [b"xxGATTACAxx", b"TTGACCA", b"", b"GATACA"]
    large = small * 3 + [b"GATTAC"]

    def per_record(hs, pats, recs):
        buf, off = joined(recs)
        hs.upload(buf)
        hs.set_records(off)
        return [c.tolist() for c in hs.nearest_best_per_record(pats)[0]]

    def whole(hs, pats, recs):
        hs.upload(joined(recs)[0])
        return [c.tolist() for c in hs.nearest_distance_batch(pats)[:2]]

    hs = F.Haystack.from_host(joined(large)[0])
    good = {(f, len(p), len(r)): f(hs, p, r) for f in (per_record, whole) for p in (few, many) for r in (small, large)}
    hs.close()
    gc.collect()
    raised = 0
    for first, pats, recs, grown in ((whole, few, small, False), (per_record, few, small, False),
                                     (per_record, many, large, True), (whole, many, small, True)):
        for nth in range(1, 7):
            live = F.lib().fzb_emu_live_allocations()
            hs = F.Haystack.from_host(joined(large)[0])
            if grown:  # the group exists: it has to grow
                assert per_record(hs, few, small) == good[per_record, len(few), len(small)]
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", str(nth))
            try:
                assert first(hs, pats, recs) == good[first, len(pats), len(recs)], nth
            except F.CudaError:
                raised += 1
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", "")
            assert first(hs, pats, recs) == good[first, len(pats), len(recs)], nth
            assert whole(hs, few, small) == good[whole, len(few), len(small)], nth
            hs.close()
            gc.collect()
            assert F.lib().fzb_emu_live_allocations() == live
    assert raised >= 8, raised
