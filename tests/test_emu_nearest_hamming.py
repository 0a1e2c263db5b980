"""The nearest calls under substitutions only replayed on the emulated build: the bodies of the -m gpu tests of
test_gpu_nearest_hamming.py at the sizes the CPU emulator takes, in reverse and random thread order and on grids of one
and three SMs, and allocation failures in the calls' own buffer groups."""
import gc

import numpy as np
import pytest

import test_gpu_nearest_hamming as G
from fuzzysearch_b200 import _native as F
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)
from test_gpu_records import joined, rand

SUB = F.F_SUBSTITUTIONS_ONLY


def test_emu_nearest_hamming_single(emu_device):
    G.test_pattern_sizes_and_short_texts(emu_device, small=True)
    G.test_lengths_around_segments_tiles_and_grid_passes(emu_device, small=True)
    G.test_best_window_at_every_offset_around_the_seams(emu_device, small=True)
    G.test_ties_extremes_and_byte_values(emu_device)
    G.test_record_sets(emu_device, small=True)
    G.test_one_million_reads_one_adapter(emu_device, small=True)


def test_emu_nearest_hamming_batch(emu_device):
    G.test_batch_geometry(emu_device, small=True)
    G.test_batch_patterns_longer_than_records_and_ties(emu_device)
    G.test_batch_byte_values_and_seams(emu_device, small=True)
    G.test_one_million_reads_96_barcodes(emu_device, small=True)


def test_emu_nearest_hamming_api_and_refusals(emu_device):
    G.test_public_api(emu_device, small=True)
    G.test_searches_around_the_call_and_refusals(emu_device)


@pytest.mark.parametrize("sched,sms", [("reverse", "1"), ("reverse", "3"), ("", "1"), ("random", "3")])
def test_emu_nearest_hamming_thread_order_and_grid_size(emu_device, monkeypatch, sched, sms):
    """The answers depend neither on the order the threads run in nor on the number of CTAs."""
    monkeypatch.setenv("FZB_EMU_SCHED", sched)
    monkeypatch.setenv("FZB_EMU_SMS", sms)
    rng = np.random.default_rng(73)
    tile = G.THREADS * G.MIN_SEG
    S = bytearray(rand(rng, b"ACGT", 3 * tile + 77))
    pats = G.mixed_patterns(rng, b"ACGT", 40) + [rand(rng, b"ACGT", 100)]
    for k, at in enumerate((0, G.MIN_SEG - 3, tile - 10, 2 * tile + 5, len(S) - 70)):
        P = pats[k * 7]
        S[at:at + len(P)] = P[:len(P) // 2] + b"N" + P[len(P) // 2 + 1:]
    hs = F.Haystack.from_host(bytes(S))
    for P in pats[::7] + pats[-1:]:
        G.check_handle(hs, P, bytes(S), (sched, sms))
    G.check_whole(hs, pats, bytes(S), (sched, sms))
    hs.close()
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 300, size=60)] + [bytes(S[:2 * tile + 9])]
    hs = F.Haystack.alloc(len(joined(recs)[0]))
    G.check_records(hs, pats[3], recs, (sched, sms))
    G.check_batch_records(hs, pats, recs, ctx=(sched, sms))
    hs.close()


def test_emu_nearest_hamming_allocation_failures(emu_device, monkeypatch):
    """FZB_EMU_FAIL_ALLOC=N on a live handle: the calls' buffer groups are built whole or not at all, also when more
    patterns or a larger record set make them grow; the failed call raises CudaError, nothing leaks, the same call
    then answers."""
    few = [b"GATTACA", b"TTGA"]
    many = few * 20 + [b"GATTACA" * 12]  # more lanes, and a long pattern's record words
    small = [b"xxGATTACAxx", b"TTGACCA", b"", b"GATACA"]
    large = small * 3 + [b"GATTAC"]

    def per_record(hs, pats, recs):
        buf, off = joined(recs)
        hs.upload(buf)
        hs.set_records(off)
        if len(pats) == 1:
            return [c.tolist() for c in hs.nearest_per_record(pats[0], SUB)[:2]]
        return [c.tolist() for c in hs.nearest_best_per_record(pats, SUB)[0]]

    def whole(hs, pats, recs):
        hs.set_records(None)
        hs.upload(joined(recs)[0])
        if len(pats) == 1:
            return hs.nearest_distance(pats[0], SUB)[:3]
        return [c.tolist() for c in hs.nearest_distance_batch(pats, SUB)[:2]]

    hs = F.Haystack.from_host(joined(large)[0])
    cases = [(f, p, r) for f in (per_record, whole) for p in ([few[0]], few, many) for r in (small, large)]
    good = {(f, len(p), len(r)): f(hs, p, r) for f, p, r in cases}
    hs.close()
    gc.collect()
    raised = 0
    for first, pats, grown in ((whole, [few[0]], False), (per_record, [few[0]], True), (whole, few, False),
                               (per_record, few, False), (per_record, many, True)):
        for nth in range(1, 7):
            live = F.lib().fzb_emu_live_allocations()
            hs = F.Haystack.from_host(joined(large)[0])
            recs = large if grown else small
            if grown:  # the group exists: it has to grow
                pre = few if len(pats) > 2 else pats
                assert per_record(hs, pre, small) == good[per_record, len(pre), len(small)]
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", str(nth))
            try:
                assert first(hs, pats, recs) == good[first, len(pats), len(recs)], nth
            except F.CudaError:
                raised += 1
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", "")
            assert first(hs, pats, recs) == good[first, len(pats), len(recs)], nth
            assert whole(hs, [few[0]], small) == good[whole, 1, len(small)], nth
            hs.close()
            gc.collect()
            assert F.lib().fzb_emu_live_allocations() == live
    assert raised >= 5, raised
