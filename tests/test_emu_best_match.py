"""best_match_in_each / fzb_best_per_record replayed on the emulated build: the bodies of the -m gpu tests of
test_gpu_best_match.py at the sizes the CPU emulator takes, and allocation failures in the call's own buffer group."""
import gc

import numpy as np
import pytest

import test_gpu_best_match as G
from fuzzysearch_b200 import _native as F
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)
from test_gpu_records import joined


def test_emu_best_match_passes(emu_device):
    G.test_every_shared_pass(emu_device, small=True)
    G.test_dna_levenshtein_pass_and_chunk_seams(emu_device, small=True)


def test_emu_best_match_overflows_and_refusals(emu_device):
    G.test_overflowing_passes_leave_nothing_behind(emu_device, small=True)
    G.test_refusals_leave_the_handle_as_it_was(emu_device)


def test_emu_best_match_ties_edges_and_public_api(emu_device):
    G.test_ties(emu_device)
    G.test_record_edges(emu_device, small=True)
    G.test_public_api(emu_device, small=True)


def test_emu_best_match_allocation_failures(emu_device, monkeypatch):
    """FZB_EMU_FAIL_ALLOC=N on a live handle: the call's buffer group (the words, the ordinals) is built whole or not
    at all, also when a larger record set makes it grow; the failed call raises CudaError, the same call then answers."""
    pats = [b"GATTACA", b"TTGACCA", b"CATCAT"]
    lims = list(zip(*[G.lev4(1)] * 3))
    small = [b"xxGATTACAxx", b"TTGACCA", b"", b"CATCAT"]
    large = small * 3 + [b"GATACA"]

    def call(hs, recs):
        buf, off = joined(recs)
        hs.upload(buf)
        hs.set_records(off)
        return [c.tolist() for c in hs.best_per_record(pats, *lims)[0]]

    hs = F.Haystack.from_host(joined(large)[0])
    good_small, good_large = call(hs, small), call(hs, large)
    hs.close()
    raised = 0
    for recs_first, good_first in ((small, good_small), (large, good_large)):
        for nth in range(1, 12):
            hs = F.Haystack.from_host(joined(large)[0])
            if recs_first is large:
                assert call(hs, small) == good_small  # the group exists: the larger set makes it grow
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", str(nth))
            try:
                assert call(hs, recs_first) == good_first, nth
            except F.CudaError:
                raised += 1
            monkeypatch.setenv("FZB_EMU_FAIL_ALLOC", "")
            assert call(hs, recs_first) == good_first, nth
            assert call(hs, small) == good_small, nth
            hs.close()
            gc.collect()
    assert raised >= 4, raised
