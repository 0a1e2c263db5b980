"""Batches over record sets (FZB_F_PER_RECORD) and find_near_matches_batch_in_each replayed on the emulated build: the
bodies of the -m gpu tests of test_gpu_records_batch.py at the sizes the CPU emulator takes."""
import test_gpu_records_batch as G
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)


def test_emu_records_batch_passes(emu_device):
    G.test_levenshtein_passes_per_record(emu_device, small=True)
    G.test_hamming_passes_per_record(emu_device, small=True)
    G.test_generic_passes_per_record(emu_device, small=True)


def test_emu_records_batch_edges_and_refusals(emu_device):
    G.test_pattern_holding_the_separator_byte(emu_device, small=True)
    G.test_overflow_fallbacks_and_repeats(emu_device, small=True)
    G.test_refusals(emu_device)


def test_emu_records_batch_golden_and_public_api(emu_device):
    G.test_golden_records_in_batches_over_a_set(emu_device, stride=5)
    G.test_public_api(emu_device, small=True)
