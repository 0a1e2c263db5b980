"""The 2-bit n-gram pass of Levenshtein batches on DNA (k_filter_mdense2 and its host side) replayed on the emulated
build: the bodies of the -m gpu tests of test_gpu_dna_lev_batch.py at the sizes the CPU emulator takes."""
import test_gpu_dna_lev_batch as G
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)


def test_emu_dna_lev_batch_shapes(emu_device):
    G.test_key_lengths_and_pattern_shapes(emu_device, small=True)
    G.test_tile_packed_with_occurrences(emu_device, small=True)


def test_emu_dna_lev_batch_chunks_and_offsets(emu_device):
    G.test_tiny_lists_chunk_seams_and_overflow(emu_device, small=True)
    G.test_at_64_bit_offsets(emu_device, small=True)


def test_emu_dna_lev_batch_records_and_one_by_one(emu_device):
    G.test_records_and_public_api(emu_device, small=True)
    G.test_patterns_left_one_by_one(emu_device, small=True)
