"""The generic-limit batch (generic_batch_kernels.cuh and its host side) replayed on the emulated build: the bodies of
the -m gpu tests of test_gpu_generic_batch.py, on the CPU."""
import test_gpu_generic_batch as G
from test_emu_kernels import _run, emu_device, emu_lib  # noqa: F401  (fixtures)


def test_emu_generic_batch_mixes(emu_device):
    G.test_ascii_and_dna_mixes(emu_device)
    G.test_duplicates_prefixes_and_sequence_ends(emu_device)
    G.test_window_match_shifted_past_the_hit(emu_device)
    G.test_refusals_come_first(emu_device)


def test_emu_generic_batch_shards(emu_device):
    G.test_batch_at_64_bit_offsets(emu_device)
    _run(G.test_sharded_union_equals_whole, emu_device)


def test_emu_generic_batch_pass_limits(emu_device):
    G.test_overflows_then_a_normal_batch(emu_device)
    _run(G.test_lp_passes_of_64, emu_device)


def test_emu_generic_batch_golden_and_public_api(emu_device):
    G.test_golden_generic_records_in_one_batch_per_sequence(emu_device)
    G.test_public_api_mixes_every_search_class(emu_device)
