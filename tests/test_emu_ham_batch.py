"""The substitutions-only batch (k_ham_batch_scan and its host side) replayed on the emulated build: the bodies of the
-m gpu tests of test_gpu_ham_batch.py, on the CPU."""
import test_gpu_ham_batch as G
from test_emu_kernels import _run, emu_device, emu_lib  # noqa: F401  (fixtures)


def test_emu_ham_batch_mixes(emu_device):
    G.test_dna_and_ascii_mixes(emu_device)
    G.test_two_bit_keys_on_wide_symbols(emu_device)


def test_emu_ham_batch_exactly_once(emu_device):
    G.test_each_start_exactly_once(emu_device)


def test_emu_ham_batch_shards(emu_device):
    G.test_batch_at_64_bit_offsets(emu_device)
    _run(G.test_sharded_union_equals_whole, emu_device)


def test_emu_ham_batch_pass_limits(emu_device):
    G.test_pass_limits(emu_device)


def test_emu_ham_batch_public_api(emu_device):
    G.test_public_api_mixes_every_search_class(emu_device)
