"""The ring geometry of k_filter_sampled replayed on the emulated build: the bodies of the -m gpu tests of
test_gpu_sampled_scan.py, with one pass of the emulated grid (4 CTAs) in place of the H100's."""
import test_gpu_sampled_scan as G
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)


def test_emu_sampled_scan_lengths(emu_device):
    G.test_buffer_lengths_around_stages_and_the_grid_pass(emu_device, small=True)


def test_emu_sampled_scan_edges(emu_device):
    G.test_pattern_with_nul_bytes_against_the_zero_padding(emu_device, small=True)
    G.test_shards_at_offsets(emu_device, small=True)
    G.test_exact_search_windows(emu_device, small=True)
    G.test_tiny_work_list_overflows_into_bitmap_mode(emu_device, small=True)
