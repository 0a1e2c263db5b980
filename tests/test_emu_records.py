"""Record sets (fzb_haystack_set_records) and find_near_matches_in_each replayed on the emulated build: the bodies of
the -m gpu tests of test_gpu_records.py at the sizes the CPU emulator takes."""
import test_gpu_records as G
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)


def test_emu_records_every_route(emu_device):
    for case in G.ROUTES:
        G.route_case(case, small=True)


def test_emu_records_edges_and_refusals(emu_device):
    G.test_granule_edges_and_separators(emu_device, small=True)
    G.test_pattern_holding_the_separator_byte(emu_device, small=True)
    G.test_refusals_leave_the_handle_usable(emu_device)


def test_emu_records_golden_and_public_api(emu_device):
    G.test_golden_records_over_a_set(emu_device, stride=7)
    G.test_public_api_kinds(emu_device)
    G.test_threads_share_one_set(emu_device, n_threads=2)
