"""The Python layers' own paths replayed on the emulated build: the bodies of the -m gpu tests of
test_gpu_python_layers.py at the sizes the CPU emulator takes."""
import test_gpu_python_layers as G
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)


def test_emu_align_in_each_without_a_common_alphabet(emu_device):
    G.test_align_in_each_without_a_common_alphabet(emu_device, small=True)


def test_emu_anchored_nearest_patterns_without_a_common_alphabet(emu_device):
    for anchor in ("start", "end"):
        G.test_anchored_nearest_patterns_without_a_common_alphabet(emu_device, anchor, small=True)


def test_emu_row_checks_and_pattern_packing(emu_device):
    G.test_align_in_each_row_checks(emu_device)
    G.test_pattern_packing_at_its_empty_edges(emu_device)
