"""The small cases of test_gpu_nearest_limits.py replayed on the emulated build: the windowed restatement against the
whole-text restatement and the scans, and 65 535 patterns over a dozen records and a short sequence."""
import test_gpu_nearest_limits as G
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)


def test_emu_windowed_restatement(emu_device):
    G.test_windowed_restatement(emu_device)


def test_emu_65535_patterns(emu_device):
    G.test_65535_patterns(emu_device, small=True)
