import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on a machine with an H100)")


def load_emulated_library():
    """tests/emu: the product sources compiled for the CPU CUDA-emulator, bound exactly like libfuzzb200.so.
    Test infrastructure -- the product never loads it."""
    import ctypes
    import importlib.util

    from fuzzysearch_b200 import _native
    spec = importlib.util.spec_from_file_location("fzb_build_emu", os.path.join(ROOT, "tests", "emu", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lib = ctypes.CDLL(mod.build())
    for name, (res, args) in _native.SYMBOLS.items():
        f = getattr(lib, name)
        f.restype = res
        f.argtypes = args
    return lib


def pytest_sessionstart(session):
    # FZB_TEST_BACKEND=emu python -m pytest tests -m gpu : replay the GPU parity tests on the CPU emulator
    # (developer tool for boxes without a GPU; sizes that need a real GPU are skipped by the tests themselves)
    if os.environ.get("FZB_TEST_BACKEND") == "emu":
        from fuzzysearch_b200 import _native
        _native._lib = load_emulated_library()


def _cuda_available():
    try:
        from fuzzysearch_b200 import _native
        return _native.device_count() > 0
    except Exception:
        return False


def needs_real_gpu(what):
    """For the handful of gpu tests the CPU emulator cannot stand in for (FZB_TEST_BACKEND=emu replays): NCCL,
    CUDA IPC between processes, 4 GiB inputs."""
    if os.environ.get("FZB_TEST_BACKEND") == "emu":
        pytest.skip("needs a real GPU: " + what)


@pytest.fixture(scope="session")
def cuda_device():
    if not _cuda_available():
        pytest.fail("gpu-marked test ran without a usable CUDA device / libfuzzb200.so")
    return 0
