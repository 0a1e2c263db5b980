"""The route plans of api.cu replayed on the emulated build: the bodies of the -m gpu tests of
test_gpu_route_plan.py, on the CPU."""
import test_gpu_route_plan as G
from test_emu_kernels import emu_device, emu_lib  # noqa: F401  (fixtures)


def test_emu_one_refusal_for_every_caller(emu_device):
    G.test_one_refusal_for_the_single_search_its_batch_and_best_per_record(emu_device)


def test_emu_unbounded_total_limit(emu_device):
    G.test_unbounded_total_limit_runs_the_lowered_lp_route(emu_device)
