"""The in-place map update's cheapest parity case (tests/test_gpu_lazy_map.py) on the CPU executor for the CUDA sources,
in the default CPU tier: pipeline scans that leave dead slots, then render, the operator-level update with its index map,
and a download, each against the oracle."""
from test_cusim import _child


def test_operators_on_a_map_with_dead_slots_on_the_cpu_executor():
    assert _child(["tests/test_gpu_lazy_map.py"], "operators_on_a_map_with_dead_slots") == 1
