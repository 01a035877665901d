"""The cheapest designed map-update case of tests/test_gpu_update_edges.py on the CPU executor for the CUDA sources, in
the default CPU tier: k_index_scatter, k_radius, k_update_surfels and k_gen_compact against the oracle and the exact
model at the thresholds of the radius map and the generation pass."""
from test_cusim import _child


def test_radius_threshold_case_on_the_cpu_executor():
    assert _child(["tests/test_gpu_update_edges.py"], "test_update_case and radius_threshold and 16x96") == 1
