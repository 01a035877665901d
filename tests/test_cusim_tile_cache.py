"""The managed tile cache (tests/test_gpu_tile_cache.py) on the CPU executor for the CUDA sources, in the default CPU tier:
reclaim in a small pool, the cut when both tiers are full, and the argument and state checks of sb_set_tile_cache."""
from test_cusim import _child


def test_tile_cache_on_the_cpu_executor():
    assert _child(["tests/test_gpu_tile_cache.py"], "reclaim_in_a_small_pool or both_tiers_full or set_tile_cache_arguments") == 3
