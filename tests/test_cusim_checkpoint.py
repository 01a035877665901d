"""Checkpoint and resume (tests/test_gpu_checkpoint.py) on the CPU executor for the CUDA sources, in the default CPU tier:
the ordered gather of a map with dead slots, the scatter back, the digest on both sides, and paging state across a load."""
from test_cusim import _child


def test_checkpoint_resume_on_the_cpu_executor():
    assert _child(["tests/test_gpu_checkpoint.py"], "resume_is_bit_exact and 900 and not semantic or resume_paging") == 2


def test_cpp_checkpoint_example_compiles_without_gpu(tmp_path):
    """tests/cpp/checkpoint_example.cpp against -Iinclude -lsuma_b200"""
    from test_gpu_checkpoint import _compile_cpp
    _compile_cpp(tmp_path)
