"""The library's CUDA sources, executed on the CPU (tests/cusim: one fiber per CUDA thread, one OS thread per block, warp
collectives and barriers as rendezvous points), against the oracle -- the `-m gpu` parity tests themselves, run in a child
pytest with the test-side switch --cusim. This is a check of the kernels' LOGIC in a container without a GPU (every branch
the parity suite reaches, bit for bit); it is not a GPU run and says nothing about speed. The product never loads the
executor: the swap is done by tests/conftest.py only."""
import os
import re
import subprocess
import sys

import pytest

FULL = os.environ.get("SUMA_B200_CUSIM_FULL") == "1"
long_run = pytest.mark.skipif(not FULL, reason="kept out of the default CPU tier for its run time: SUMA_B200_CUSIM_FULL=1")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _child(files, k, env=None, timeout=1500):
    e = dict(os.environ)
    e.pop("SUMA_B200_TEST_CUSIM", None)
    e.update(env or {})
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "--cusim", "-p", "no:cacheprovider", "-k", k] + files
    r = subprocess.run(cmd, cwd=ROOT, env=e, capture_output=True, text=True, timeout=timeout)
    tail = (r.stdout + r.stderr)[-4000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m, tail
    assert " skipped" not in r.stdout.splitlines()[-1], tail  # every selected test really ran on the executor
    return int(m.group(1))


def test_launch_rewrite_is_mechanical():
    from cusim import build_sim
    src = "  {\n    ScopedKernel sk(L, K);\n    k_foo<4><<<grid, kThreads, 0, L.stream>>>(kp, s,\n        n_dev);\n  }\n"
    out, n = build_sim.rewrite_launches(src, "x")
    assert n == 1
    assert 'cusim::launch("k_foo<4>", cusim::cfg(grid, kThreads, 0, L.stream), [&] { k_foo<4>(kp, s,\n        n_dev); });' in out
    out, n = build_sim.rewrite_asm('  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));\n', "x")
    assert n == 1 and "t = cusim::globaltimer();" in out


def test_cuda_sources_on_the_cpu_executor_equal_the_oracle():
    """preprocessing, Jacobian sums, Gauss-Newton (persistent kernel), map update / rendering, whole processScan runs at
    64x900 (geometric and semantic; 64x2048 and 128x4096 in the full run), track-loss fallback, submap paging, the in-kernel peer exchange in loop-back,
    the 24 parameter variants, the 6 image geometries and the reference-generated digests"""
    n = _child(["tests/test_gpu_parity.py", "tests/test_zz_gpu_late.py", "tests/test_golden.py"],
               "not loop_closure and not ouster and not 2048")  # the 2048-wide cases: SUMA_B200_CUSIM_FULL=1 (whole suite)
    assert n >= 28


def test_map_update_on_an_image_under_256_pixels():
    """three updates of a 3.6 M-surfel map with a 16x8 frame: all 256 group totals of the update pass are cleared, not only
    the first P (tests/test_gpu_shapes.py)"""
    assert _child(["tests/test_gpu_shapes.py"], "test_map_updates_on_an_image_under_256_pixels") == 1


def test_render_edges_on_the_cpu_executor():
    """the render pass at the switch points of its fast paths (small / large quads, corner span, azimuth seam, degenerate
    and crossed quads, the tie rule, depth ties, z clip, block loads, a 65536-wide model image) against the exact reference
    rasteriser and the oracle, and the refusal of model sides over 65536 (tests/test_gpu_render_edges.py)"""
    assert _child(["tests/test_gpu_render_edges.py"], "test_") == 15


def test_submap_paging_on_the_cpu_executor():
    """several tiles extracted per update, a tile over the 500 000-surfel extract cap and paging an empty map, each against
    the oracle (tests/test_gpu_paging.py; the pool exhaustion case runs in the full tier)"""
    assert _child(["tests/test_gpu_paging.py"], "not exhaustion") == 3


@long_run
def test_kernel_results_do_not_depend_on_the_execution_order():
    """CUDA promises no order between the lanes of a warp or the warps of a block outside its synchronisation primitives:
    the same bits with the lanes / warps run in reverse and in a shuffled order (this is how the unsynchronised pivot search
    of the warp-parallel LDLT was found)"""
    k = "pipeline_bit_exact and 900 or icp_minimize or map_update_and_render_bit_exact_semantic or track_loss or fused_peer"
    order = os.environ.get("SUMA_B200_CUSIM_ORDER", "random:3")  # also: reverse, random:<seed>
    assert _child(["tests/test_gpu_parity.py"], k, env={"CUSIM_ORDER": order}) >= 6


@long_run
def test_persistent_kernel_with_a_gpu_sized_grid():
    """the executor's default device has 4 SMs (8 cooperative blocks); with 64 SMs the persistent Gauss-Newton kernel runs 128
    co-resident blocks and its shared-memory pixel cache engages at 64x900, as on an H100"""
    k = "pipeline_bit_exact and 900 and False or icp_minimize or track_loss or fused_peer"
    assert _child(["tests/test_gpu_parity.py"], k, env={"CUSIM_SMS": "64"}) >= 4


@pytest.mark.parametrize("ranks,extra", [(2, ["900", "64", "5", "jump"]), pytest.param(4, ["900", "64", "5", "jump"], marks=long_run),
                                         pytest.param(8, ["900", "64", "5", "jump"], marks=long_run)])
def test_in_kernel_peer_exchange_on_n_ranks(ranks, extra):
    """SURVEY.md 8e on 2 / 4 / 8 "GPUs" of the executor (one host thread and one context per rank, mailboxes exchanged through
    sb_comm_export / sb_comm_init): every rank holds the bits of the un-striped run after every scan; every case drives
    a 1.5 m jump through the striped track-loss recovery. (Real GPUs: tests/test_gpu_multi.py, 2 ranks.)"""
    r = subprocess.run([sys.executable, os.path.join(HERE, "cusim", "multirank_check.py"), str(ranks)] + extra, cwd=ROOT,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "multirank ok: %d ranks" % ranks in r.stdout, (r.stdout + r.stderr)[-3000:]


def test_racecheck_of_the_kernels():
    """the executor built with ThreadSanitizer (CUDA threads = TSan fibers; only barriers, warp collectives, atomics and
    volatile hand-overs order anything): first the tool on two toy kernels -- a missing __syncthreads / __syncwarp is reported,
    a present one is not --, then a semantic run with the in-kernel exchange: only the two known by-design report kinds
    (tests/cusim/racecheck.py)"""
    for args in (["--selftest"], ["2"]):
        r = subprocess.run([sys.executable, os.path.join(HERE, "cusim", "racecheck.py")] + args, cwd=ROOT, capture_output=True,
                           text=True, timeout=1500)
        if r.returncode == 77:
            pytest.skip(r.stdout.strip()[-200:])
        assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert "racecheck ok" in r.stdout, r.stdout[-2000:]


def test_a_missing_peer_ends_in_an_error_not_a_hang():
    """two ranks set up for the in-kernel exchange, only one runs: its persistent kernel gives up after the bounded spin, the
    scan returns SB_ERR_STATE, the contexts close (tests/cusim/peer_timeout_check.py)"""
    r = subprocess.run([sys.executable, os.path.join(HERE, "cusim", "peer_timeout_check.py")], cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "peer timeout ok" in r.stdout and "contexts closed" in r.stdout, (r.stdout + r.stderr)[-3000:]


def test_bench_native_arm_dry_run():
    """bench.py's own Python path at N = 1 (pre-roll, device-resident pass, end-to-end pass with input staging, per-kernel pass,
    CPU baseline, the JSON line with every key of the contract) with the CUDA sources on the executor and torch's CUDA calls
    stubbed: the line is complete. Its numbers mean nothing."""
    r = subprocess.run([sys.executable, os.path.join(HERE, "cusim", "bench_dryrun.py"), "--steps", "3", "--warmup", "3", "--preroll", "2",
                        "--cpu-budget", "1", "--workload", "hdl64_900_geometric"], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "bench dry run ok" in r.stdout, (r.stdout + r.stderr)[-3000:]


@long_run
def test_the_whole_gpu_suite_on_the_cpu_executor():
    """everything `-m gpu` selects that does not need real devices: also 128x4096 / 15 iterations and the two 120-scan
    loop-closure runs (about four minutes on 8 cores)"""
    assert _child(["tests/"], "not cusim", timeout=3000) >= 38
