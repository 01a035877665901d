#!/usr/bin/env python
"""Cost of a long run's pose table: the bench.py workload (64x2048 hdl64_2048_geometric, synthetic, seed 1337) with the
map started at map timestamps 0, 1e4, 1e5 and 1e6 (sb_map_upload of an empty map at that timestamp: the pose table has
then grown to hold the entry of every scan, exactly as after that many scans).

For each start: --warmup scans, then --steps timed scans (wall clock around each sb_process_scan, which ends in a device
synchronisation), then the same number of scans again with the per-kernel profiler on: device ms per scan (sum of all
kernels), the time in pose_products and in the two Gauss-Newton launches (which fill the product tables at their end),
the window [begin, end) of the product tables and the bytes of the four pose tables. Separately, the stall of each
doubling of the table (sb_map_set_pose at the current capacity, host clock around the call). Prints one JSON line with
the device it ran on.

    python posetablebench.py [--steps 60] [--warmup 60]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

STARTS = (0, 10_000, 100_000, 1_000_000)


def run_start(api, np, pp, scans, start, warmup, steps):
    s = api.SurfelMapping(pp)
    if start:
        s.getMap().upload(np.zeros(0, api.SURFEL_DTYPE), start)
    it = iter(scans)
    for _ in range(warmup):
        s.processScan(next(it)[0])
    wall = []
    for _ in range(steps):
        p = next(it)[0]
        t0 = time.perf_counter()
        s.processScan(p)
        wall.append(time.perf_counter() - t0)
    s.ctx.profile(True)
    for _ in range(steps):
        s.processScan(next(it)[0])
    prof = s.ctx.profile_collect()
    s.ctx.profile(False)
    info = s.getMap().pose_table_info()
    dev_ms = sum(ms for ms, _ in prof.values())
    rec = {
        "start": start,
        "wall_ms_per_scan_median": round(statistics.median(wall) * 1e3, 4),
        "wall_ms_per_scan_mean": round(statistics.mean(wall) * 1e3, 4),
        "device_ms_per_scan": round(dev_ms / steps, 4),
        "pose_products_us_per_scan": round(prof.get("pose_products", (0.0, 0))[0] / steps * 1e3, 3),
        "gauss_newton_us_per_scan": round((prof.get("icp_fused", (0.0, 0))[0] + prof.get("icp_post", (0.0, 0))[0])
                                          / steps * 1e3, 3),
        "pose_table": info,
        "table_bytes": 4 * info["capacity"] * 64,
    }
    s.ctx.close()
    return rec


def doubling_stalls(api, np, pp):
    ctx = api.Context(pp)
    m = api.SurfelMap(ctx)
    pose = np.eye(4, dtype=np.float32)
    out = []
    cap = m.pose_table_info()["capacity"]
    while cap < (1 << 24):
        t0 = time.perf_counter()
        m.set_pose(cap, pose)
        ctx.synchronize()
        dt = time.perf_counter() - t0
        new = m.pose_table_info()["capacity"]
        out.append({"from": cap, "to": new, "ms": round(dt * 1e3, 3)})
        cap = new
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=60)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    import numpy as np

    import bench
    from gnbench import device_info
    from semantic_suma_b200 import api

    if api.lib().sb_device_count() <= 0:
        raise SystemExit("posetablebench: no CUDA device")
    w = bench.WORKLOADS["hdl64_2048_geometric"]
    n = args.warmup + 2 * args.steps
    scans = bench.generate_scans(w, n, seed=1337)
    pp = api.default_params(**bench.param_kwargs(w))
    runs = [run_start(api, np, pp, scans, k, args.warmup, args.steps) for k in STARTS]
    # the starts once more in reverse order: the spread between the two passes is the run-to-run noise
    again = [run_start(api, np, pp, scans, k, args.warmup, args.steps) for k in reversed(STARTS)]
    print(json.dumps({"bench": "posetablebench", "workload": "hdl64_2048_geometric", "warmup": args.warmup,
                      "steps": args.steps, "device": device_info(args.device), "runs": runs,
                      "runs_reversed": again, "doublings": doubling_stalls(api, np, pp)}))


if __name__ == "__main__":
    main()
