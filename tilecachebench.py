#!/usr/bin/env python
"""Cost of the managed submap tile cache (sb_set_tile_cache) on the bench.py sequence.

The bench workload (64x2048 hdl64_2048_geometric, seed 1337) runs --scans scans twice: once with the default cache, once
in a managed context whose pool is shrunk to --pool surfels with an unbounded host tier, so that reclaims and evictions
recur. With --submap-extent below the default of 10 m, tiles leave every few scans. Per run: the wall time of every
processScan (it ends in a device synchronisation), median and worst; for the managed run also the k_pool_reclaim
launches from the per-kernel profiler (a separate pass, so that the profiler's events stay out of the step times), the
surfels they moved and their rate against the 3.35 TB/s HBM3 bound (read + write), and the cache's counters. The poses
of both runs must agree bit for bit. Prints one JSON line with the device it ran on.

    python tilecachebench.py [--scans 200] [--pool 500000] [--submap-extent 4]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def run(api, pp, scans, device, pool=None, profile=False):
    g = api.SurfelMapping(pp, device=device)
    if pool:
        g.setTileCache(pool, None)
    g.ctx.profile(profile)
    times, poses = [], []
    for p, _, _ in scans:
        t0 = time.perf_counter()
        g.processScan(p)
        times.append(time.perf_counter() - t0)
        poses.append(g.getCurrentPose())
    out = {"times": times, "poses": poses, "info": g.tile_cache_info() if pool else None}
    if profile:
        out["kernels"] = g.ctx.profile_collect()
    g.ctx.close()
    return out


def step_stats(times):
    return {"median_ms": round(1e3 * statistics.median(times), 3), "worst_ms": round(1e3 * max(times), 3),
            "mean_ms": round(1e3 * statistics.mean(times), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--pool", type=int, default=500_000)
    ap.add_argument("--submap-extent", type=float, default=4.0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    import numpy as np

    import bench
    from gnbench import device_info
    from semantic_suma_b200 import api

    w = bench.WORKLOADS["hdl64_2048_geometric"]
    scans = bench.generate_scans(w, args.scans, seed=1337)
    kw = bench.param_kwargs(w)
    kw["submap_extent"] = args.submap_extent
    pp = api.default_params(**kw)
    run(api, pp, scans[:5], args.device)  # module load, first launches
    default = run(api, pp, scans, args.device)
    managed = run(api, pp, scans, args.device, pool=args.pool)
    same = all(np.array_equal(a, b) for a, b in zip(default["poses"], managed["poses"]))
    prof = run(api, pp, scans, args.device, pool=args.pool, profile=True)
    ms, launches = prof["kernels"].get("pool_reclaim", (0.0, 0))
    moved = prof["info"]["reclaim_moved"]
    out = {"metric": "tile_cache_step_ms", "unit": "ms", "scans": args.scans, "poses_bit_identical": bool(same),
           "default": step_stats(default["times"]), "managed": step_stats(managed["times"]),
           "managed_cache": managed["info"],
           "pool_reclaim": {"launches": launches, "total_ms": round(ms, 4),
                            "us_per_launch": round(1e3 * ms / launches, 2) if launches else None,
                            "surfels_moved": moved, "bytes_read_written": 4 * 64 * moved,
                            "share_of_hbm_bound": (round(4 * 64 * moved / HBM_BYTES_PER_S / (ms * 1e-3), 3)
                                                   if ms else None)},
           "config": {"workload": "hdl64_2048_geometric", "pool_surfels": args.pool, "host_surfels": "unbounded",
                      "submap_extent": args.submap_extent},
           "device": device_info(args.device)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
