#!/usr/bin/env python
"""Cost of per-point deskewing (sb_set_deskew; DESIGN.md section 11) on the bench.py sequence.

The bench workload (64x2048 hdl64_2048_geometric, seed 1337) runs --scans scans in contexts with deskewing off and with
azimuth deskewing on, alternating off / on for --rounds rounds so that clock and thermal drift fall on both alike. Per
run: scans/s over the timed scans (every processScan ends in a device synchronisation). A separate profiled pass of each
mode reports K1a's (k_project_scatter) device time per launch from the per-kernel profiler, so that the profiler's
events stay out of the timed runs. Prints one JSON line with the device, its power limit and SM clock.

    python deskewbench.py [--scans 200] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def run(api, pp, scans, device, mode, profile=False):
    g = api.SurfelMapping(pp, device=device)
    g.setDeskew(mode)
    g.ctx.profile(profile)
    g.processScan(scans[0][0])  # first scan outside the timed region (identity motion: nothing to deskew)
    t0 = time.perf_counter()
    for p, _, _ in scans[1:]:
        g.processScan(p)
    dt = time.perf_counter() - t0
    out = {"scans_per_s": (len(scans) - 1) / dt, "pose": g.getCurrentPose()}
    if profile:
        out["kernels"] = g.ctx.profile_collect()
    g.ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import bench
    from gnbench import device_info
    from semantic_suma_b200 import api

    w = bench.WORKLOADS["hdl64_2048_geometric"]
    scans = bench.generate_scans(w, args.scans, seed=1337)
    pp = api.default_params(**bench.param_kwargs(w))
    run(api, pp, scans[:5], args.device, "off")  # module load, first launches
    rates = {"off": [], "azimuth": []}
    for _ in range(args.rounds):
        for mode in ("off", "azimuth"):
            rates[mode].append(run(api, pp, scans, args.device, mode)["scans_per_s"])
    k1a = {}
    for mode in ("off", "azimuth"):
        ms, launches = run(api, pp, scans, args.device, mode, profile=True)["kernels"].get("project_scatter", (0.0, 0))
        k1a[mode] = {"launches": launches, "us_per_launch": round(1e3 * ms / launches, 3) if launches else None}
    out = {"metric": "deskew_cost", "scans": args.scans, "points_per_scan": int(statistics.mean(len(s[0]) for s in scans)),
           "k1a_us": k1a,
           "k1a_added_us": (round(k1a["azimuth"]["us_per_launch"] - k1a["off"]["us_per_launch"], 3)
                            if k1a["off"]["us_per_launch"] and k1a["azimuth"]["us_per_launch"] else None),
           "scans_per_s": {m: {"median": round(statistics.median(v), 1), "min": round(min(v), 1), "max": round(max(v), 1),
                               "runs": [round(x, 1) for x in v]} for m, v in rates.items()},
           "config": {"workload": "hdl64_2048_geometric", "deskew": "azimuth (defaults: ref 0.5, a0 +pi, clockwise)"},
           "device": device_info(args.device)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
