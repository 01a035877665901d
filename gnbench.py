#!/usr/bin/env python
"""Launch-time benchmark of the persistent Gauss-Newton kernel (k_gn_persistent) on the bench.py workload.

bench.py measures whole scans; here the two Gauss-Newton launches of a scan are taken apart:

* pipeline: the per-scan `icp_fused` (GN_MAIN: 10 iterations + pose bookkeeping + product table) and `icp_post`
  (GN_POST: statistics pass + pose chaining + product table) launch times, medians over --scans scans after the bench's
  pre-roll (60 + 20 scans of the hdl64_2048_geometric sequence, seed 1337);
* minimize: LieGaussNewton.minimize (sb_icp_minimize, GN_PLAIN) on one frame pair of that sequence with
  max_iterations = 1, 2, 5, 10, 20 and epsilon = delta = 0, so that every launch runs all its iterations. A least-squares
  line through the median launch times gives the time of one iteration (slope) and the fixed cost of a launch
  (intercept).

Times are CUDA events around each launch (the library's profiler). Prints one JSON line with the device it ran on.

    python gnbench.py [--scans 40] [--reps 50]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

ITERATIONS = (1, 2, 5, 10, 20)


def device_info(index):
    """name, power limit and SM clocks of the device, read now (the numbers below are only worth something with them)"""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split("\n")[0]
        f = [x.strip() for x in out.split(",")]
        return {"gpu": f[0], "power_limit_w": float(f[1]), "sm_mhz": float(f[2]), "sm_max_mhz": float(f[3])}
    except Exception as e:  # noqa: BLE001 -- the timings stand; say why the device record is missing
        return {"gpu": None, "error": "%s: %s" % (type(e).__name__, str(e)[:200])}


def launch_us(ctx, call, kernel):
    """device time of the one `kernel` launch that call() makes, in microseconds"""
    ctx.synchronize()
    ctx.profile(True)
    call()
    prof = ctx.profile_collect()
    ctx.profile(False)
    ms, cnt = prof[kernel]
    assert cnt == 1, (kernel, cnt)
    return 1e3 * ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=40, help="profiled pipeline scans after the pre-roll (>= 30)")
    ap.add_argument("--reps", type=int, default=50, help="minimize launches per iteration count")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    import bench
    from semantic_suma_b200 import api

    w = bench.WORKLOADS["hdl64_2048_geometric"]
    pre = 60 + 20  # bench.py's --preroll default + the --warmup of its measuring command
    scans = bench.generate_scans(w, pre + args.scans, seed=1337)
    pp = api.default_params(**bench.param_kwargs(w))
    slam = api.SurfelMapping(pp, device=args.device)
    ctx = slam.ctx
    for p, _, _ in scans[:pre]:
        slam.processScan(p)
    ctx.synchronize()

    per_scan = {"icp_fused": [], "icp_post": []}
    for p, _, _ in scans[pre:]:
        ctx.synchronize()
        ctx.profile(True)
        slam.processScan(p)
        prof = ctx.profile_collect()
        ctx.profile(False)
        for k in per_scan:
            ms, cnt = prof[k]
            per_scan[k].append(1e3 * ms / cnt)
    pipeline = {k: {"median_us": round(statistics.median(v), 2), "min_us": round(min(v), 2), "max_us": round(max(v), 2)}
                for k, v in per_scan.items()}

    # the frame pair: the last scan's data frame against the model rendered at its pose
    obj = api.Frame2Model(ctx)
    obj.setData(slam.getCurrentFrame(), slam.getCurrentModelFrame())
    gn = api.LieGaussNewton(ctx)
    gn.epsilon = gn.delta = 0.0
    medians = {}
    for n in ITERATIONS:
        gn.maxIter = n
        gn.minimize(obj, np.eye(4))  # warm-up
        t = [launch_us(ctx, lambda: gn.minimize(obj, np.eye(4)), "icp_fused") for _ in range(args.reps)]
        assert gn.iterationCount() == n, (n, gn.iterationCount())
        medians[n] = statistics.median(t)
    x = np.array(ITERATIONS, np.float64)
    y = np.array([medians[n] for n in ITERATIONS])
    slope, intercept = np.polyfit(x, y, 1)
    resid = y - (slope * x + intercept)

    out = {"metric": "gn_us_per_iteration", "value": round(float(slope), 3), "unit": "us",
           "fixed_us_per_launch": round(float(intercept), 2), "fit_max_residual_us": round(float(np.abs(resid).max()), 2),
           "minimize_median_us": {str(n): round(medians[n], 2) for n in ITERATIONS},
           "pipeline": pipeline, "pipeline_scans": args.scans, "reps": args.reps,
           "config": {"workload": "hdl64_2048_geometric", "range_image": "%dx%d" % (w["height"], w["width"]),
                      "map_preroll_scans": pre, "surfels": int(slam.getMap().size())},
           "device": device_info(args.device)}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
