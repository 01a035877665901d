#!/usr/bin/env python
"""Launch-time benchmark of the surfel rendering pass (k_render_scatter) on the bench.py workload.

Every scan of the per-scan pipeline renders the map twice at the same pose, with two instances of the kernel:

* post-ICP (`k_render_scatter<4, true>`): the model frame at the new pose, and the map update's index keys;
* post-update (`k_render_scatter<4, false>`): the model frame of the updated map that the next scan registers against.

The library's CUDA-event profiler sums both under one name (`render_scatter`), so the instances are taken apart with a
`torch.profiler` trace of --scans scans after the bench's pre-roll (60 + 20 scans of the hdl64_2048_geometric sequence,
seed 1337), and the medians of the per-launch device times are reported. The CUDA-event average over the
same number of scans, taken in a separate pass without the tracer, is reported beside them. Prints one JSON line with the
device it ran on.

    python renderbench.py [--scans 30]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

INSTANCES = {"post_icp": "k_render_scatter<4, true>", "post_update": "k_render_scatter<4, false>"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=30,
                    help="scans per measuring pass after the pre-roll (two passes: 30 cover bench.py's 60 timed steps)")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from gnbench import device_info
    from semantic_suma_b200 import api

    w = bench.WORKLOADS["hdl64_2048_geometric"]
    pre = 60 + 20  # bench.py's --preroll default + the --warmup of its measuring command
    scans = bench.generate_scans(w, pre + 2 * args.scans, seed=1337)
    pp = api.default_params(**bench.param_kwargs(w))
    slam = api.SurfelMapping(pp, device=args.device)
    ctx = slam.ctx
    for p, _, _ in scans[:pre]:
        slam.processScan(p)
    ctx.synchronize()
    torch.cuda.synchronize(args.device)  # the CUDA runtime of the tracer is up before the traced window

    # pass 1: the library's CUDA events, both instances together
    ctx.profile(True)
    for p, _, _ in scans[pre:pre + args.scans]:
        slam.processScan(p)
    prof = ctx.profile_collect()
    ctx.profile(False)
    ms, cnt = prof["render_scatter"]
    events = {"avg_us_per_launch": round(1e3 * ms / cnt, 2), "launches_per_scan": round(cnt / args.scans, 2)}

    # pass 2: per-launch device times of each instance from a kernel trace
    times = {k: [] for k in INSTANCES}
    with profile(activities=[ProfilerActivity.CUDA]) as tr:
        for p, _, _ in scans[pre + args.scans:]:
            slam.processScan(p)
        ctx.synchronize()
    for e in tr.events():
        for k, sig in INSTANCES.items():
            if sig in e.name:
                times[k].append(e.time_range.elapsed_us())
    per_instance = {}
    for k, v in times.items():
        if not v:
            raise RuntimeError("no %s launch in the trace" % INSTANCES[k])
        per_instance[k] = {"kernel": INSTANCES[k], "median_us": round(statistics.median(v), 2),
                           "min_us": round(min(v), 2), "max_us": round(max(v), 2), "launches": len(v)}

    out = {"metric": "render_scatter_us_per_launch", "unit": "us",
           "value": round(statistics.median(times["post_icp"] + times["post_update"]), 2),
           "instances": per_instance, "cuda_events": events, "scans_per_pass": args.scans,
           "config": {"workload": "hdl64_2048_geometric", "range_image": "%dx%d" % (w["height"], w["width"]),
                      "map_preroll_scans": pre, "surfels": int(slam.getMap().size())},
           "device": device_info(args.device)}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
