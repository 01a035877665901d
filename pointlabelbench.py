#!/usr/bin/env python
"""Cost of the per-point label records (sb_set_point_labels / sb_get_point_labels; DESIGN.md section 13), and what they
say about the map's labels.

On the bench.py sequences (seed 1337) at 64x2048 (hdl64_2048_semantic) and 128x4096 (ouster128_4096_geometric):
  * k_point_labels' device time per launch, from the per-kernel profiler in a separate profiled run with the mode on;
  * end-to-end scans/s with the mode off and on, alternating off / on for --rounds rounds so that clock and thermal
    drift fall on both alike (every processScan ends in a device synchronisation; the records are not copied out);
  * sb_get_point_labels of the last scan's records into pinned host memory and into pageable numpy memory (each call
    ends in a synchronisation), median over --copies calls.
Label quality (--quality-scans, 64x2048 semantic synthetic sequence with 2 % label flips): over the points that won
their pixel and have a map label, how often the map's label equals the label before the flips, against how often the
input label does; the same over the flipped points alone. Prints one JSON line with the device, its power limit and SM
clock, read in the same call.

    python pointlabelbench.py [--scans 200] [--rounds 3] [--copies 50] [--quality-scans 40]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = {"64x2048": "hdl64_2048_semantic", "128x4096": "ouster128_4096_geometric"}


def run(api, pp, scans, device, on, profile=False):
    g = api.SurfelMapping(pp, device=device)
    g.setPointLabels(on)
    g.ctx.profile(profile)
    g.processScan(*scans[0])  # first scan outside the timed region
    t0 = time.perf_counter()
    for s in scans[1:]:
        g.processScan(*s)
    dt = time.perf_counter() - t0
    out = {"scans_per_s": (len(scans) - 1) / dt, "pose": g.getCurrentPose()}
    if profile:
        out["kernels"] = g.ctx.profile_collect()
    return g, out


def copy_cost(api, g, copies):
    """median wall time of sb_get_point_labels into pinned and into pageable host memory (us)"""
    import torch
    n = C.c_uint32(0)
    L = api.lib()
    L.sb_get_point_labels(g.ctx.h, None, 0, C.byref(n), 0)
    pinned = torch.empty(n.value * 32, dtype=torch.uint8).pin_memory()
    pageable = np.empty(n.value, api.POINT_LABEL_DTYPE)
    out = {"records": n.value, "bytes": 32 * n.value}
    for name, ptr in (("pinned", pinned.data_ptr()), ("pageable", pageable.ctypes.data)):
        ts = []
        for _ in range(copies + 3):
            t0 = time.perf_counter()
            rc = L.sb_get_point_labels(g.ctx.h, C.c_void_p(ptr), n.value, C.byref(n), 0)
            ts.append(time.perf_counter() - t0)
            assert rc == 0
        med = statistics.median(ts[3:])
        out[name] = {"us": round(1e6 * med, 1), "GB_per_s": round(32 * n.value / med / 1e9, 2)}
    assert pinned.numpy().tobytes() == pageable.tobytes()
    return out


def quality(api, n_scans, device):
    from semantic_suma_b200 import synth
    sc = synth.Scene(width=2048, height=64, semantic=True)
    poses = synth.trajectory(n_scans)
    g = api.SurfelMapping(api.default_params(data_width=2048, model_width=2048), device=device)
    g.setPointLabels(True)
    tot = dict(mapped=0, map_ok=0, input_ok=0, flipped=0, flipped_map_ok=0)
    for f in range(n_scans):
        pts, lab, prb, clean = sc.scan(f, poses[f], clean_labels=True)
        g.processScan(pts, lab, prb)
        r = g.getPointLabels()
        m = ((r["flags"] & api.POINT_WON) != 0) & ((r["flags"] & api.POINT_MAP) != 0)
        fl = m & (lab != clean)
        tot["mapped"] += int(m.sum())
        tot["map_ok"] += int((r["map_label"][m] == clean[m]).sum())
        tot["input_ok"] += int((lab[m] == clean[m]).sum())
        tot["flipped"] += int(fl.sum())
        tot["flipped_map_ok"] += int((r["map_label"][fl] == clean[fl]).sum())
    g.ctx.close()
    return {"scans": n_scans, "won_and_mapped_points": tot["mapped"],
            "map_label_equals_clean": round(tot["map_ok"] / tot["mapped"], 4),
            "input_label_equals_clean": round(tot["input_ok"] / tot["mapped"], 4),
            "flipped_points": tot["flipped"],
            "map_label_equals_clean_on_flipped": round(tot["flipped_map_ok"] / max(tot["flipped"], 1), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--copies", type=int, default=50)
    ap.add_argument("--quality-scans", type=int, default=40)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import bench
    from gnbench import device_info
    from semantic_suma_b200 import api

    res = {}
    for size, wname in WORKLOADS.items():
        w = bench.WORKLOADS[wname]
        scans = bench.generate_scans(w, args.scans, seed=1337)
        pp = api.default_params(**bench.param_kwargs(w))
        run(api, pp, scans[:5], args.device, False)[0].ctx.close()  # module load, first launches
        rates = {"off": [], "on": []}
        for _ in range(args.rounds):
            for mode in ("off", "on"):
                g, o = run(api, pp, scans, args.device, mode == "on")
                rates[mode].append(o["scans_per_s"])
                g.ctx.close()
        g, o = run(api, pp, scans, args.device, True, profile=True)
        ms, launches = o["kernels"].get("point_labels", (0.0, 0))
        copy = copy_cost(api, g, args.copies)
        g.ctx.close()
        med = {m: statistics.median(v) for m, v in rates.items()}
        res[size] = {"workload": wname, "points_per_scan": int(statistics.mean(len(s[0]) for s in scans)),
                     "kernel": {"launches": launches, "us_per_launch": round(1e3 * ms / launches, 3) if launches else None},
                     "scans_per_s": {m: {"median": round(med[m], 1), "min": round(min(v), 1), "max": round(max(v), 1),
                                         "runs": [round(x, 1) for x in v]} for m, v in rates.items()},
                     "us_per_scan_added": round(1e6 / med["on"] - 1e6 / med["off"], 1),
                     "get_point_labels": copy}
    out = {"metric": "point_label_cost", "scans": args.scans, "sizes": res,
           "quality": quality(api, args.quality_scans, args.device) if args.quality_scans else None,
           "device": device_info(args.device)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
