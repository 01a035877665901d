#!/usr/bin/env python
"""Wall time of a checkpoint (sb_state_save / sb_state_load) of the bench.py map.

The map is the steady state bench.py measures at: 64x2048 hdl64_2048_geometric, seed 1337, its 60 + 20 pre-roll scans
(the sensor has moved far enough by then to page submap tiles out into the HBM tile pool). Then --repeat saves into one
preallocated (pageable) host buffer and as many loads of it into a second context; medians are reported with the bytes
and GB/s. Beside them: the pinned host<->device copy bandwidth measured in the same run with torch (256 MiB, CUDA
events), the ceiling of a copy that crosses PCIe, and the rate of one host thread copying the checkpoint's bytes out of a
pinned buffer into the pageable one, which every save and load also does. Prints one JSON line with the device it ran on.

    python checkpointbench.py [--repeat 5]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def pinned_gbps(torch, device, nbytes=256 << 20, reps=5):
    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device=device)
    out = {}
    for name, dst, src in (("h2d", d, h), ("d2h", h, d)):
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dst.copy_(src, non_blocking=True)
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e-3)
        out[name] = round(nbytes / statistics.median(ts) / 1e9, 2)
    return out


def host_copy_gbps(torch, dst, chunk=16 << 20, reps=3):
    """one host thread copying len(dst) bytes out of a pinned buffer in `chunk`-sized pieces (what a save does between
    the pinned double buffer and the caller's memory)"""
    import numpy as np
    src = torch.empty(chunk, dtype=torch.uint8, pin_memory=True).numpy()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for o in range(0, dst.size, chunk):
            n = min(chunk, dst.size - o)
            np.copyto(dst[o:o + n], src[:n])
        ts.append(time.perf_counter() - t0)
    return round(dst.size / statistics.median(ts) / 1e9, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    import numpy as np
    import torch

    import bench
    from gnbench import device_info
    from semantic_suma_b200 import api

    w = bench.WORKLOADS["hdl64_2048_geometric"]
    pre = 60 + 20
    scans = bench.generate_scans(w, pre, seed=1337)
    pp = api.default_params(**bench.param_kwargs(w))
    src = api.SurfelMapping(pp, device=args.device)
    for p, _, _ in scans:
        src.processScan(p)
    src.ctx.synchronize()
    L = api.lib()
    n = C.c_uint64()
    src.ctx.check(L.sb_state_size(src.ctx.h, C.byref(n)), "state_size")
    buf = np.empty(n.value, np.uint8)
    buf[:] = 0  # pages touched before the first timed save
    written = C.c_uint64()
    saves, loads = [], []
    dst = api.SurfelMapping(pp, device=args.device)
    for _ in range(args.repeat + 1):  # the first round allocates the pinned staging of both contexts: not timed
        t0 = time.perf_counter()
        src.ctx.check(L.sb_state_save(src.ctx.h, api._vp(buf), n.value, C.byref(written)), "state_save")
        t1 = time.perf_counter()
        dst.ctx.check(L.sb_state_load(dst.ctx.h, api._vp(buf), written.value), "state_load")
        t2 = time.perf_counter()
        saves.append(t1 - t0)
        loads.append(t2 - t1)
    saves, loads = saves[1:], loads[1:]
    nbytes = int(written.value)
    surfels = int(src.getMap().size())
    ts, tl = statistics.median(saves), statistics.median(loads)
    out = {"metric": "checkpoint_save_load_s", "unit": "s",
           "save": {"median_s": round(ts, 4), "min_s": round(min(saves), 4), "gb_per_s": round(nbytes / ts / 1e9, 2)},
           "load": {"median_s": round(tl, 4), "min_s": round(min(loads), 4), "gb_per_s": round(nbytes / tl / 1e9, 2)},
           "bytes": nbytes, "surfels": surfels, "surfel_bytes": 64 * surfels,
           "pinned_copy_gb_per_s": pinned_gbps(torch, args.device), "host_copy_gb_per_s": host_copy_gbps(torch, buf),
           "repeat": args.repeat,
           "config": {"workload": "hdl64_2048_geometric", "range_image": "%dx%d" % (w["height"], w["width"]),
                      "map_preroll_scans": pre},
           "device": device_info(args.device)}
    dst.ctx.close()
    src.ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
