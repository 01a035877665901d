#!/usr/bin/env python
"""Phase budget of the surfel rendering pass (k_render_scatter) on the bench.py workload.

An instrumented copy of the library is built in a temporary directory (never the product build): csrc/ is copied,
sb_map.cu gets %globaltimer stamps that thread 0 of every block of k_render_scatter takes at the phase boundaries, and
the block sums each phase into a device counter per instance. The stamps sit behind the block's barriers, so a
barrier-closed phase includes the block's slowest thread; the raster phases and the large quads are those of warp 0.

    --variant time   mean µs per block of each phase, per instance
    --variant count  what the phases work on, per launch: surfels through stage A/B, small quads with pixels, large
                     quads, box pixels tested, covered small-quad fragments queued, atomicMin issued (depth and index keys)

The counting build adds atomics and is never timed. The sequence is renderbench.py's: the bench's pre-roll
(60 + 20 scans of hdl64_2048_geometric, seed 1337), then --scans measured scans. --csrc budgets another version of the
sources (the instrumentation anchors on code that k_render_scatter has kept across versions). Prints one JSON line.

    python renderphases.py --variant time [--scans 30] [--csrc DIR]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

PRE = r'''
__device__ unsigned long long sbx_ph[2][16];
__device__ unsigned long long sbx_cnt[2][16];
__device__ int sbx_inst;
__device__ __forceinline__ unsigned long long sbx_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void sbx_count(int i, unsigned long long v) { atomicAdd(&sbx_cnt[sbx_inst][i], v); }
// ts: 0 entry, 1 stage A/B done, 2 packed, 3 stage C done, 4 prefix done, 5 / 6 phase 1 / 2 sums, 7 scratch,
// 8 warp 0's raster done, 9 warp 0's large quads done
__device__ void sbx_block_end(int inst, const unsigned long long* ts, bool early) {
  unsigned long long* p = sbx_ph[inst];
  const unsigned long long now = sbx_now();
  atomicAdd(p + 0, ts[1] - ts[0]);
  atomicAdd(p + 11, now - ts[0]);
  atomicAdd(p + 12, 1ull);
  if (early) {
    atomicAdd(p + 13, 1ull);
    return;
  }
  atomicAdd(p + 1, ts[2] - ts[1]);
  atomicAdd(p + 2, ts[3] - ts[2]);
  atomicAdd(p + 3, ts[4] - ts[3]);
  atomicAdd(p + 4, ts[5]);
  atomicAdd(p + 5, ts[6]);
  atomicAdd(p + 6, ts[8] - ts[4]);
  atomicAdd(p + 7, ts[9] - ts[8]);
  atomicAdd(p + 8, now - ts[9]);
}
#ifdef SBX_COUNT
#define atomicMin(p, v) (sbx_count(7, 1ull), ::atomicMin(p, v))
#define SBX_C(...) __VA_ARGS__
#else
#define SBX_C(...)
#endif
'''

POST = r'''
extern "C" int sbx_take(unsigned long long* ph, unsigned long long* cnt) {
  static const unsigned long long zero[2][16] = {};
  if (cudaMemcpyFromSymbol(ph, sb::sbx_ph, sizeof(zero)) != cudaSuccess) return 1;
  if (cudaMemcpyFromSymbol(cnt, sb::sbx_cnt, sizeof(zero)) != cudaSuccess) return 1;
  if (cudaMemcpyToSymbol(sb::sbx_ph, zero, sizeof(zero)) != cudaSuccess) return 1;
  if (cudaMemcpyToSymbol(sb::sbx_cnt, zero, sizeof(zero)) != cudaSuccess) return 1;
  return cudaDeviceSynchronize() == cudaSuccess ? 0 : 1;
}
'''

# (anchor, replacement): each anchor must occur exactly once in sb_map.cu
EDITS = [
    ("namespace sb {\nusing namespace sbm;\n", "namespace sb {\nusing namespace sbm;\n" + PRE),
    ("  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;\n",
     "  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;\n"
     "  __shared__ unsigned long long sbx_ts[10];\n"
     "  SBX_C(if (tid == 0) sbx_inst = kIndex ? 1 : 0; __syncthreads();)\n"
     "  if (tid == 0) { sbx_ts[0] = sbx_now(); sbx_ts[5] = 0; sbx_ts[6] = 0; }\n"),
    ("  if (lane == 0) s_warp_cnt[warp] = __popc(ballot);\n  __syncthreads();\n",
     "  if (lane == 0) s_warp_cnt[warp] = __popc(ballot);\n  __syncthreads();\n"
     "  if (tid == 0) sbx_ts[1] = sbx_now();\n"),
    ("  if (total == 0) return;\n",
     "  if (total == 0) {\n    if (tid == 0) sbx_block_end(kIndex ? 1 : 0, sbx_ts, true);\n    return;\n  }\n"),
    ("  __syncthreads();\n  // ---- stage C on dense lanes",
     "  __syncthreads();\n  if (tid == 0) sbx_ts[2] = sbx_now();\n  // ---- stage C on dense lanes"),
    ("          npix = (ni + 1) * (nj + 1);\n", "          npix = (ni + 1) * (nj + 1);\n          SBX_C(sbx_count(3, 1ull);)\n"),
    ("  __syncthreads();  // everybody is done with s_warp_cnt (read above) before it is reused\n",
     "  __syncthreads();  // everybody is done with s_warp_cnt (read above) before it is reused\n"
     "  if (tid == 0) sbx_ts[3] = sbx_now();\n"),
    ("  if (tid == 0) Q.prefix[0] = 0;\n  __syncthreads();\n",
     "  if (tid == 0) Q.prefix[0] = 0;\n  __syncthreads();\n  if (tid == 0) sbx_ts[4] = sbx_now();\n"
     "  SBX_C(if (tid == 0) { sbx_count(0, 1ull); sbx_count(1, (unsigned long long)total); sbx_count(4, s_nbig); "
     "sbx_count(5, (unsigned long long)T); })\n"),
    ("      int qn = 0;  // queue length, warp-uniform\n",
     "      int qn = 0;  // queue length, warp-uniform\n      if (tid == 0) sbx_ts[7] = sbx_now();\n"),
    ("          qn += __popc(bm);\n", "          qn += __popc(bm);\n          SBX_C(if (lane == 0) sbx_count(6, __popc(bm));)\n"),
    ("      __syncwarp();\n      // phase 2\n",
     "      __syncwarp();\n      if (tid == 0) { const unsigned long long n = sbx_now(); sbx_ts[5] += n - sbx_ts[7]; "
     "sbx_ts[7] = n; }\n      // phase 2\n"),
    ("      __syncwarp();\n    }\n  }\n  // ---- large quads: one warp each ----\n",
     "      __syncwarp();\n      if (tid == 0) sbx_ts[6] += sbx_now() - sbx_ts[7];\n    }\n  }\n"
     "  if (tid == 0) sbx_ts[8] = sbx_now();\n  // ---- large quads: one warp each ----\n"),
    ("  }\n}\n\nvoid launch_render_scatter(",
     "  }\n  if (tid == 0) sbx_ts[9] = sbx_now();\n  __syncthreads();\n"
     "  if (tid == 0) sbx_block_end(kIndex ? 1 : 0, sbx_ts, false);\n}\n#ifdef SBX_COUNT\n#undef atomicMin\n#endif\n\n"
     "void launch_render_scatter("),
]

PHASES = ["lane loads + stage A/B", "dense packing", "stage C + warp scan", "pixel-count prefix",
          "raster phase 1 (warp 0, all rounds)", "raster phase 2 (warp 0, all rounds)",
          "raster incl. binary search (warp 0)", "large quads (warp 0)", "wait for the block's other warps"]
COUNTS = ["blocks with survivors", "stage A/B survivors", "-", "small quads with pixels", "large quads", "box pixels tested",
          "covered small-quad fragments", "atomicMin issued"]  # sbx_cnt slots (2 unused)
INSTANCES = ["post_update", "post_icp"]  # kIndex = 0 / 1


def instrument(src):
    for anchor, repl in EDITS:
        n = src.count(anchor)
        if n != 1:
            raise RuntimeError("instrumentation anchor found %d times: %r" % (n, anchor[:60]))
        src = src.replace(anchor, repl)
    return src + POST


def build_lib(csrc, tmp, count):
    from semantic_suma_b200 import build as B
    d = os.path.join(tmp, "semantic_suma_b200", "csrc")  # the sources include ../../include/suma_b200.h
    shutil.copytree(csrc, d)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
    p = os.path.join(d, "sb_map.cu")
    with open(p) as f:
        src = f.read()
    with open(p, "w") as f:
        f.write(instrument(src))
    nvcc = B.nvcc_path()
    flags = B.NVCC_FLAGS + (["-DSBX_COUNT"] if count else [])
    procs, objs = [], []
    for s in B.SOURCES:
        o = os.path.join(tmp, s.replace(".cu", ".o"))
        procs.append(subprocess.Popen([nvcc] + flags + ["-c", "-o", o, os.path.join(d, s)], stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT))
        objs.append(o)
    for s, pr in zip(B.SOURCES, procs):
        out, _ = pr.communicate()
        if pr.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (s, out.decode()))
    lib = os.path.join(tmp, "libsuma_b200.so")
    subprocess.check_call([nvcc, "-shared", "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib]
                          + objs)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", choices=["time", "count"], default="time")
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--csrc", default=os.path.join(ROOT, "semantic_suma_b200", "csrc"))
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--build-only", action="store_true", help="build the instrumented library and stop")
    args = ap.parse_args()
    import ctypes as C

    tmp = tempfile.mkdtemp(prefix="renderphases_")
    try:
        lib_path = build_lib(os.path.abspath(args.csrc), tmp, args.variant == "count")
        if args.build_only:
            print(json.dumps({"built": True, "variant": args.variant}))
            return
        import bench
        from gnbench import device_info
        from semantic_suma_b200 import api
        from semantic_suma_b200 import build as B
        B.LIB = lib_path  # the instrumented copy, not the product library
        L = api.lib(build_if_missing=False)
        L.sbx_take.argtypes = [C.c_void_p, C.c_void_p]
        ph = np.zeros((2, 16), np.uint64)
        cnt = np.zeros((2, 16), np.uint64)

        def take():
            if L.sbx_take(ph.ctypes.data, cnt.ctypes.data) != 0:
                raise RuntimeError("sbx_take failed")

        w = bench.WORKLOADS["hdl64_2048_geometric"]
        pre = 60 + 20
        scans = bench.generate_scans(w, pre + args.scans, seed=1337)
        pp = api.default_params(**bench.param_kwargs(w))
        slam = api.SurfelMapping(pp, device=args.device)
        ctx = slam.ctx
        for p, _, _ in scans[:pre]:
            slam.processScan(p)
        ctx.synchronize()
        take()
        ctx.profile(True)
        for p, _, _ in scans[pre:]:
            slam.processScan(p)
        prof = ctx.profile_collect()
        ctx.profile(False)
        take()
        out = {"metric": "render_scatter_phase_budget", "variant": args.variant, "scans": args.scans,
               "csrc": os.path.relpath(os.path.abspath(args.csrc), ROOT)}
        for i, name in enumerate(INSTANCES):
            if args.variant == "time":
                blocks = int(ph[i, 12])
                full = blocks - int(ph[i, 13])
                rec = {"blocks_per_launch": round(blocks / args.scans, 1),
                       "blocks_without_survivors": round(int(ph[i, 13]) / args.scans, 1),
                       "block_us_mean": round(float(ph[i, 11]) / blocks / 1e3, 3)}
                rec["phases_us_mean_per_block"] = {
                    PHASES[j]: round(float(ph[i, j]) / (blocks if j == 0 else full) / 1e3, 3) for j in range(9)}
            else:
                rec = {"per_launch": {COUNTS[j]: round(int(cnt[i, j]) / args.scans, 1) for j in range(8)
                                      if COUNTS[j] != "-"}}
            out[name] = rec
        ms, c = prof["render_scatter"]
        out["render_scatter_us_per_launch_instrumented"] = round(1e3 * ms / c, 2)
        out["surfels"] = int(slam.getMap().size())
        out["device"] = device_info(args.device)
        ctx.close()
        print(json.dumps(out))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
