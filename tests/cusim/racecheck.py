"""TEST INFRASTRUCTURE: racecheck of the kernels -- the CPU executor built with ThreadSanitizer (CUSIM_TSAN=1: every CUDA
thread is a TSan fiber, fiber switches order nothing, barriers / warp collectives / atomics / volatile hand-overs do), a
short semantic run with the in-kernel exchange in loop-back, and the list of report sites. Known, by design:

  emit_fragment / k_render_scatter / k_index_scatter (+ atomicMin)   a plain, possibly stale read of a depth key that only ever
                                                                      decreases, ahead of the atomicMin on it
  k_update_surfels                                                    many surfels store the same 1 into one "integrated" flag

Anything else fails. usage: python tests/cusim/racecheck.py [scans=3] [width=450]   (re-executes itself under libtsan)"""
import glob
import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
KNOWN = ("emit_fragment", "k_render_scatter", "k_index_scatter", "atomicMin", "k_update_surfels")


def child(n_scans, width):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.dirname(HERE))
    import ctypes as C
    import numpy as np
    from cusim import build_sim
    path = build_sim.build()
    from semantic_suma_b200 import build as product_build
    product_build.LIB = path
    product_build.build = lambda *a, **k: path
    from semantic_suma_b200 import api, synth
    pp = api.default_params(data_width=width, model_width=width, max_iterations=4, stopping_threshold=0.0, delta=0.0)
    sl = api.SurfelMapping(pp)
    h = np.zeros(64, np.uint8)
    L = api.lib()
    sl.ctx.check(L.sb_comm_export(sl.ctx.h, C.c_void_p(h.ctypes.data)), "export")
    sl.ctx.check(L.sb_comm_init(sl.ctx.h, 0, 1, C.c_void_p(h.ctypes.data), 0, pp.data_height), "init")
    scene = synth.Scene(width=width, height=64, semantic=True)
    poses = synth.trajectory(n_scans)
    for t in range(n_scans):
        sl.processScan(*scene.scan(t, poses[t]))
    print("racecheck run: %d scans, %d surfels" % (n_scans, sl.getMap().size()))
    sl.ctx.close()


def selftest():
    """the tool itself: a missing __syncthreads / __syncwarp is reported, a present one is not"""
    os.environ["CUSIM_TSAN"] = "1"
    sys.path.insert(0, os.path.dirname(HERE))
    from cusim import build_sim
    so = build_sim.build()
    bdir = os.path.dirname(so)
    exe = os.path.join(bdir, "selftest_race")
    flags = [f for f in build_sim.CXXFLAGS if f != "-fPIC"]
    subprocess.check_call(["g++"] + flags + ["-I", HERE, os.path.join(HERE, "selftest_race.cpp"), os.path.join(bdir, "cusim_rt.o"),
                                             "-fsanitize=thread", "-pthread", "-o", exe])
    res = {0: set(), 1: set(), 2: set()}
    # a dynamic detector with a finite history (256 thread slots recycled among thousands of fibers): a report is a fact, one
    # silent run is not -- the seeded races get three attempts, the clean kernels must stay silent in all of them
    for attempt in range(3):
        for which in (0, 1, 2):
            r = subprocess.run([exe, str(which)], capture_output=True, text=True, timeout=300,
                               env=dict(os.environ, TSAN_OPTIONS="exitcode=0:halt_on_error=0:report_signal_unsafe=0:history_size=7"))
            if "FATAL: ThreadSanitizer" in r.stderr:  # e.g. an address-space layout this libtsan cannot map
                print("ThreadSanitizer does not start here: " + r.stderr.strip().splitlines()[0])
                sys.exit(77)
            assert "selftest ran" in r.stdout, r.stdout + r.stderr
            res[which] |= set(re.findall(r"SUMMARY: ThreadSanitizer: data race \S+ in (\w+)", r.stderr))
        if res[1] == {"k_block"} and res[2] == {"k_warp"}:
            break
    res = {k: sorted(v) for k, v in res.items()}
    print("selftest: barriers present -> %r; no __syncthreads -> %r; no __syncwarp -> %r" % (res[0], res[1], res[2]))
    assert res[0] == [] and res[1] == ["k_block"] and res[2] == ["k_warp"], res


def main():
    if "--selftest" in sys.argv:
        return selftest()
    n_scans = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    width = int(sys.argv[2]) if len(sys.argv) > 2 else 450
    if os.environ.get("CUSIM_RACECHECK_CHILD") == "1":
        return child(n_scans, width)
    libtsan = subprocess.check_output(["gcc", "-print-file-name=libtsan.so"], text=True).strip()
    with tempfile.TemporaryDirectory() as d:
        env = dict(os.environ, CUSIM_TSAN="1", CUSIM_RACECHECK_CHILD="1", LD_PRELOAD=libtsan,
                   TSAN_OPTIONS="report_signal_unsafe=0:halt_on_error=0:history_size=7:exitcode=0:log_path=%s/tsan:suppressions=%s"
                   % (d, os.path.join(HERE, "tsan.supp")))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), str(n_scans), str(width)], env=env, capture_output=True,
                           text=True, timeout=1500)
        if "FATAL: ThreadSanitizer" in r.stderr:
            print("ThreadSanitizer does not start here: " + r.stderr.strip().splitlines()[0])
            sys.exit(77)
        assert r.returncode == 0 and "racecheck run:" in r.stdout, (r.stdout + r.stderr)[-3000:]
        sites = {}
        for f in glob.glob(os.path.join(d, "tsan.*")):
            for m in re.finditer(r"SUMMARY: ThreadSanitizer: (.*?) (\S+:\d+) in (.*)", open(f).read()):
                sites[(m.group(2).replace(ROOT + "/", ""), m.group(3).split("(")[0])] = m.group(1)
    unknown = {k: v for k, v in sites.items() if not any(name in k[1] for name in KNOWN)}
    print(r.stdout.strip())
    for (loc, fn), kind in sorted(sites.items()):
        print("  %-9s %-48s %s%s" % (kind, loc, fn[:70], "" if (loc, fn) not in unknown else "   <-- NOT KNOWN"))
    assert not unknown, "racecheck: unexpected reports"
    print("racecheck ok: %d report sites, all of the known by-design kind" % len(sites))


if __name__ == "__main__":
    main()
