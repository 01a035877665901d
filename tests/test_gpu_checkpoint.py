"""Checkpoint and resume (sb_state_save / sb_state_load): N scans, save, load into another context, M scans must give the
bits of N + M scans without a break. After the load and after every following scan the resumed run is compared with the
uninterrupted one: current and last pose, the statistics (but the wall times), every surfel record in order, the seven
frames, the loop-closure info and edges, the submap origin."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api, synth
from helpers import assert_bits_equal, both_params, scans, sized, surfel_fields_equal
from test_gpu_lazy_map import scan_modes
from test_gpu_paging import pose_at, tile_surfels

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make(pp, loop=None):
    g = api.SurfelMapping(pp)
    if loop:
        g.enableLoopClosure(True, **loop)
    return g


def observe(g):
    """everything a getter returns (the map download compacts the map: both runs are observed at the same scans)"""
    st = np.zeros(16)
    api.lib().sb_get_statistics(g.ctx.h, api._dp(st))
    st[8:12] = 0.0  # wall times
    m = g.getMap()
    frames = [f.maps() for f in (g.getCurrentFrame(), g.getLastFrame(), g.getCurrentModelFrame(), g.getLastModelFrame(),
                                 m.oldMapFrame(), m.newMapFrame(), m.composedFrame())]
    return dict(pose=g.getCurrentPose(), last=g.getLastPose(), stats=st, t=g.timestamp(), mt=m.timestamp(),
                surfels=m.getAllSurfels(), frames=frames, info=g.getLoopInfo(), edges=g.getLoopEdges(),
                origin=m.submap_origin())


def same(a, b, what):
    assert a["t"] == b["t"] and a["mt"] == b["mt"], what + " timestamps"
    assert_bits_equal(a["pose"], b["pose"], what + " current pose")
    assert_bits_equal(a["last"], b["last"], what + " last pose")
    assert_bits_equal(a["stats"], b["stats"], what + " statistics")
    surfel_fields_equal(a["surfels"], b["surfels"], what + " surfels")
    for i, (fa, fb) in enumerate(zip(a["frames"], b["frames"])):
        for k in range(3):
            assert_bits_equal(fa[k], fb[k], "%s frame %d image %d" % (what, i, k))
    for k, v in a["info"].items():
        assert_bits_equal(np.asarray(v), np.asarray(b["info"][k]), "%s loop info %s" % (what, k))
    assert len(a["edges"]) == len(b["edges"]), what + " loop edges"
    for (f1, t1, r1), (f2, t2, r2) in zip(a["edges"], b["edges"]):
        assert (f1, t1) == (f2, t2), what + " loop edge"
        assert_bits_equal(r1, r2, what + " loop edge pose")
    assert a["origin"] == b["origin"], what + " submap origin / pending extractions"


def reference(pp, sc, first, loop=None, hook=None):
    """the uninterrupted run: obs[n] = observe() after n scans, for n >= first"""
    g = make(pp, loop)
    obs = {}
    try:
        for t, s in enumerate(sc):
            g.processScan(*s)
            if hook:
                hook(g, t)
            if t + 1 >= first:
                obs[t + 1] = observe(g)
    finally:
        g.ctx.close()
    return obs


def resume(pp, sc, blob, n_done, obs, what, target=None, hook=None):
    """load `blob` (taken after n_done scans) into `target` (a fresh context if None) and run the rest of `sc`"""
    g = target or make(pp)
    try:
        g.load_state(blob)
        if hook:
            hook(g, n_done - 1)
        same(observe(g), obs[n_done], what + " after the load")
        for t in range(n_done, len(sc)):
            g.processScan(*sc[t])
            if hook:
                hook(g, t)
            same(observe(g), obs[t + 1], "%s t=%d" % (what, t))
        return g.save_state()
    finally:
        g.ctx.close()


@pytest.mark.parametrize("width,semantic", [(900, False), (900, True), (2048, False), (2048, True)],
                         ids=["900", "900-semantic", "2048", "2048-semantic"])
def test_resume_is_bit_exact(width, semantic):
    """save at scan 6 with surfels removed in place (dead slots), destroy, load into a new context, 4 more scans; the
    saving context continues too (a save changes nothing); save(load(save(x))) == save(x)"""
    po, pp = both_params(**sized(width))
    sc, _ = scans(width, n=10, semantic=semantic)
    N = 6
    obs = reference(pp, sc, N)
    src = make(pp)
    src.ctx.profile(True)
    modes = []
    for s in sc[:N]:
        src.processScan(*s)
        modes.append(scan_modes(src)[0])
    src.ctx.profile(False)
    assert modes[-1] == "lazy", "the save must see dead slots: %r" % modes
    blob = src.save_state()
    n = C.c_uint64()
    assert api.lib().sb_state_size(src.ctx.h, C.byref(n)) == 0 and n.value == len(blob)
    for t in range(N, len(sc)):  # the saving context goes on as if nothing happened
        src.processScan(*sc[t])
        same(observe(src), obs[t + 1], "saving context t=%d" % t)
    src.ctx.close()
    g = make(pp)
    g.load_state(blob)
    assert g.save_state() == blob, "save(load(save(x))) != save(x)"
    g.ctx.close()
    resume(pp, sc, blob, N, obs, "resumed")
    if width == 900:  # and the resumed run against the oracle over N + M scans
        osl = O.Slam(po)
        g = make(pp)
        g.load_state(blob)
        for t, s in enumerate(sc):
            osl.process_scan(*s)
            if t >= N:
                g.processScan(*s)
                assert_bits_equal(g.getCurrentPose(), osl.pose(), "oracle t=%d pose" % t)
        surfel_fields_equal(g.getMap().getAllSurfels(), osl.map.download(), "oracle surfels")
        g.ctx.close()


def test_resume_right_after_a_dense_scan_into_a_used_context():
    """save after scan 1 (the first update is dense), load into a context that has mapped another sequence with other
    parameters: the checkpoint's parameters and state replace everything"""
    _, pp = both_params(**sized(900))
    sc, _ = scans(900, n=5)
    obs = reference(pp, sc, 1)
    src = make(pp)
    src.processScan(*sc[0])
    blob = src.save_state()
    src.ctx.close()
    _, other = both_params(**sized(900, icp_max_distance=1.0, partial_extraction=0))
    g = make(other, loop=dict(search_distance=3.0))
    for s in scans(900, n=3, semantic=True)[0]:
        g.processScan(*s)
    resume(pp, sc, blob, 1, obs, "into a used context", target=g)


def test_resume_through_a_track_loss_recovery():
    """save one scan before a pose jump: the resumed run's frame-to-frame recovery reads the restored last frame"""
    _, pp = both_params(**sized(900))
    scene = synth.Scene(width=900, height=64)
    poses = synth.trajectory(8)
    J = synth.translate(0.8, 0.3, 0) @ synth.rot_z(np.deg2rad(8.0))
    sc = [scene.scan(f, poses[f] if f < 4 else poses[f] @ J) for f in range(7)]
    obs = reference(pp, sc, 4)
    assert obs[7]["stats"][6] >= 1, "the sequence must trigger the recovery"
    assert obs[4]["stats"][6] == 0
    src = make(pp)
    for s in sc[:4]:
        src.processScan(*s)
    blob = src.save_state()
    src.ctx.close()
    resume(pp, sc, blob, 4, obs, "track loss")


def test_resume_loop_closure_with_pending_candidates_and_an_optimisation_request():
    """the synthetic loop of test_loop_closure_detection_and_verification_bit_exact: save while unverified candidates are
    pending, and again while optimisation_requested is raised; integrateLoopClosures (identity) follows at that scan"""
    _, pp = both_params(**sized(900))
    scene = synth.Scene(width=900, height=64)
    poses = synth.trajectory(124, step=0.2618, yaw_deg=3.0)
    sc = [scene.scan(f, poses[f]) for f in range(124)]
    lp = dict(search_distance=3.0, min_trajectory_distance=15.0, min_verifications=2)
    g = make(pp, lp)
    blobs = {}
    try:
        for t, s in enumerate(sc):
            g.processScan(*s)
            info = g.getLoopInfo()
            if "pending" not in blobs and info["unverified"] > 0:
                blobs["pending"] = (t + 1, g.save_state())
            if "request" not in blobs and info["optimisation_requested"]:
                blobs["request"] = (t + 1, g.save_state())
                break
    finally:
        g.ctx.close()
    assert set(blobs) == {"pending", "request"}, "the sequence must raise both: %r" % sorted(blobs)
    n_req = blobs["request"][0]
    last = min(n_req + 4, len(sc))
    sc = sc[:last]

    def integrate(g, t):
        if t + 1 == n_req:
            assert g.integrateLoopClosures() > 0

    obs = reference(pp, sc, blobs["pending"][0], loop=lp, hook=integrate)
    for name, (n, blob) in blobs.items():
        resume(pp, sc, blob, n, obs, "loop closure (%s)" % name, hook=integrate)


class _Paged:
    """operator-level map updates with frames that measure nothing (tests/test_gpu_paging.py): only paging moves surfels"""

    def __init__(self, pp, state=None):
        self.g = api.SurfelMapping(pp)
        self.m = self.g.getMap()
        self.f = api.Frame(self.g.ctx, 128, 16)
        if state is not None:
            self.g.load_state(state)

    def close(self):
        del self.f
        self.g.ctx.close()


def test_resume_paging_with_a_pending_extraction_and_before_a_reinsertion():
    """partial extraction pending and tiles in the HBM pool at the save; another save one update before a cached column
    comes back"""
    _, pp = both_params(**sized(128, 16))
    xs = [12, 12, 12, 32, 32, 12, -12, -12]
    up = np.concatenate([tile_surfels(3000, -4, k, 10 + k) for k in range(-4, 5)] +
                        [tile_surfels(2000, 0, 0, 30), tile_surfels(2500, 5, 1, 31)])
    ref = _Paged(pp)
    ref.m.upload(up, 1)
    blobs, obs = {}, {}
    for t, x in enumerate(xs):
        ref.m.update(pose_at(x), ref.f)
        if t == 1:
            i, j, pending = ref.m.submap_origin()
            assert pending > 0, "partial extraction must be pending"
            blobs[t] = ref.g.save_state()
        if t == 5:  # x = -12 next: origin 0 again, the cached column -4 comes back from the pool
            blobs[t] = ref.g.save_state()
        obs[t] = observe(ref.g)
    ref.close()
    for t0, blob in blobs.items():
        r = _Paged(pp, blob)
        try:
            same(observe(r.g), obs[t0], "paging t=%d after the load" % t0)
            for t in range(t0 + 1, len(xs)):
                r.m.update(pose_at(xs[t]), r.f)
                same(observe(r.g), obs[t], "paging from %d, t=%d" % (t0, t))
        finally:
            r.close()


def test_a_checkpoint_moves_to_another_process(tmp_path):
    """saved here, loaded in a spawned interpreter, which runs the rest of the sequence"""
    _, pp = both_params(**sized(900))
    sc, _ = scans(900, n=6, semantic=True)
    obs = reference(pp, sc, 3)
    src = make(pp)
    for s in sc[:3]:
        src.processScan(*s)
    path = tmp_path / "state.bin"
    src.save_state_file(str(path))
    src.ctx.close()
    out = tmp_path / "out.npz"
    code = (
        "import sys; sys.path[:0] = [%r, %r]\n"
        "import numpy as np\n"
        "from helpers import scans, sized\n"
        "from semantic_suma_b200 import api\n"
        "g = api.SurfelMapping(api.default_params(**sized(900)))\n"
        "g.load_state_file(%r)\n"
        "for s in scans(900, n=6, semantic=True)[0][3:]:\n"
        "    g.processScan(*s)\n"
        "np.savez(%r, pose=g.getCurrentPose(), surfels=g.getMap().getAllSurfels())\n"
    ) % (ROOT, os.path.join(ROOT, "tests"), str(path), str(out))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    got = np.load(out)
    assert_bits_equal(got["pose"], obs[6]["pose"], "spawned process pose")
    surfel_fields_equal(got["surfels"], obs[6]["surfels"], "spawned process surfels")


def _section(blob, sid):
    """payload offset of section `sid` (after the 280-byte header: u32 id, u32 0, u64 length, payload)"""
    off = 280
    while True:
        i, n = int(np.frombuffer(blob, np.uint32, 1, off)[0]), int(np.frombuffer(blob, np.uint64, 1, off + 8)[0])
        if i == sid:
            return off + 16
        off += 16 + n


def _tile_table(blob):
    """offset and rows (i, j, slot, known, base, count) of the tile table in section S_HOST, offset of tiles_pending"""
    n_ext = int(np.frombuffer(blob, np.uint32, 1, _section(blob, 1) + 952)[0])
    at = _section(blob, 1) + 956 + 8 * n_ext
    n = int(np.frombuffer(blob, np.uint32, 1, at)[0])
    return at + 4, np.frombuffer(blob, np.uint32, 6 * n, at + 4).reshape(-1, 6), at + 4 + 24 * n + 4


def _rc_load(g, blob):
    a = np.frombuffer(blob, np.uint8)
    rc = api.lib().sb_state_load(g.ctx.h, api._vp(a) if a.size else None, a.size)
    return rc, api.lib().sb_last_error(g.ctx.h).decode()


def test_bad_checkpoints_are_refused():
    """wrong magic / version, another image size, a truncated blob: SB_ERR_INVALID with a reason and the context goes on
    bit-exactly; one flipped payload byte: SB_ERR_INVALID and the context is reset; SB_ERR_STATE while a multi-GPU
    exchange is set up"""
    _, pp = both_params(**sized(900))
    sc, _ = scans(900, n=6)
    obs = reference(pp, sc, 3)
    src = make(pp)
    for s in sc[:3]:
        src.processScan(*s)
    blob = src.save_state()
    src.ctx.close()
    bad = bytearray(blob); bad[0] ^= 0xff
    ver = bytearray(blob); ver[8] += 1
    _, p2048 = both_params(**sized(2048))
    other = make(p2048)
    for s in scans(2048, n=1)[0]:
        other.processScan(*s)
    blob_2048 = other.save_state()
    other.ctx.close()
    g = make(pp)
    g.load_state(blob)
    for what, b, reason in [("magic", bytes(bad), "magic"), ("version", bytes(ver), "version"),
                            ("image size", blob_2048, "geometry"), ("truncated", blob[:len(blob) // 2], "truncated"),
                            ("empty", b"", "magic")]:
        rc, msg = _rc_load(g, b)
        assert rc == -1 and reason in msg, "%s: %d %r" % (what, rc, msg)
    # fields that size copies or index device memory are range-checked before the digest is even looked at
    for what, sid, off, reason in [("surfel count of the result block", 4, 8192, "result block"),
                                   ("pose-table reference", 1, 932, "pose-table")]:
        crafted = bytearray(blob)
        at = _section(blob, sid) + off
        crafted[at:at + 4] = np.uint32(0xfffffff0).tobytes()
        rc, msg = _rc_load(g, bytes(crafted))
        assert rc == -1 and reason in msg, "%s: %d %r" % (what, rc, msg)
    # the context continues as if the calls had not happened
    for t in range(3, 6):
        g.processScan(*sc[t])
        same(observe(g), obs[t + 1], "after refused loads t=%d" % t)
    # tile tables whose records read back are not those of the lowest slots, or whose pending flag disagrees with them
    _, ppp = both_params(**sized(128, 16))
    paged = _Paged(ppp)
    try:
        paged.m.upload(np.concatenate([tile_surfels(3000, -4, k, 10 + k) for k in range(-4, 5)]), 1)
        for x in (12, 12):  # two tiles of column -4 extracted (partial extraction), neither read back
            paged.m.update(pose_at(x), paged.f)
        pblob = paged.g.save_state()
        before = observe(paged.g)
        at, tiles, pending_at = _tile_table(pblob)
        assert (tiles[:, 3] == 0).all() and len(tiles) == 2 and np.frombuffer(pblob, np.uint32, 1, pending_at)[0] == 1
        rec = np.frombuffer(pblob, np.uint32, 2 * 2, _section(pblob, 5) + 4).reshape(-1, 2)
        k = int(np.argmax(tiles[:, 2]))  # the later extraction marked as read back, with its slot's exact range
        base = int(rec[tiles[k, 2] - 1, 0]) if tiles[k, 2] else 0
        not_prefix = bytearray(pblob)
        not_prefix[at + 24 * k + 12:at + 24 * k + 24] = np.array([1, base, rec[tiles[k, 2], 0] - base], np.uint32).tobytes()
        not_pending = bytearray(pblob)
        not_pending[pending_at:pending_at + 4] = np.uint32(0).tobytes()
        for what, b in [("a tile read back above one that is not", not_prefix), ("pending flag cleared", not_pending)]:
            rc, msg = _rc_load(paged.g, bytes(b))
            assert rc == -1 and "malformed tile table" in msg, "%s: %d %r" % (what, rc, msg)
        same(observe(paged.g), before, "after refused tile tables")
    finally:
        paged.close()
    # multi-GPU exchange set up: both calls refuse
    cb = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_int64))(lambda u, s: 0)
    assert api.lib().sb_comm_set_callback(g.ctx.h, C.cast(cb, C.c_void_p), None, 0, 64) == 0
    n = C.c_uint64()
    buf = np.zeros(16, np.uint8)
    assert api.lib().sb_state_size(g.ctx.h, C.byref(n)) == -5
    assert api.lib().sb_state_save(g.ctx.h, api._vp(buf), 16, C.byref(n)) == -5
    assert _rc_load(g, blob)[0] == -5
    assert api.lib().sb_comm_set_callback(g.ctx.h, None, None, 0, 0) == 0
    # a flipped byte in the surfel payload: refused after the bulk upload, the context is left reset
    flip = bytearray(blob)
    flip[len(blob) // 3] ^= 0x01
    rc, msg = _rc_load(g, bytes(flip))
    assert rc == -1 and "digest" in msg, msg
    assert g.timestamp() == 0 and g.getMap().size() == 0 and g.getMap().timestamp() == 0
    assert_bits_equal(g.getCurrentPose(), np.eye(4), "pose after a refused load")
    g.ctx.close()


def _compile_cpp(tmp_path):
    from semantic_suma_b200 import build as product_build
    api.lib()
    lib_dir = os.path.dirname(product_build.LIB)
    exe = os.path.join(str(tmp_path), "checkpoint_example")
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "checkpoint_example.cpp"), "-L" + lib_dir, "-lsuma_b200",
                           "-Wl,-rpath," + lib_dir])
    return exe


def test_cpp_mirror_file_overloads_match_the_python_mirror(tmp_path):
    """tests/cpp/checkpoint_example.cpp: 3 scans, saveState(file), loadState(file) in a new SurfelMapping, 2 scans"""
    exe = _compile_cpp(tmp_path)
    sc, _ = scans(900, n=5)
    path = os.path.join(str(tmp_path), "scans.bin")
    with open(path, "wb") as f:
        for pts, _, _ in sc:
            f.write(np.uint32(pts.shape[0]).tobytes())
            f.write(np.ascontiguousarray(pts, np.float32).tobytes())
    state = os.path.join(str(tmp_path), "state.bin")
    out = subprocess.check_output([exe, path, "900", "3", state], text=True)
    lines = {l.split()[0]: l.split()[1:] for l in out.strip().splitlines()}
    pp = api.default_params(**sized(900))
    g = make(pp)
    for pts, _, _ in sc[:3]:
        g.processScan(pts)
    # the same layout (the bytes differ in the wall-time statistics of each run, and so in the digest)
    assert len(g.save_state()) == os.path.getsize(state)
    g.ctx.close()
    g = make(pp)
    g.load_state_file(state)
    for pts, _, _ in sc[3:]:
        g.processScan(pts)
    assert_bits_equal(api.from_colmajor(np.array([float(x) for x in lines["pose"]])), g.getCurrentPose(), "C++ pose")
    assert int(lines["surfels"][0]) == g.getMap().size()
    assert lines["refused"] == ["1"]
    g.ctx.close()


def test_run_kitti_resume_writes_the_pose_file_of_an_uninterrupted_run(tmp_path):
    """run_kitti --save-state / --save-every, then --resume, on a --make-synthetic sequence: byte-identical pose files"""
    from semantic_suma_b200 import run_kitti
    seq = str(tmp_path / "seq")
    run_kitti.make_synthetic_sequence(seq, 10, width=900, semantic=True)
    whole, resumed, state = str(tmp_path / "whole.txt"), str(tmp_path / "resumed.txt"), str(tmp_path / "state.bin")
    common = [seq, "--width", "900", "--semantic"]
    assert run_kitti.main(common + ["--out", whole]) == 0
    assert run_kitti.main(common + ["--max-scans", "6", "--save-state", state, "--save-every", "4"]) == 0
    assert len(np.load(run_kitti.trajectory_path(state))) == 6
    assert run_kitti.main(common + ["--resume", state, "--out", resumed]) == 0
    assert open(resumed, "rb").read() == open(whole, "rb").read()
