"""Per-point deskewing (sb_set_deskew, sb_process_scan_timed, sb_preprocess_deskew; DESIGN.md section 11) against the
oracle bit for bit: the operator at three image shapes, whole rolling-shutter runs in both modes (with paging, loop
closure and a checkpoint in between), zero motion giving the bits of deskewing off, and the refusals."""
import struct

import numpy as np
import pytest

from oracle import deskew as OD
from oracle import oracle as O
from semantic_suma_b200 import api, synth
from helpers import assert_bits_equal, both_params, sized, surfel_fields_equal

pytestmark = pytest.mark.gpu
MODES = {1: "times", 2: "azimuth"}
# the turning sequence of the rolling-shutter runs: 1.2 m and 3 deg per sweep
STEP, YAW = 1.2, 3.0
INC = synth.translate(STEP, 0, 0) @ synth.rot_z(np.deg2rad(YAW))
_seq = {}


def rolling_scans(width, height=64, n=4, semantic=False):
    key = (width, height, n, semantic)
    if key not in _seq:
        sc = synth.Scene(width=width, height=height, semantic=semantic)
        poses = synth.trajectory(n, step=STEP, yaw_deg=YAW)
        _seq[key] = [sc.scan(f, poses[f], rolling=INC) for f in range(n)]
    return _seq[key]


def random_motion(rng, deg=30.0, m=3.0):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    T = np.eye(4)
    T[:3, :3] = synth.so3_exp(np.deg2rad(rng.uniform(-deg, deg)) * axis)
    T[:3, 3] = rng.uniform(-m, m, 3)
    return T


def gpu_preprocess(ctx, p, pts, labels, probs, **kw):
    f = api.Frame(ctx, p.data_width, p.data_height)
    api.Preprocessing(ctx).process(pts, f, labels, probs, **kw)
    return f.maps()


def assert_frames(a, b, what):
    for k, name in enumerate(("vertex", "normal", "semantic")):
        assert_bits_equal(a[k], b[k], "%s %s" % (what, name))


# ---- the operator ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(900, 64), (2048, 64), (333, 37)], ids=["64x900", "64x2048", "37x333"])
@pytest.mark.parametrize("semantic", [False, True], ids=["geometric", "semantic"])
def test_preprocess_deskew_equals_the_oracle(shape, semantic):
    W, H = shape
    po, pp = both_params(**sized(W, H))
    ctx = api.Context(pp)
    rng = np.random.default_rng(W + H + semantic)
    pts, lab, prb, s = rolling_scans(W, H, n=2, semantic=semantic)[1]
    times = s.copy()
    times[::97] = np.nan
    times[1::89] = 1.7
    times[2::83] = -0.4
    times[3::79] = np.inf
    for mode in (1, 2):
        for cw in (True, False):
            M = random_motion(rng)
            d = dict(mode=mode, ref_time=float(rng.uniform(0, 1)), start_azimuth=float(rng.uniform(-4, 4)), clockwise=cw)
            t = times if mode == 1 else None
            g = gpu_preprocess(ctx, pp, pts, lab, prb, times=t, deskew=d, motion=M, timestamp=12)
            o = OD.preprocess_deskew(po, pts, lab, prb, times=t, timestamp=12, motion=M, **d)
            assert_frames(g, o, "mode %d clockwise %s" % (mode, cw))
            plain = O.preprocess(po, pts, lab, prb, timestamp=12)
            assert not np.array_equal(plain[0], o[0])  # the motion did move points
    ctx.close()


def test_zero_motion_passes_the_bits_through():
    """times all s_ref, an identity motion, and seam points with y = -0 (atan2 puts them in column 0, +0 in W-1)"""
    po, pp = both_params(**sized(900))
    ctx = api.Context(pp)
    pts, lab, prb, s = rolling_scans(900, n=2, semantic=True)[1]
    seam = np.array([[-10.0, -0.0, -1.0, 1.0], [-12.0, 0.0, -1.5, 1.0], [-0.0, -0.0, -2.0, 1.0]], np.float32)
    pts = np.concatenate([seam, pts])
    lab = np.concatenate([np.full(3, 40.0, np.float32), lab])
    prb = np.concatenate([np.full(3, 0.9, np.float32), prb])
    s = np.concatenate([np.zeros(3, np.float32), s])
    plain = gpu_preprocess(ctx, pp, pts, lab, prb)
    assert_frames(plain, O.preprocess(po, pts, lab, prb), "plain")
    M = random_motion(np.random.default_rng(3))
    same = [
        dict(times=np.full(len(pts), 0.25, np.float32), deskew=dict(mode=1, ref_time=0.25), motion=M),
        dict(times=s, deskew=dict(mode=1), motion=np.eye(4)),
        dict(deskew=dict(mode=2), motion=np.eye(4)),
        dict(deskew=dict(mode=2), motion=None),
    ]
    for k, kw in enumerate(same):
        assert_frames(gpu_preprocess(ctx, pp, pts, lab, prb, **kw), plain, "zero motion case %d" % k)
    d = OD.deskew_points(pts, np.full(len(pts), 0.25, np.float32), mode=1, ref_time=0.25, motion=M)
    assert d[:3].tobytes() == pts[:3].tobytes()  # -0 stays -0
    ctx.close()


# ---- whole runs ------------------------------------------------------------------------------------------------------
def run_pair(width, semantic, mode, n=4, setup=None, **kw):
    po, pp = both_params(**sized(width, **kw))
    g, o = api.SurfelMapping(pp), OD.Slam(po)
    g.setDeskew(MODES[mode])
    o.set_deskew(mode)
    if setup:
        setup(o, g)
    for f, (pts, lab, prb, s) in enumerate(rolling_scans(width, n=n, semantic=semantic)):
        t = s if mode == 1 else None
        g.processScan(pts, lab, prb, times=t)
        o.process_scan(pts, lab, prb, times=t)
        check_pair(g, o, "scan %d" % f)
    return g, o


def check_pair(g, o, what):
    assert_bits_equal(g.getCurrentPose(), o.pose(), what + " pose")
    assert g.getStatistics()["num_iterations"] == o.stats()["iterations"], what + " iterations"
    surfel_fields_equal(g.getMap().getAllSurfels(), o.map.download(), what + " surfels")


@pytest.mark.parametrize("mode", [1, 2], ids=["times", "azimuth"])
@pytest.mark.parametrize("semantic", [False, True], ids=["geometric", "semantic"])
@pytest.mark.parametrize("width", [900, 2048])
def test_rolling_shutter_run_equals_the_oracle(width, semantic, mode):
    g, _ = run_pair(width, semantic, mode)
    g.ctx.close()


def test_rolling_shutter_run_with_paging():
    g, _ = run_pair(900, False, 2, n=8, submap_extent=3.0, submap_dimension=1)
    assert g.getMap().submap_origin()[:2] != (0, 0)  # the window has moved: tiles were paged
    g.ctx.close()


def test_rolling_shutter_run_with_loop_closure():
    lp = dict(search_distance=3.0, min_trajectory_distance=15.0, min_verifications=2)

    def setup(o, g):
        o.enable_loop_closure(**lp)
        g.enableLoopClosure(True, **lp)

    g, _ = run_pair(900, False, 1, n=4, setup=setup)
    g.ctx.close()


def test_checkpoint_resume_keeps_deskewing():
    """N scans, save, load into a fresh context, M more scans == N + M straight; the setting travels with the blob"""
    _, pp = both_params(**sized(900))
    seq = rolling_scans(900, n=5, semantic=True)
    straight = api.SurfelMapping(pp)
    straight.setDeskew("times", ref_time=0.4)
    first = api.SurfelMapping(pp)
    first.setDeskew("times", ref_time=0.4)
    for f in range(2):
        for m in (straight, first):
            m.processScan(*seq[f][:3], times=seq[f][3])
    blob = first.save_state()
    resumed = api.SurfelMapping(pp)
    resumed.load_state(blob)
    assert resumed.getDeskew() == straight.getDeskew()
    for f in range(2, 5):
        for m in (straight, resumed):
            m.processScan(*seq[f][:3], times=seq[f][3])
        assert_bits_equal(resumed.getCurrentPose(), straight.getCurrentPose(), "scan %d pose" % f)
        surfel_fields_equal(resumed.getMap().getAllSurfels(), straight.getMap().getAllSurfels(), "scan %d" % f)
    for m in (straight, first, resumed):
        m.ctx.close()


def test_default_checkpoint_has_no_section_and_loads_deskewing_off():
    _, pp = both_params(**sized(900))
    pts, _, _, _ = rolling_scans(900, n=1)[0]
    a, b, on = api.SurfelMapping(pp), api.SurfelMapping(pp), api.SurfelMapping(pp)
    b.setDeskew("azimuth")
    b.setDeskew("off")
    on.setDeskew("azimuth")
    for m in (a, b, on):
        m.processScan(pts)
    # (the blobs differ in the wall-clock statistics only: compare their layout)
    assert len(a.save_state()) == len(b.save_state()) == len(on.save_state()) - 32  # one 32-byte section when on
    assert struct.pack("<IIQ", 10, 0, 16) not in a.save_state()
    c = api.SurfelMapping(pp)
    c.setDeskew("azimuth", clockwise=False)
    c.load_state(a.save_state())
    assert c.getDeskew()["mode"] == 0
    for m in (a, b, c, on):
        m.ctx.close()


def test_same_launches_with_deskewing_on_and_off():
    _, pp = both_params(**sized(900))
    seq = rolling_scans(900, n=3)
    counts = []
    for mode in ("off", "azimuth"):
        m = api.SurfelMapping(pp)
        m.setDeskew(mode)
        per = []
        for pts, _, _, _ in seq:
            c0 = m.ctx.launch_count()
            m.processScan(pts)
            per.append(m.ctx.launch_count() - c0)
        counts.append(per)
        m.ctx.close()
    assert counts[0] == counts[1]


def test_first_scan_with_deskewing_equals_deskewing_off():
    _, pp = both_params(**sized(900))
    pts, lab, prb, s = rolling_scans(900, n=1, semantic=True)[0]
    off, on = api.SurfelMapping(pp), api.SurfelMapping(pp)
    on.setDeskew("times")
    off.processScan(pts, lab, prb)
    on.processScan(pts, lab, prb, times=s)  # scan 0: lastIncrement_ is the identity
    assert_frames(on.getCurrentFrame().maps(), off.getCurrentFrame().maps(), "scan 0")
    surfel_fields_equal(on.getMap().getAllSurfels(), off.getMap().getAllSurfels(), "scan 0")
    off.ctx.close()
    on.ctx.close()


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_state_unchanged():
    _, pp = both_params(**sized(900))
    pts, _, _, s = rolling_scans(900, n=1)[0]
    m = api.SurfelMapping(pp)
    m.setDeskew("azimuth", ref_time=0.3)
    before = m.getDeskew()
    for bad in (dict(mode=3), dict(mode=-1), dict(mode=2, ref_time=1.5), dict(mode=2, ref_time=-0.1),
                dict(mode=2, ref_time=float("nan")), dict(mode=2, start_azimuth=float("inf")),
                dict(mode=2, start_azimuth=float("nan"))):
        with pytest.raises(api.SumaError):
            m.setDeskew(**bad)
        assert m.getDeskew() == before
    with pytest.raises(api.SumaError):
        m.processScan(pts, times=s)  # times while the mode is 2
    assert m.timestamp() == 0
    m.setDeskew("times")
    with pytest.raises(api.SumaError):
        m.processScan(pts)  # mode 1 without times
    assert m.timestamp() == 0
    m.processScan(pts, times=s)
    assert m.timestamp() == 1
    m.ctx.close()


def test_checkpoint_with_a_deskew_section_out_of_range_is_refused():
    _, pp = both_params(**sized(900))
    pts, _, _, s = rolling_scans(900, n=1)[0]
    m = api.SurfelMapping(pp)
    m.setDeskew("times", ref_time=0.25)
    m.processScan(pts, times=s)
    blob = bytearray(m.save_state())
    # section S_DESKEW = 10: id, 0, length 16, then mode, ref_time, start_azimuth, clockwise
    head = struct.pack("<IIQi", 10, 0, 16, 1) + struct.pack("<f", 0.25)
    at = bytes(blob).find(head)
    assert at > 0
    fresh = api.SurfelMapping(pp)
    fresh.setDeskew("azimuth", ref_time=0.75)
    for off, val in ((16, struct.pack("<i", 7)), (20, struct.pack("<f", 2.0)), (24, struct.pack("<f", float("inf"))),
                     (28, struct.pack("<i", 5))):
        bad = bytearray(blob)
        bad[at + off:at + off + 4] = val
        with pytest.raises(api.SumaError, match="deskew"):
            fresh.load_state(bytes(bad))
        assert fresh.getDeskew()["mode"] == 2 and fresh.timestamp() == 0
    fresh.load_state(bytes(blob))
    assert fresh.getDeskew()["mode"] == 1 and fresh.getDeskew()["ref_time"] == 0.25 and fresh.timestamp() == 1
    m.ctx.close()
    fresh.ctx.close()


# ---- row-striped ranks -----------------------------------------------------------------------------------------------
def test_two_striped_ranks_deskew_like_one(request):
    """Two ranks on one device, each in its own thread and context, row-striped through the host all-reduce callback
    (sb_comm_set_callback: the mode for ranks that share a GPU). Preprocessing is replicated per rank, so both deskew
    every scan identically and end with the poses and surfels of a one-rank run."""
    import ctypes as C
    import threading

    from semantic_suma_b200 import stripes

    if getattr(request.config, "_cusim", False):
        pytest.skip("two host threads driving two contexts: a GPU run")
    _, pp = both_params(**sized(900))
    seq = rolling_scans(900, n=4, semantic=True)
    solo = api.SurfelMapping(pp)
    solo.setDeskew("times")
    for pts, lab, prb, s in seq:
        solo.processScan(pts, lab, prb, times=s)
    barrier = threading.Barrier(2, timeout=60.0)
    parts = [None, None]

    def make_cb(rank):
        def cb(user, ptr):
            try:
                a = np.ctypeslib.as_array(ptr, shape=(32,))
                parts[rank] = a.copy()
                barrier.wait()
                total = parts[0] + parts[1]  # exact: integer sums
                barrier.wait()  # both have read before either deposits the next iteration's sums
                a[:] = total
                return 0
            except Exception:  # noqa: BLE001 -- a broken barrier fails the scan instead of waiting forever
                barrier.abort()
                return 1
        return stripes.ALLREDUCE_FN(cb)

    ranks, errors = [], []
    for r in range(2):
        m = api.SurfelMapping(pp)
        m.setDeskew("times")
        r0, r1 = stripes.row_stripe(r, 2, pp.data_height)
        m.ctx._allreduce_cb = make_cb(r)
        m.ctx.check(api.lib().sb_comm_set_callback(m.ctx.h, C.cast(m.ctx._allreduce_cb, C.c_void_p), None, r0, r1),
                    "comm_set_callback")
        ranks.append(m)

    def drive(m):
        try:
            for pts, lab, prb, s in seq:
                m.processScan(pts, lab, prb, times=s)
        except Exception as e:  # noqa: BLE001
            errors.append(e)
            barrier.abort()

    threads = [threading.Thread(target=drive, args=(m,)) for m in ranks]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for r, m in enumerate(ranks):
        assert_bits_equal(m.getCurrentPose(), solo.getCurrentPose(), "rank %d pose" % r)
        surfel_fields_equal(m.getMap().getAllSurfels(), solo.getMap().getAllSurfels(), "rank %d surfels" % r)
        m.ctx.close()
    solo.ctx.close()
