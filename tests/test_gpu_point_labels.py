"""Per-point label records (sb_set_point_labels / sb_get_point_labels; DESIGN.md section 13) against the oracle bit for
bit after every scan of whole runs: semantic and geometric, three image shapes, both deskewing modes, model images that
differ from the data image, a track-loss recovery, loop closure, input staged by sb_prefetch_scan and device-resident
points and records. Also: the mode changes no other result (poses, frames, map, statistics, checkpoints) and adds one
launch per scan, the rules for when records exist, and the C++ mirror.

On the CPU executor (pytest --cusim) the long runs at 64x2048 and 128x4096 are cut to their first scans unless
SUMA_B200_POINT_LABELS_FULL=1."""
import os
import struct
import subprocess

import numpy as np
import pytest

from oracle import point_labels as OPL
from semantic_suma_b200 import api, synth
from helpers import assert_bits_equal, both_params, sized, surfel_fields_equal

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FULL = os.environ.get("SUMA_B200_POINT_LABELS_FULL") == "1"
LOOP = dict(search_distance=3.0, min_trajectory_distance=15.0, min_verifications=2)


@pytest.fixture
def short(request):
    """the number of scans a long run is cut to on the CPU executor (None: the whole run)"""
    return 3 if getattr(request.config, "_cusim", False) and not FULL else None


def as_words(rec):
    return np.ascontiguousarray(rec).view(np.uint32).reshape(-1, 8)


def assert_records(g, o, what):
    assert g.dtype.itemsize == 32 and o.dtype.itemsize == 32
    assert_bits_equal(as_words(g), as_words(o), what + " records")


def sequence(width, height=64, n=4, semantic=False, jump_at=None, rolling=None, clean=False, **scene):
    sc = synth.Scene(width=width, height=height, semantic=semantic, **scene)
    poses = synth.trajectory(n, **({} if rolling is None else dict(step=1.2, yaw_deg=3.0)))
    J = synth.translate(0.8, 0.3, 0) @ synth.rot_z(np.deg2rad(8.0))
    out = []
    for f in range(n):
        P = poses[f] if jump_at is None or f < jump_at else poses[f] @ J
        out.append(sc.scan(f, P, rolling=rolling, clean_labels=clean) if clean else sc.scan(f, P, rolling=rolling))
    return out


def run_pair(params, seq, deskew=0, setup=None, each=None):
    """both engines over seq with the records on; the records, poses and map compared after every scan"""
    po, pp = both_params(**params)
    g, o = api.SurfelMapping(pp), OPL.Slam(po)
    try:
        g.setPointLabels(True)
        if deskew:
            g.setDeskew({1: "times", 2: "azimuth"}[deskew])
            o.set_deskew(deskew)
        if setup:
            setup(g, o)
        for t, scan in enumerate(seq):
            pts, lab, prb = scan[:3]
            times = scan[3] if deskew == 1 else None
            if each:
                each(g, t, pts, lab, prb)
            else:
                g.processScan(pts, lab, prb, times=times)
            o.process_scan(pts, lab, prb, times=times)
            what = "t=%d" % t
            assert_bits_equal(g.getCurrentPose(), o.pose(), what + " pose")
            rec = g.getPointLabels()
            assert rec.shape[0] == pts.shape[0]
            assert_records(rec, o.records, what)
        surfel_fields_equal(g.getMap().getAllSurfels(), o.map.download(), "end surfels")
        return g.getStatistics(), o.records
    finally:
        g.ctx.close()


# ---- whole runs against the oracle ---------------------------------------------------------------------------------
def test_semantic_64x2048_with_moving_cars_flips_and_paging(short):
    """the semantic synthetic sequence; a 4 m submap extent makes the window move and page tiles out within the run"""
    n = short or 12
    st, rec = run_pair(sized(2048, submap_extent=4.0), sequence(2048, n=n, semantic=True))
    assert (rec["flags"] & api.POINT_MAP).any() and (rec["flags"] & api.POINT_INTEGRATED).any()
    assert len(np.unique(rec["map_label"])) >= 3  # ground, buildings and cars reach the map


def test_geometric_64x900():
    _, rec = run_pair(sized(900), sequence(900, n=5))
    assert not rec["frame_label"].any() and not rec["map_label"].any()


def test_128x4096_with_15_iterations(short):
    run_pair(sized(4096, 128, max_iterations=15), sequence(4096, 128, n=short or 4))


@pytest.mark.parametrize("mode", [1, 2], ids=["times", "azimuth"])
def test_deskewed_runs(mode):
    inc = synth.translate(1.2, 0, 0) @ synth.rot_z(np.deg2rad(3.0))
    run_pair(sized(900), sequence(900, n=4, semantic=True, rolling=inc), deskew=mode)


@pytest.mark.parametrize("model", [
    dict(data_width=513, data_height=33, model_width=451, model_height=47),
    dict(sized(900), model_fov_up=4.0, model_fov_down=-26.0),
], ids=["model_451x47_data_513x33", "model_fov_differs"])
def test_model_image_differs_from_the_data_image(model):
    _, rec = run_pair(model, sequence(model["data_width"], model["data_height"], n=4, semantic=True))
    hit = rec["pixel"] >= 0
    assert (rec["map_pixel"][hit] != rec["pixel"][hit]).any()


def test_track_loss_recovery():
    st, _ = run_pair(sized(900), sequence(900, n=7, jump_at=4))
    assert st["track_loss"] >= 1, "the sequence must trigger the recovery"


def test_loop_closure_on():
    run_pair(sized(900), sequence(900, n=5, semantic=True),
             setup=lambda g, o: (g.enableLoopClosure(**LOOP), o.enable_loop_closure(**LOOP)))


def test_render_after_update_off_sets_no_map_flag():
    _, rec = run_pair(sized(900, render_after_update=0), sequence(900, n=3, semantic=True))
    assert not (rec["flags"] & api.POINT_MAP).any() and (rec["map_pixel"] >= 0).any()


def test_prefetched_input():
    seq = sequence(900, n=4, semantic=True)
    bufs = [tuple(np.ascontiguousarray(a, np.float32) for a in s[:3]) for s in seq]

    def each(g, t, pts, lab, prb):
        p, l, q = bufs[t]
        if t == 0:
            g.prefetch_scan_raw(p.ctypes.data, l.ctypes.data, q.ctypes.data, p.shape[0])
        if t + 1 < len(bufs):
            pn, ln, qn = bufs[t + 1]
            g.prefetch_scan_raw(pn.ctypes.data, ln.ctypes.data, qn.ctypes.data, pn.shape[0])
        g.process_scan_raw(p.ctypes.data, l.ctypes.data, q.ctypes.data, p.shape[0], False)

    run_pair(sized(900), [b for b in bufs], each=each)


class DeviceBuffers:
    """device memory for the points and the records: torch on a CUDA device; on the CPU executor, whose device memory is
    host memory, numpy arrays"""

    def __init__(self):
        try:
            import torch
            self.torch = torch if torch.cuda.is_available() else None
        except ImportError:
            self.torch = None
        self.keep = []

    def put(self, a):
        a = np.ascontiguousarray(a, np.float32)
        if self.torch is None:
            self.keep.append(a)
            return a.ctypes.data
        t = self.torch.from_numpy(a).cuda()
        self.keep.append(t)
        return t.data_ptr()

    def empty_records(self, n):
        if self.torch is None:
            a = np.zeros(n, api.POINT_LABEL_DTYPE)
            self.keep.append(a)
            return a.ctypes.data, lambda: a.copy()
        t = self.torch.zeros(n * 32, dtype=self.torch.uint8, device="cuda")
        self.keep.append(t)
        return t.data_ptr(), lambda: t.cpu().numpy().view(api.POINT_LABEL_DTYPE).copy()


def test_points_and_records_on_the_device():
    seq = sequence(900, n=4, semantic=True)
    dev = DeviceBuffers()
    po, pp = both_params(**sized(900))
    g, o = api.SurfelMapping(pp), OPL.Slam(po)
    try:
        g.setPointLabels(True)
        for t, (pts, lab, prb) in enumerate(seq):
            g.processScan((dev.put(pts), dev.put(lab), dev.put(prb), pts.shape[0]), on_device=True)
            o.process_scan(pts, lab, prb)
            ptr, fetch = dev.empty_records(pts.shape[0])
            assert g.getPointLabels(out=ptr) == pts.shape[0]
            assert_records(fetch(), o.records, "t=%d device copy" % t)
            assert_records(g.getPointLabels(), o.records, "t=%d host copy" % t)
    finally:
        g.ctx.close()


# ---- the mode changes nothing else ---------------------------------------------------------------------------------
def untimed_checkpoint(g):
    """the checkpoint's bytes without the wall-clock slots [8, 12) of its statistics and without the digest over them"""
    blob = g.save_state()
    st = np.zeros(16)
    api.lib().sb_get_statistics(g.ctx.h, api._dp(st))
    head = st[:8].tobytes()
    pos = blob.find(head)
    assert pos >= 0 and blob.find(head, pos + 1) < 0 and blob[pos + 64:pos + 96] == st[8:12].tobytes()
    return blob[:pos + 64] + blob[pos + 96:-8]


def _session(on, seq, params):
    g = api.SurfelMapping(api.default_params(**params))
    try:
        g.setPointLabels(on)
        launches, poses, stats = [], [], []
        for pts, lab, prb in seq:
            c0 = g.ctx.launch_count()
            g.processScan(pts, lab, prb)
            launches.append(g.ctx.launch_count() - c0)
            poses.append(g.getCurrentPose())
            s = g.getStatistics()
            stats.append([v for k, v in sorted(s.items()) if not k.endswith("-time")])
        frames = [g._frame(k).maps() for k in range(4)] + [g.getMap()._frame(k).maps() for k in range(3)]
        return dict(launches=launches, poses=poses, stats=stats, frames=frames, map=g.getMap().getAllSurfels(),
                    state=untimed_checkpoint(g))
    finally:
        g.ctx.close()


def test_mode_on_changes_no_other_result():
    seq = sequence(900, n=5, semantic=True)
    off, on = _session(False, seq, sized(900)), _session(True, seq, sized(900))
    assert [b - a for a, b in zip(off["launches"], on["launches"])] == [1] * len(seq)
    for a, b in zip(off["poses"], on["poses"]):
        assert_bits_equal(a, b, "pose")
    assert_bits_equal(np.array(off["stats"]), np.array(on["stats"]), "statistics")
    for k, (fa, fb) in enumerate(zip(off["frames"], on["frames"])):
        for a, b in zip(fa, fb):
            assert_bits_equal(a, b, "frame %d" % k)
    surfel_fields_equal(off["map"], on["map"])
    assert off["state"] == on["state"], "checkpoint bytes"


def _refused(fn, code):
    with pytest.raises(api.SumaError) as e:
        fn()
    assert code in str(e.value)


def test_when_records_exist():
    seq = sequence(450, n=3, semantic=True)
    pp = api.default_params(**sized(450))
    g = api.SurfelMapping(pp)
    try:
        _refused(g.getPointLabels, "SB_ERR_STATE")  # mode off
        g.processScan(*seq[0])
        _refused(g.getPointLabels, "SB_ERR_STATE")  # a scan with the mode off leaves none
        g.setPointLabels(True)
        _refused(g.getPointLabels, "SB_ERR_STATE")  # none before the first scan with the mode on
        g.processScan(*seq[1])
        n = seq[1][0].shape[0]
        assert g.getPointLabels().shape[0] == n
        # cap too small: SB_ERR_INVALID, *n set, nothing written
        cnt = api.C.c_uint32(0)
        small = np.full((n - 1) * 32, 0x5a, np.uint8)
        rc = api.lib().sb_get_point_labels(g.ctx.h, api._vp(small), n - 1, api.C.byref(cnt), 0)
        assert rc == api.SB_ERR_INVALID and cnt.value == n and (small == 0x5a).all()
        blob = g.save_state()
        g.reset()
        _refused(g.getPointLabels, "SB_ERR_STATE")
        g.processScan(*seq[0])  # the mode is kept across reset
        assert g.getPointLabels().shape[0] == seq[0][0].shape[0]
        g.load_state(blob)
        _refused(g.getPointLabels, "SB_ERR_STATE")
        g.processScan(*seq[2])
        g.ctx.set_params(pp)
        _refused(g.getPointLabels, "SB_ERR_STATE")
        g.processScan(*seq[2])
        g.setPointLabels(False)
        _refused(g.getPointLabels, "SB_ERR_STATE")
        g.setPointLabels(True)
        g.processScan(np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros(0, np.float32))
        assert g.getPointLabels().shape == (0,)  # a scan of no points has zero records
    finally:
        g.ctx.close()


def test_profile_class_is_named():
    names = [api.lib().sb_profile_name(k).decode() for k in range(api.lib().sb_profile_kernels())]
    assert "point_labels" in names


# ---- the C++ mirror ------------------------------------------------------------------------------------------------
def test_cpp_shim_point_labels(tmp_path):
    from semantic_suma_b200 import build as product_build
    api.lib()
    so = product_build.LIB  # under pytest --cusim the CPU executor's build of the same sources (conftest)
    exe = os.path.join(str(tmp_path), "point_labels_example")
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "point_labels_example.cpp"), so,
                           "-Wl,-rpath," + os.path.dirname(so)])
    seq = sequence(900, n=3)
    path, out = os.path.join(str(tmp_path), "scans.bin"), os.path.join(str(tmp_path), "records.bin")
    with open(path, "wb") as f:
        for pts, _, _ in seq:
            f.write(struct.pack("<I", pts.shape[0]))
            f.write(np.ascontiguousarray(pts, np.float32).tobytes())
    log = subprocess.check_output([exe, path, "900", out], text=True)
    assert "size 32" in log
    pp = api.default_params(data_width=900, model_width=900, max_iterations=10)
    g = api.SurfelMapping(pp)
    try:
        g.setPointLabels(True)
        for pts, _, _ in seq:
            g.processScan(pts)
        assert open(out, "rb").read() == g.getPointLabels().tobytes()
    finally:
        g.ctx.close()


# ---- label quality (reported, not a gate) --------------------------------------------------------------------------
def test_report_map_label_agreement_with_the_labels_before_the_flips(short, capsys):
    """how often the map's label of a WON point equals the synthetic label before the 2 % flips, beside how often the
    input label does; printed for DESIGN.md section 13"""
    n = short or 12
    seq = sequence(2048, n=n, semantic=True, clean=True)
    g = api.SurfelMapping(api.default_params(**sized(2048)))
    rows = []
    try:
        g.setPointLabels(True)
        for t, (pts, lab, prb, clean) in enumerate(seq):
            g.processScan(pts, lab, prb)
            r = g.getPointLabels()
            won = (r["flags"] & api.POINT_WON) != 0
            mapped = won & ((r["flags"] & api.POINT_MAP) != 0)
            flipped = lab != clean
            rows.append((t, won.sum(), mapped.sum(), (r["map_label"][mapped] == clean[mapped]).mean(),
                         (lab[mapped] == clean[mapped]).mean(), flipped[mapped].sum(),
                         (r["map_label"][mapped & flipped] == clean[mapped & flipped]).mean()))
    finally:
        g.ctx.close()
    with capsys.disabled():
        print("\nscan won mapped map==clean input==clean flipped map==clean(flipped)")
        for row in rows:
            print("%4d %6d %6d %9.4f %11.4f %7d %9.4f" % row)
