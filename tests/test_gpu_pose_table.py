"""The pose table past the reference's 10 000 entries: it doubles on demand up to 2^24 entries, and the per-scan product
tables inv(P) * poses[t] cover only the entries the active map can refer to. Checked bit for bit against the oracle
built with a pose table large enough for the run (oracle/poses.py), and against itself under a shift of every timestamp
(DESIGN.md section 12)."""
import struct

import numpy as np
import pytest

from oracle import oracle as O
from oracle import poses as OP
from semantic_suma_b200 import api, synth
from helpers import assert_bits_equal, both_params, sized, surfel_fields_equal

pytestmark = pytest.mark.gpu

CAP0 = 10_000   # SurfelMap.h:205
CAP_MAX = 1 << 24


def uturn(n, reach=25.0):
    """out along x and back (the window moves both ways: tiles are extracted and re-inserted)"""
    out = []
    for i in range(n):
        T = synth.translate(reach * np.sin(np.pi * i / n), 0.0, 2.0)
        out.append(T @ synth.rot_z(np.deg2rad(0.3 * i)))
    return out


def sequence(width, height, n, reach=25.0):
    sc = synth.Scene(width=width, height=height)
    return [sc.scan(f, P)[0] for f, P in enumerate(uturn(n, reach))]


def run_pair(pts, start=0, width=900, height=64, extent=5.0, check_each=True):
    po, pp = both_params(**sized(width, height, submap_extent=extent))
    g, o = api.SurfelMapping(pp), O.Slam(po)
    if start:
        empty = np.zeros(0, O.SURFEL_DTYPE)
        g.getMap().upload(empty, start)
        o.map.upload(empty, start)
    for t, p in enumerate(pts):
        g.processScan(p)
        o.process_scan(p)
        if check_each:
            assert_bits_equal(g.getCurrentPose(), o.pose(), "pose after scan %d (map timestamp %d)" % (t, start + t))
    return g, o


def run_lib(pts, start=0, width=900, height=64, extent=5.0):
    _, pp = both_params(**sized(width, height, submap_extent=extent))
    g = api.SurfelMapping(pp)
    if start:
        g.getMap().upload(np.zeros(0, O.SURFEL_DTYPE), start)
    poses = []
    for p in pts:
        g.processScan(p)
        poses.append(g.getCurrentPose())
    return g, poses


def raw_sums(g):
    st = np.zeros(16)
    api.lib().sb_get_statistics(g.ctx.h, api._dp(st))
    return st[:6]


def test_the_oracle_copy_is_the_oracle():
    """at the reference's 10 000 entries the copy of oracle/poses.py computes what liborc.so computes"""
    pts = sequence(900, 64, 4)
    _, o = run_pair(pts, check_each=False)
    with OP.oracle(CAP0):
        _, c = run_pair(pts, check_each=False)
        assert_bits_equal(c.pose(), o.pose(), "pose")
        surfel_fields_equal(c.map.download(), o.map.download(), "surfels")
        del c


def test_crossing_the_old_limit_matches_the_oracle():
    pts = sequence(900, 64, 40)
    with OP.oracle(2 * CAP0):
        g, o = run_pair(pts, start=9990)
        o_surfels, so = o.map.download(), o.stats()
        del o
    surfel_fields_equal(g.getMap().getAllSurfels(), o_surfels, "surfels after 9990 + 40 scans")
    assert_bits_equal(raw_sums(g), np.asarray([so[k] for k in ("iterations", "F", "inlier", "outlier", "invalid",
                                                               "inlier_residual")]), "the last scan's ICP sums")
    info = g.getMap().pose_table_info()
    assert info["capacity"] == 2 * CAP0
    assert info["begin"] > 0 and info["begin"] <= 9990 + 40 and info["end"] == 9990 + 40 + 1
    tc = g.getMap().tile_cache_info()
    assert tc["tiles_in_pool"] > 0, "the sequence extracts tiles"
    assert o_surfels["count"].min() >= info["begin"], "the window's begin is a lower bound of the live entries"


@pytest.mark.parametrize("K", [CAP0, 1 << 23])
def test_shift_invariance(K):
    """the same scans from map timestamp 0 and from K: equal poses, and surfels equal once count and timestamp are
    shifted by K (no shader formula depends on the absolute timestamp at these K)"""
    pts = sequence(900, 64, 14, reach=12.0)
    g0, p0 = run_lib(pts, 0)
    gk, pk = run_lib(pts, K)
    for t, (a, b) in enumerate(zip(p0, pk)):
        assert_bits_equal(a, b, "pose after scan %d" % t)
    s0, sk = g0.getMap().getAllSurfels(), gk.getMap().getAllSurfels()
    assert s0.shape == sk.shape
    s0 = s0.copy()
    s0["count"] = s0["count"] + np.float32(K)
    s0["timestamp"] = s0["timestamp"] + np.uint32(K)
    surfel_fields_equal(s0, sk, "shifted surfels")
    # the oracle on the CPU shows the same invariance at K
    with OP.oracle(K + 7):
        o0, ok = run_pair(pts[:6], 0, check_each=False)[1], run_pair(pts[:6], K, check_each=False)[1]
        assert_bits_equal(o0.pose(), ok.pose(), "oracle pose")
        del o0, ok
    assert gk.getMap().pose_table_info()["capacity"] >= K + len(pts)


def test_one_long_run_matches_the_oracle(request):
    if getattr(request.config, "_cusim", False):
        pytest.skip("10 050 scans: GPU only")
    n = 10_050
    sc = synth.Scene(width=256, height=16)
    # small tiles: paging keeps the active map (and the oracle's time per scan) bounded over the whole run
    po, pp = both_params(**sized(256, 16, submap_extent=5.0))
    T = synth.translate(0, 0, 2.0)
    inc = synth.translate(0.1, 0, 0) @ synth.rot_z(np.deg2rad(0.05))
    with OP.oracle(2 * CAP0):
        g, o = api.SurfelMapping(pp), O.Slam(po)
        for t in range(n):
            p = sc.scan(t % 50, T)[0]
            T = T @ inc
            g.processScan(p)
            o.process_scan(p)
            assert_bits_equal(g.getCurrentPose(), o.pose(), "pose after scan %d" % t)
        surfel_fields_equal(g.getMap().getAllSurfels(), o.map.download(), "surfels after 10 050 scans")
        del o
    assert g.getMap().pose_table_info()["capacity"] == 2 * CAP0


def _map_pair(width=128, height=16):
    po, pp = both_params(**sized(width, height))
    ctx = api.Context(pp)
    return po, pp, ctx, api.SurfelMap(ctx), O.Map(po)


def test_set_pose_grows_and_refuses_past_the_last_entry():
    _, _, ctx, gm, _ = _map_pair()
    pose = np.eye(4, dtype=np.float32)
    pose[0, 3] = 3.0
    for t, cap in ((CAP0 - 1, CAP0), (CAP0, 2 * CAP0), (65_535, 80_000), (CAP_MAX - 1, CAP_MAX)):
        gm.set_pose(t, pose)
        assert gm.pose_table_info()["capacity"] == cap, t
    before = gm.pose_table_info()
    with pytest.raises(api.SumaError):
        gm.set_pose(CAP_MAX, pose)
    assert "16777215" in api.lib().sb_last_error(ctx.h).decode()
    assert gm.pose_table_info() == before
    ctx.check(api.lib().sb_reset(ctx.h), "reset")
    assert gm.pose_table_info()["capacity"] == CAP0
    ctx.close()


def _surfels(n, entry_lo, entry_hi, seed=5):
    rng = np.random.default_rng(seed)
    s = np.zeros(n, O.SURFEL_DTYPE)
    s["x"] = rng.uniform(-20, 20, n); s["y"] = rng.uniform(-20, 20, n); s["z"] = rng.uniform(-1, 2, n)
    s["nx"] = -s["x"]; s["ny"] = -s["y"]
    nrm = np.sqrt(s["nx"] ** 2 + s["ny"] ** 2)
    s["nx"] /= nrm; s["ny"] /= nrm
    s["radius"] = rng.uniform(0.2, 0.6, n)
    s["confidence"] = 10.0
    s["weight"] = 1.0
    e = rng.integers(entry_lo, entry_hi, n)
    s["count"] = e.astype(np.float32)
    s["timestamp"] = e.astype(np.uint32)
    return s


def _frames_equal(ctx, gm, om, pose, what):
    f = api.Frame(ctx, 128, 16)
    gm.render(pose, pose, f, 0.0)
    ov = om.render(pose, pose, 0.0)
    for i, (a, b) in enumerate(zip(f.maps(), ov)):
        assert_bits_equal(a, b, "%s: rendered image %d" % (what, i))


def test_update_poses_and_upload_beyond_the_old_limit_render_like_the_oracle():
    with OP.oracle(2 * CAP0):
        _update_poses_and_upload()


def _update_poses_and_upload():
    po, pp, ctx, gm, om = _map_pair()
    rng = np.random.default_rng(2)
    poses = []
    for t in range(12_000):
        P = np.eye(4, dtype=np.float32)
        P[:3, 3] = rng.uniform(-0.5, 0.5, 3)
        poses.append(P)
    s = _surfels(3000, 9_000, 12_000)
    gm.upload(s, 12_000)
    om.upload(s, 12_000)
    gm.updatePoses(poses)
    for t, P in enumerate(poses):
        om.set_pose(t, P)
    assert gm.pose_table_info()["capacity"] == 2 * CAP0
    _frames_equal(ctx, gm, om, np.eye(4, dtype=np.float32), "after update_poses")
    # one map update on top: the entries at and above 10 000 place the surfels it fuses
    f = api.Frame(ctx, 128, 16)
    ov = [np.zeros((16, 128, 4), np.float32) for _ in range(3)]
    gm.update(np.eye(4, dtype=np.float32), f)
    om.update(np.eye(4, dtype=np.float32), ov)
    surfel_fields_equal(gm.getAllSurfels(), om.download(), "after an update")
    with pytest.raises(api.SumaError):
        bad = s[:1].copy()
        bad["count"] = np.float32(CAP_MAX)
        gm.upload(bad, 5)
    assert gm.size() == om.size()
    del om
    ctx.close()


def test_checkpoint_of_a_grown_table():
    pts = sequence(900, 64, 16, reach=10.0)
    po, pp = both_params(**sized(900, 64, submap_extent=5.0))
    a = api.SurfelMapping(pp)
    a.getMap().upload(np.zeros(0, O.SURFEL_DTYPE), 9_995)
    for p in pts[:10]:
        a.processScan(p)
    blob = a.save_state()
    assert struct.unpack_from("<I", blob, 20)[0] == 2 * CAP0, "header pose capacity"
    b = api.SurfelMapping(pp)
    b.load_state(blob)
    assert b.getMap().pose_table_info()["capacity"] == 2 * CAP0
    assert b.save_state() == blob, "save(load(save(x))) == save(x)"
    for p in pts[10:]:
        a.processScan(p)
        b.processScan(p)
        assert_bits_equal(a.getCurrentPose(), b.getCurrentPose(), "pose after the load")
    surfel_fields_equal(a.getMap().getAllSurfels(), b.getMap().getAllSurfels(), "surfels after the load")
    # a run that never grew writes the initial capacity; a grown context loading it shrinks back
    c = api.SurfelMapping(pp)
    for p in pts[:3]:
        c.processScan(p)
    small = c.save_state()
    assert struct.unpack_from("<I", small, 20)[0] == CAP0
    b.load_state(small)
    assert b.getMap().pose_table_info()["capacity"] == CAP0
    assert b.save_state() == small
