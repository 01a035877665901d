"""The in-place (lazy) map update of the per-scan pipeline against the oracle. Most scans store only the lanes that changed
and leave removed surfels behind as dead slots; a dense scan (update into the scratch set + ordered compaction) runs once
the dead slots reach 1/8 of the physical end or the capacity could be reached. Observers (size, download, the
operator-level update, paging) must see exactly the compacted map of the reference."""
import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api, synth
from helpers import assert_bits_equal, both_params, scans, sized, surfel_fields_equal

pytestmark = pytest.mark.gpu

MAX_SURFELS = 2048 * 2048


def scan_modes(gsl):
    """'dense' / 'lazy' / None (no update launch) for the scan just processed, from the profiler's launch counts: every
    dense update ends in one compaction of its own, tile extractions and map compactions pair one with extract_flags;
    and the launch counts"""
    prof = gsl.ctx.profile_collect()
    cnt = {k: v[1] for k, v in prof.items()}
    dense = cnt.get("compact_scatter", 0) - cnt.get("extract_flags", 0)
    assert dense in (0, 1), prof
    if dense:
        return "dense", cnt
    return ("lazy" if cnt.get("update_surfels", 0) else None), cnt


def lockstep(osl, gsl, scan_list, what, sizes=None, launches=None):
    """process every scan on both, no map observation in between but size(); pose bits and size after every scan"""
    modes = []
    sizes = [] if sizes is None else sizes
    launches = [] if launches is None else launches
    gsl.ctx.profile(True)
    gsl.ctx.profile_collect()
    for t, (pts, lab, prb) in enumerate(scan_list):
        osl.process_scan(pts, lab, prb)
        gsl.processScan(pts, lab, prb)
        mode, cnt = scan_modes(gsl)
        modes.append(mode)
        launches.append(cnt)
        assert_bits_equal(gsl.getCurrentPose(), osl.pose(), "%s t=%d pose" % (what, t))
        assert gsl.getMap().size() == osl.map.size(), "%s t=%d size %d vs %d" % (what, t, gsl.getMap().size(),
                                                                               osl.map.size())
        sizes.append(osl.map.size())
    gsl.ctx.profile(False)
    return modes


@pytest.mark.parametrize("width", [900, 2048])
def test_thirty_scans_in_place_and_dense(width):
    """(a) 32 pipeline scans: both kinds of update occur, every pose and size on the way and every surfel at the end"""
    po, pp = both_params(**sized(width))
    sc, _ = scans(width, n=32)
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    try:
        modes = lockstep(osl, gsl, sc, "%d" % width)
        assert modes.count("lazy") >= 10, modes
        assert "dense" in modes[1:], modes  # (scan 0 updates the empty map densely)
        surfel_fields_equal(gsl.getMap().getAllSurfels(), osl.map.download(), "surfels")
        for g, o in zip(gsl.getLastModelFrame().maps(), osl.frame(1)):
            assert_bits_equal(g, o, "model frame")
    finally:
        gsl.ctx.close()


def test_operators_on_a_map_with_dead_slots():
    """(b) pipeline scans ending in an in-place update, then render, operator-level update + update_debug (the index map
    indexes the compacted map) and download"""
    po, pp = both_params(**sized(900))
    sc, poses = scans(900, n=6)
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    try:
        modes = lockstep(osl, gsl, sc[:5], "pipeline")
        assert modes[-1] == "lazy", modes
        om, gm = osl.map, gsl.getMap()
        pose = gsl.getCurrentPose().astype(np.float32)
        out = api.Frame(gsl.ctx, 900, 64)
        orr = om.render(pose, pose, -1.0)
        gm.render(pose, pose, out, -1.0)
        for g, o in zip(out.maps(), orr):
            assert_bits_equal(g, o, "render with dead slots")
        pts, lab, prb = sc[5]
        ov = O.preprocess(po, pts, lab, prb, 5)
        f = api.Frame(gsl.ctx, 900, 64)
        api.Preprocessing(gsl.ctx).process(pts, f, lab, prb, 5)
        om.update(pose, ov)
        gm.update(pose, f)
        oi, orad, oint, onu, onn = om.update_debug()
        gi, grad, gint, gnu, gnn = gm.update_debug()
        assert_bits_equal(gi, oi, "index map")
        assert_bits_equal(grad, orad, "radius map")
        assert_bits_equal(gint, oint, "integrated flags")
        assert (gnu, gnn) == (onu, onn)
        assert gm.size() == om.size()
        surfel_fields_equal(gm.getAllSurfels(), om.download(), "surfels after the operator-level update")
    finally:
        gsl.ctx.close()


def test_paging_while_dead_slots_exist():
    """(c) small tiles, partial_extraction = 0: whole columns leave on the way out and come back on the way back, while
    the in-place updates leave dead slots behind"""
    kw = sized(900, submap_extent=3.0, submap_dimension=1, partial_extraction=0)
    po, pp = both_params(**kw)
    scene = synth.Scene(width=900, height=64)
    poses = synth.trajectory(14)
    order = list(range(14)) + list(range(12, -1, -1))
    sc = [scene.scan(i, poses[j]) for i, j in enumerate(order)]
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    try:
        modes = lockstep(osl, gsl, sc, "paging")
        assert modes.count("lazy") >= 5, modes
        assert osl.map.submap_origin()[:2] == gsl.getMap().submap_origin()[:2]
        surfel_fields_equal(gsl.getMap().getAllSurfels(), osl.map.download(), "surfels after paging")
    finally:
        gsl.ctx.close()


def _hidden_surfels(n, seed, unstable):
    """n surfels below the field of view (never rendered, matched or fused, kept by the submap window); a fraction
    `unstable` of them is unconfident and dies at the update of scan 3 + its timestamp (0..7)"""
    rng = np.random.default_rng(seed)
    s = np.zeros(n, O.SURFEL_DTYPE)
    s["x"] = rng.uniform(-60.0, 60.0, n)
    s["y"] = rng.uniform(-60.0, 60.0, n)
    s["z"] = -60.0
    s["nz"] = 1.0
    s["radius"] = 0.2
    s["confidence"] = 10.0
    s["weight"] = 1.0
    s["color"] = np.float32(0.5)
    u = rng.random(n) < unstable
    s["confidence"][u] = -1.0
    s["timestamp"][u] = rng.integers(0, 8, int(u.sum()))
    return s


def test_capacity_near_the_surfel_limit():
    """(d) a map uploaded just over one image's worth of pixels below the 4 194 304-surfel capacity, with unstable
    surfels dying on the way: in place while the new surfels cannot reach the capacity, dense after, and the generation
    pass cut at the capacity exactly where the compacted map of the reference is cut"""
    po, pp = both_params(**sized(900))
    sc, _ = scans(900, n=8)
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    try:
        s = _hidden_surfels(MAX_SURFELS - 900 * 64 - 1000, 11, 0.003)
        osl.map.upload(s, 0)
        gsl.getMap().upload(s, 0)
        sizes = []
        modes = lockstep(osl, gsl, sc, "near capacity", sizes)
        assert modes[0] == "lazy" and "dense" in modes, modes
        assert MAX_SURFELS in sizes, sizes  # the generation pass was cut at the capacity
        surfel_fields_equal(gsl.getMap().getAllSurfels(), osl.map.download(), "surfels at the capacity")
    finally:
        gsl.ctx.close()


def test_adversarial_records_then_in_place_updates():
    """(e) records the update must carry bit for bit: -0.0, NaN lanes, confidences above the clamp of 20, colours that
    are no colour the update writes; then in-place scans and a download"""
    po, pp = both_params(**sized(900))
    sc, _ = scans(900, n=9)
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    try:
        lockstep(osl, gsl, sc[:4], "before")
        s = osl.map.download()
        surfel_fields_equal(gsl.getMap().getAllSurfels(), s, "before the upload")
        rng = np.random.default_rng(5)
        n = s.shape[0]
        pick = lambda frac: rng.random(n) < frac  # noqa: E731
        s["confidence"][pick(0.03)] = 25.0
        s["confidence"][pick(0.01)] = 1e30
        s["x"][pick(0.01)] = -0.0
        s["ny"][pick(0.02)] = -0.0
        s["g"][pick(0.05)] = np.nan
        s["b"].view(np.uint32)[pick(0.02)] = 0x7fc12345  # a NaN with a payload
        c = pick(0.05)
        s["color"].view(np.uint32)[c] = rng.integers(0, 2**32, int(c.sum()), dtype=np.uint64).astype(np.uint32)
        t = osl.map.timestamp()
        osl.map.upload(s, t)
        gsl.getMap().upload(s, t)
        modes = lockstep(osl, gsl, sc[4:], "after")
        assert "lazy" in modes, modes
        g, o = gsl.getMap().getAllSurfels(), osl.map.download()
        surfel_fields_equal(g, o, "surfels")  # (NaNs compare equal there, whatever their payload)
        for f in ("r", "g", "b"):  # lanes the update only carries: NaN payloads included, every bit survives
            assert np.array_equal(g[f].view(np.uint32), o[f].view(np.uint32)), f
        assert (g["b"].view(np.uint32) == 0x7fc12345).any()
    finally:
        gsl.ctx.close()


def _hidden_block(n, x0, x1, y0, y1, seed):
    """n stable surfels at z = -60 over [x0, x1] x [y0, y1]: below the field of view of every pose used here"""
    rng = np.random.default_rng(seed)
    s = np.zeros(n, O.SURFEL_DTYPE)
    s["x"] = rng.uniform(x0, x1, n)
    s["y"] = rng.uniform(y0, y1, n)
    s["z"] = -60.0
    s["nz"] = 1.0
    s["radius"] = 0.2
    s["confidence"] = 10.0
    s["weight"] = 1.0
    s["color"] = np.float32(0.5)
    return s


def _set_current_pose(osl, gsl, x):
    """SurfelMapping::setCurrentPose on both: the library's call, and the oracle's currentPose member"""
    import ctypes as C
    P = np.eye(4)
    P[0, 3] = x
    gsl.setCurrentPose(P)
    f = O.lib().orc_slam_pose_member
    f.restype, f.argtypes = C.POINTER(C.c_double), [C.c_void_p, C.c_int]
    dst = f(osl.h, 0)
    for i, v in enumerate(P.T.reshape(-1)):  # column-major
        dst[i] = v


def test_reinserted_tiles_use_the_room_of_the_dead_slots():
    """(f) paging near the capacity while dead slots exist. Tiles of 6 m, partial_extraction = 0; a map uploaded 250 000
    surfels below the capacity, with 1 000 surfels in tile (-1, -1) and 300 000 in tile (-1, 0). Moving the pose to x = 4
    extracts column -1, and the in-place updates that follow leave its surfels behind as dead slots; moving back re-inserts
    (-1, -1), which fits behind the physical end, and then (-1, 0), which fits only after a compaction -- of the map
    including the tile just re-inserted."""
    po, pp = both_params(**sized(900, submap_extent=3.0, submap_dimension=1, partial_extraction=0))
    scene = synth.Scene(width=900, height=64)
    home = synth.trajectory(1)[0]
    sc = [scene.scan(i, home) for i in range(8)]
    a1 = _hidden_block(1000, -8.5, -3.5, -8.5, -3.5, 21)
    a2 = _hidden_block(300_000, -8.5, -3.5, -2.5, 2.5, 22)
    fill = _hidden_block(MAX_SURFELS - 250_000 - a1.size - a2.size, -2.5, 2.5, -2.5, 2.5, 23)
    s = np.concatenate([a1, a2, fill])
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    try:
        osl.map.upload(s, 0)
        gsl.getMap().upload(s, 0)
        modes, launches = [], []
        for part, x in ((sc[0:3], None), (sc[3:6], 4.0), (sc[6:8], 0.0)):
            if x is not None:
                _set_current_pose(osl, gsl, x)
            modes += lockstep(osl, gsl, part, "x=%s" % x, launches=launches)
            assert gsl.getMap().submap_origin() == osl.map.submap_origin()
        assert modes[1:] == ["lazy"] * 7, modes  # dead slots are never compacted away by a dense update here
        ext = [d.get("extract_flags", 0) for d in launches]
        assert ext[3] == 3, ext  # column -1 leaves
        assert ext[6] == 4, ext  # column 2 leaves, column -1 comes back: one compaction
        assert osl.map.size() > MAX_SURFELS - 250_000, osl.map.size()
        surfel_fields_equal(gsl.getMap().getAllSurfels(), osl.map.download(), "surfels after re-insertion")
    finally:
        gsl.ctx.close()
