"""The managed submap tile cache (sb_set_tile_cache) against the oracle, whose tile cache is host RAM without a bound
(oracle/orc_map.c), bit for bit: pool reclaim, eviction to the host tier and re-insertion from it, the cut when both
tiers are full, record slot reuse, whole sb_process_scan runs, checkpoints and the KITTI runner."""
import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api, run_kitti, synth
from helpers import assert_bits_equal, both_params, sized, surfel_fields_equal
from test_gpu_paging import EXTRACT_CAP, POOL_CAP, Pair, pose_at, tile_surfels

pytestmark = pytest.mark.gpu
INF = float("inf")


def cusim(request):
    return getattr(request.config, "_cusim", False)


@pytest.fixture
def pair():
    made = []

    def make(pool, host, **kw):
        p = Pair(**kw)
        p.ctx.set_tile_cache(pool, host)
        made.append(p)
        return p

    yield make
    for p in made:
        p.ctx.close()


def test_reclaim_keeps_a_tile_that_cycles_through_more_than_the_pool(pair, request):
    """test_pool_exhaustion_... in a managed context with the full pool and no host tier: the 500 000-surfel tile leaves
    and comes back until more than 16 M surfels have been extracted; reclaims keep the pool from filling up"""
    if cusim(request):
        pytest.skip("passes 16 M surfels through the pool: too slow for the CPU executor (the small-pool cases below "
                    "reclaim there)")
    p = pair(POOL_CAP, 0, partial_extraction=0)
    p.upload(tile_surfels(EXTRACT_CAP, -4, 0, 5))
    cycles = POOL_CAP // EXTRACT_CAP + 2
    for k in range(cycles):
        for x in (12, 12, -12):
            p.update(x, check=False)
        assert p.gm.size() == p.om.size() == EXTRACT_CAP, "cycle %d" % k
        if k % 8 == 0 or k == cycles - 1:
            p.check("cycle %d" % k)
    info = p.ctx.tile_cache_info()
    assert p.dropped()[0] == 0 and info["dropped"] == 0
    assert info["reclaims"] > 0 and info["host_used"] == 0 and info["evictions"] == 0, info


def test_reclaim_in_a_small_pool(pair):
    """pool at its minimum and no host tier: every extraction after the first compacts the pool; a tile that comes back
    again and again is never cut"""
    p = pair(EXTRACT_CAP, 0, partial_extraction=0)
    p.upload(np.concatenate([tile_surfels(150_000, -4, 0, 6), tile_surfels(3000, -4, 2, 7)]))
    for k in range(4):
        for x in (12, 12, -12):
            p.update(x)
    info = p.ctx.tile_cache_info()
    assert p.dropped()[0] == 0
    assert info["reclaims"] > 0 and info["pool_used"] == info["pool_referenced"] <= EXTRACT_CAP, info


# rows and columns of tiles outside the start window: column tiles leave on the walk in x, row tiles on the walk in y
COLUMN_TILES = [(i, j) for i in (-4, -3, -2) for j in (-1, 0, 1)]
ROW_TILES = [(i, j) for i in (0, 1, 2) for j in (-4, -3)]
# poses: out in +x (columns -4..-2 leave), out in +y (rows -4, -3 leave), back in y and x (all come back), on to -x and
# back again (the tiles of column 4 and beyond are empty)
WALK = ([(x, 0) for x in (12, 12, 32, 32, 52, 52, 52)] + [(52, y) for y in (12, 12, 32, 32, 32)] +
        [(52, y) for y in (12, 12, -12, -12)] + [(x, -12) for x in (32, 32, 12, 12, -12, -12, -32, -32)] +
        [(x, 0) for x in (-12, -12, 12, 12, 32, 32)])


@pytest.mark.parametrize("partial", [0, 1], ids=["whole", "partial"])
def test_spill_and_fill(pair, partial):
    """tiles holding about twice the pool leave; the window walks back over them in rows and columns, both directions:
    tiles go to the host tier and come back from it, and the map equals the oracle's after every update"""
    p = pair(EXTRACT_CAP, INF, partial_extraction=partial)
    n = 60_000
    p.upload(np.concatenate([tile_surfels(n, i, j, 100 + k) for k, (i, j) in enumerate(COLUMN_TILES + ROW_TILES)]))
    for t, (x, y) in enumerate(WALK):
        while True:  # (partial extraction: one tile per update; stay until the queue is empty)
            p.om.update(pose_at(x, y), p.ov)
            p.gm.update(pose_at(x, y), p.f)
            p.check("t=%d (%g, %g)" % (t, x, y))
            if p.om.submap_origin()[2] == 0:
                break
    info = p.ctx.tile_cache_info()
    assert p.dropped()[0] == 0 and info["dropped"] == 0
    assert info["evictions"] > 0 and info["host_fills"] > 0 and info["reclaims"] > 0, info


def test_both_tiers_full_cut_the_extraction_with_the_default_rule(pair):
    """pool 500 000 and a host tier of 350 000: the first 300 000-surfel tile goes to the host, the second stays in the
    pool, the third finds both full and keeps the 200 000 that fit; the rest is counted and reported"""
    p = pair(EXTRACT_CAP, 350_000, partial_extraction=0)
    n = 300_000
    p.upload(np.concatenate([tile_surfels(n, i, 0, 40 + i) for i in (-4, -3, -2)]))
    for x in (12, 12, 32, 32, 52):
        p.update(x)
    p.update(52, check=False)
    assert p.gm.size() == p.om.size() == 0
    stored = EXTRACT_CAP - n
    dropped, err = p.dropped()
    assert dropped == n - stored
    assert "submap tile pool exhausted: %d surfels" % dropped in err, err
    info = p.ctx.tile_cache_info()
    assert info["dropped"] == dropped and info["host_used"] == n and info["tiles_on_host"] == 1, info
    p.update(32, check=False)  # column -2 comes back: the stored part, the oracle's prefix
    om = p.om.download()
    surfel_fields_equal(p.gm.getAllSurfels(), om[:stored], "the stored part of the cut tile")
    p.update(12, check=False)  # column -3 from the pool
    p.update(-12, check=False)  # column -4 from the host tier
    om = p.om.download()
    gm = p.gm.getAllSurfels()
    assert gm.shape[0] == om.shape[0] - (n - stored)
    surfel_fields_equal(gm[:stored], om[:stored], "cut tile")
    surfel_fields_equal(gm[stored:], om[n:], "the tiles behind it")
    assert p.ctx.tile_cache_info()["host_fills"] == 1


def test_record_slots_are_reused(pair):
    """submap-dimension 1 on a tiny map walking back and forth: more than 16 384 extractions (three per shift), which
    the default cache refuses with SB_ERR_CAPACITY"""
    p = pair(EXTRACT_CAP, INF, partial_extraction=0, submap_dimension=1)
    p.upload(np.concatenate([tile_surfels(40, -1, 0, 50), tile_surfels(30, 2, 1, 51), tile_surfels(20, 0, 0, 52)]))
    shifts = 16384 // 3 + 20
    for k in range(shifts):
        x = 12 if k % 2 == 0 else -12
        p.om.update(pose_at(x), p.ov)
        p.gm.update(pose_at(x), p.f)
        if k % 1000 == 0:
            p.check("shift %d" % k)
    p.check("after %d shifts" % shifts)
    info = p.ctx.tile_cache_info()
    assert info["reclaims"] > 0 and info["dropped"] == 0, info


# ---- whole sb_process_scan runs: out and back along a line, so that tiles leave and come back
def walk_scans(width, semantic, n_out=16):
    scene = synth.Scene(width=width, height=64, semantic=semantic)
    out = synth.trajectory(n_out, step=1.0, yaw_deg=0.0)
    poses = list(out) + list(out[-2::-1])
    return [scene.scan(f, P) for f, P in enumerate(poses)]


def managed_slam(pp, pool=EXTRACT_CAP, host=INF, loop=None):
    g = api.SurfelMapping(pp)
    g.setTileCache(pool, host)
    if loop:
        g.enableLoopClosure(True, **loop)
    return g


def stats_of(g):
    st = np.zeros(16)
    api.lib().sb_get_statistics(g.ctx.h, api._dp(st))
    return st


def compare_with_oracle(g, osl, what):
    assert_bits_equal(g.getCurrentPose(), osl.pose(), what + " pose")
    surfel_fields_equal(g.getMap().getAllSurfels(), osl.map.download(), what + " surfels")
    assert g.getMap().submap_origin() == osl.map.submap_origin(), what + " submap origin / pending"


PIPE = dict(submap_extent=3.0, submap_dimension=1)


@pytest.mark.parametrize("width,semantic", [(900, False), (900, True), (2048, False), (2048, True)],
                         ids=["900", "900-semantic", "2048", "2048-semantic"])
def test_process_scan_with_a_small_pool_equals_the_oracle(width, semantic, request):
    if cusim(request) and width == 2048:
        pytest.skip("the 64x900 runs cover the CPU executor")
    po, pp = both_params(**sized(width, **PIPE))
    sc = walk_scans(width, semantic)
    g, osl = managed_slam(pp), O.Slam(po)
    try:
        for t, s in enumerate(sc):
            g.processScan(*s)
            osl.process_scan(*s)
            compare_with_oracle(g, osl, "t=%d" % t)
            st = stats_of(g)
            assert st[12] == 0 and st[7] == osl.map.size(), "t=%d statistics" % t
        info = g.tile_cache_info()
        assert info["reclaims"] > 0 and info["evictions"] > 0 and info["host_fills"] > 0, info
    finally:
        g.ctx.close()


def test_process_scan_with_loop_closure_and_paging():
    """the synthetic loop of the checkpoint tests with loop closure on and tiles paged through a managed cache at its
    smallest pool: poses, loop state and surfels equal those of a default-cache run after every scan; an optimisation
    request, where the sequence raises one, is integrated in both"""
    _, pp = both_params(**sized(900, submap_extent=4.0, submap_dimension=1))
    scene = synth.Scene(width=900, height=64)
    poses = synth.trajectory(124, step=0.2618, yaw_deg=3.0)
    lp = dict(search_distance=3.0, min_trajectory_distance=15.0, min_verifications=2)
    g, d = managed_slam(pp, loop=lp), api.SurfelMapping(pp)
    d.enableLoopClosure(True, **lp)
    try:
        for f in range(124):
            s = scene.scan(f, poses[f])
            for e in (g, d):
                e.processScan(*s)
            assert_bits_equal(g.getCurrentPose(), d.getCurrentPose(), "t=%d pose" % f)
            li, ld = g.getLoopInfo(), d.getLoopInfo()
            for k in ("loop_count", "candidates_tested", "unverified", "optimisation_requested"):
                assert li[k] == ld[k], "t=%d loop info %s" % (f, k)
            if li["optimisation_requested"]:
                assert g.integrateLoopClosures() == d.integrateLoopClosures() > 0
            if f % 8 == 0:
                surfel_fields_equal(g.getMap().getAllSurfels(), d.getMap().getAllSurfels(), "t=%d surfels" % f)
        surfel_fields_equal(g.getMap().getAllSurfels(), d.getMap().getAllSurfels(), "surfels")
        info = g.tile_cache_info()
        assert info["evictions"] > 0 and info["reclaims"] > 0, info
    finally:
        g.ctx.close()
        d.ctx.close()


def _section(blob, sid):
    off = 280
    while off < len(blob) - 8:
        i, n = int(np.frombuffer(blob, np.uint32, 1, off)[0]), int(np.frombuffer(blob, np.uint64, 1, off + 8)[0])
        if i == sid:
            return off + 16
        off += 16 + n
    return None


S_TCACHE = 9


def test_checkpoint_with_tiles_in_both_tiers_and_a_pending_extraction():
    """save where tiles sit in the pool and on the host and an extraction is pending, load into a fresh context and go
    on: bit-exact against the uninterrupted run; save(load(save(x))) == save(x); a host tier over its saved capacity and
    a default context's checkpoint"""
    po, pp = both_params(**sized(900, partial_extraction=1, **PIPE))
    sc = walk_scans(900, False)
    g = managed_slam(pp)
    blob, n_done, obs = None, 0, {}
    try:
        for t, s in enumerate(sc):
            g.processScan(*s)
            info = g.tile_cache_info()
            if (blob is None and info["tiles_on_host"] > 0 and info["tiles_in_pool"] > 0 and
                    g.getMap().submap_origin()[2] > 0):
                blob, n_done = g.save_state(), t + 1
            if blob is not None:
                obs[t + 1] = (g.getCurrentPose(), g.getMap().getAllSurfels(), stats_of(g), info)
    finally:
        g.ctx.close()
    assert blob is not None, "the run must pass a scan with both tiers used and an extraction pending"
    assert _section(blob, S_TCACHE) is not None
    r = managed_slam(pp)  # (the checkpoint's cache replaces the setting)
    try:
        r.load_state(blob)
        assert r.save_state() == blob, "save(load(save(x))) != save(x)"
        for t in range(n_done, len(sc)):
            r.processScan(*sc[t])
            pose, surf, st, info = obs[t + 1]
            assert_bits_equal(r.getCurrentPose(), pose, "t=%d pose" % t)
            surfel_fields_equal(r.getMap().getAllSurfels(), surf, "t=%d surfels" % t)
            st2 = stats_of(r)
            st[8:12] = st2[8:12] = 0
            assert_bits_equal(st2, st, "t=%d statistics" % t)
            assert r.tile_cache_info() == info, "t=%d cache counters" % t
    finally:
        r.ctx.close()
    # host_used (the 3rd u64 after pool_cap, count) raised past host_cap: refused before anything changes
    off = _section(blob, S_TCACHE)
    bad = bytearray(blob)
    host_cap = int(np.frombuffer(blob, np.uint64, 1, off + 8)[0])
    assert host_cap == 2**64 - 1
    bad[off + 8:off + 16] = np.array([0], np.uint64).tobytes()  # capacity 0 with tiles on the host
    d = api.SurfelMapping(pp)
    try:
        a = np.frombuffer(bytes(bad), np.uint8)
        rc = api.lib().sb_state_load(d.ctx.h, api._vp(a), a.size)
        assert rc == -1 and "host tier beyond its capacity" in api.lib().sb_last_error(d.ctx.h).decode()
        # a default context's checkpoint makes a managed context default again
        d.processScan(*sc[0])
        plain = d.save_state()
        assert _section(plain, S_TCACHE) is None
        m = managed_slam(pp)
        m.load_state(plain)
        assert m.tile_cache_info()["managed"] == 0 and m.save_state() == plain
        m.ctx.close()
    finally:
        d.ctx.close()


def test_set_tile_cache_arguments_and_state():
    _, pp = both_params(**sized(128, 16))
    g = api.SurfelMapping(pp)
    try:
        with pytest.raises(api.SumaError, match="pool_surfels"):
            g.setTileCache(EXTRACT_CAP - 1, 0)
        with pytest.raises(api.SumaError, match="pool_surfels"):
            g.setTileCache(POOL_CAP + 1, 0)
        assert g.tile_cache_info()["managed"] == 0
        g.setTileCache(EXTRACT_CAP, 1000)
        info = g.tile_cache_info()
        assert (info["managed"], info["pool_capacity"], info["host_capacity"]) == (1, EXTRACT_CAP, 1000)
        m = g.getMap()
        m.upload(tile_surfels(100, -4, 0, 1), 1)
        f = api.Frame(g.ctx, 128, 16)
        m.update(pose_at(12), f)  # extracts column -4
        with pytest.raises(api.SumaError, match="not empty"):
            g.setTileCache(EXTRACT_CAP, 0)
        g.reset()  # the setting is kept, the tiers are emptied
        info = g.tile_cache_info()
        assert (info["managed"], info["pool_capacity"], info["tiles_in_pool"], info["pool_used"]) == (1, EXTRACT_CAP, 0, 0)
        g.setTileCache(POOL_CAP, 0)
        del f
    finally:
        g.ctx.close()


class OracleEngine:
    """the oracle behind run_kitti's engine surface"""

    def __init__(self, params):
        d = params.as_dict()
        self.s = O.Slam(O.default_params(**{k: v for k, v in d.items()}))

    def processScan(self, pts, labels, probs):
        self.s.process_scan(pts, labels, probs)

    def getCurrentPose(self):
        return self.s.pose()


def test_run_kitti_tile_cache_host_equals_the_oracle_and_resumes(tmp_path, capsys):
    seq = str(tmp_path / "seq")
    run_kitti.make_synthetic_sequence(seq, 12, width=900)

    def small(params):
        params.submap_extent, params.submap_dimension = 3.0, 1
        return params

    cuda = lambda p: api.SurfelMapping(small(p))  # noqa: E731
    oracle = lambda p: OracleEngine(small(p))  # noqa: E731
    common = [seq, "--width", "900"]
    ours, ref, resumed = (str(tmp_path / n) for n in ("ours.txt", "ref.txt", "resumed.txt"))
    state = str(tmp_path / "state.bin")
    assert run_kitti.main(common + ["--out", ref], make_engine=oracle) == 0
    capsys.readouterr()
    assert run_kitti.main(common + ["--out", ours, "--tile-cache-host", "inf"], make_engine=cuda) == 0
    report = capsys.readouterr().out
    assert '"tile_cache"' in report and '"managed": 1' in report, report
    assert open(ours, "rb").read() == open(ref, "rb").read()
    assert run_kitti.main(common + ["--max-scans", "7", "--save-state", state, "--tile-cache-host", "inf"],
                          make_engine=cuda) == 0
    assert run_kitti.main(common + ["--resume", state, "--out", resumed, "--tile-cache-host", "inf"],
                          make_engine=cuda) == 0
    assert open(resumed, "rb").read() == open(ref, "rb").read()
