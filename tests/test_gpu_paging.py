"""Submap paging (SurfelMap::updateActiveSubmaps, SurfelMap.cpp:744-824) on the CUDA path against the oracle: several tiles
extracted in one update, the 500 000-surfel cap of one tile, an empty map, and the device's own limit, the 16 M-surfel
HBM tile pool (the reference caches tiles in host RAM without a bound)."""
import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api
from helpers import both_params, scans, sized, surfel_fields_equal

pytestmark = pytest.mark.gpu

EXTRACT_CAP = 500_000        # surfels of one extracted tile (SurfelMap.cpp:279)
POOL_CAP = 16 * 1024 * 1024  # surfels held by the HBM tile cache


def pose_at(x, y=0.0):
    T = np.eye(4, dtype=np.float32)
    T[0, 3], T[1, 3] = x, y
    return T


def tile_surfels(n, i, j, seed, extent=10.0):
    """n surfels created at time 0 (identity pose) inside submap tile (i, j), confident enough to survive updates
    that measure nothing"""
    rng = np.random.default_rng(seed)
    s = np.zeros(n, O.SURFEL_DTYPE)
    s["x"] = 2 * extent * i + rng.uniform(-0.8 * extent, 0.8 * extent, n)
    s["y"] = 2 * extent * j + rng.uniform(-0.8 * extent, 0.8 * extent, n)
    s["z"] = rng.uniform(-1.0, 2.0, n)
    s["nz"] = 1.0
    s["radius"] = rng.uniform(0.05, 0.5, n)
    s["confidence"] = 10.0
    s["weight"] = 1.0
    return s


class Pair:
    """the oracle's map and the library's, updated in lockstep with frames that measure nothing (no surfel is generated
    or fused, so only paging moves surfels)"""

    def __init__(self, **kw):
        self.po, pp = both_params(**sized(128, 16, **kw))
        self.ctx = api.Context(pp)
        self.om, self.gm = O.Map(self.po), api.SurfelMap(self.ctx)
        self.f = api.Frame(self.ctx, 128, 16)
        self.ov = [np.zeros((16, 128, 4), np.float32) for _ in range(3)]

    def upload(self, s, t=1):
        self.om.upload(s, t)
        self.gm.upload(s, t)

    def update(self, x, check=True):
        self.om.update(pose_at(x), self.ov)
        self.gm.update(pose_at(x), self.f)
        if check:
            self.check("x=%g" % x)

    def check(self, what):
        assert self.gm.submap_origin() == self.om.submap_origin(), "%s: submap origin / pending" % what
        assert self.gm.size() == self.om.size(), "%s: size %d vs %d" % (what, self.gm.size(), self.om.size())
        surfel_fields_equal(self.gm.getAllSurfels(), self.om.download(), what + " surfels")

    def dropped(self):
        st = np.zeros(16)
        api.lib().sb_get_statistics(self.ctx.h, api._dp(st))
        return int(st[12]), api.lib().sb_last_error(self.ctx.h).decode()


@pytest.fixture
def pair():
    made = []

    def make(**kw):
        made.append(Pair(**kw))
        return made[-1]

    yield make
    for p in made:
        p.ctx.close()


def test_several_tiles_per_update_shift_extract_and_reinsert():
    """partial_extraction = 0: every tile of a leaving column is extracted in the update that shifts the window, and the
    column comes back when the sensor returns. Map size, origin / pending count and every surfel after every update."""
    po, pp = both_params(**sized(900, partial_extraction=0))
    ctx = api.Context(pp)
    try:
        sc, _ = scans(900, n=3)
        omap, gmap = O.Map(po), api.SurfelMap(ctx)
        frames = []
        for s in sc:
            pts, lab, prb = s
            f = api.Frame(ctx, 900, 64)
            api.Preprocessing(ctx).process(pts, f, lab, prb, 100)
            frames.append((O.preprocess(po, pts, lab, prb, 100), f))
        xs = [0, 12, 24, 36, 48, 36, 24, 12, 0, -12]
        ys = [0, 0, 0, 12, 12, 12, 0, 0, 0, 0]
        origins = set()
        for t, (x, y) in enumerate(zip(xs, ys)):
            ov, f = frames[t % 3]
            omap.update(pose_at(x, y), ov)
            gmap.update(pose_at(x, y), f)
            assert gmap.submap_origin() == omap.submap_origin(), "t=%d submap origin / pending" % t
            assert gmap.submap_origin()[2] == 0, "t=%d: tiles left pending" % t
            assert gmap.size() == omap.size(), "t=%d size %d vs %d" % (t, gmap.size(), omap.size())
            surfel_fields_equal(gmap.getAllSurfels(), omap.download(), "t=%d surfels" % t)
            origins.add(omap.submap_origin()[:2])
        assert len(origins) >= 4, origins
    finally:
        ctx.close()


def test_a_tile_over_the_extract_cap_comes_back_capped(pair):
    """550 000 surfels in tile (-4, 0): the shift to origin 1 extracts its column and the first 500 000 are cached
    (transform feedback drops the rest); the way back re-inserts those"""
    p = pair(partial_extraction=0)
    p.upload(np.concatenate([tile_surfels(550_000, -4, 0, 1), tile_surfels(2000, 0, 0, 2)]))
    p.update(12)  # origin 1: column -4 is extracted (the next update pass drops it from the map)
    p.update(12)
    assert p.om.size() == 2000
    p.update(-12)  # origin 0: column -4 comes back
    assert p.om.size() == 2000 + EXTRACT_CAP


def test_paging_an_empty_map(pair):
    """tiles extracted from an empty map are empty and re-inserting them adds nothing; their records carry the end of the
    pool's used range, so that the tiles extracted later land behind the earlier ones"""
    p = pair(partial_extraction=0)
    p.upload(tile_surfels(3000, -4, 1, 3))
    p.update(12)  # origin 1: column -4 goes to pool [0, 3000)
    p.update(12)
    assert p.gm.size() == 0
    p.update(32)  # origin 2: column -3 is extracted from the empty map
    p.update(12)  # origin 1: and comes back empty
    assert p.gm.size() == 0
    p.upload(tile_surfels(2000, -3, -2, 4), p.om.timestamp())
    p.update(-12)  # origin 0: column -4 comes back
    p.update(12)   # origin 1: column -4 goes to [3000, 6000), behind the empty tiles' records
    p.update(32)   # origin 2: column -3 goes to [6000, 8000)
    p.update(52)   # origin 3
    assert p.gm.size() == 0
    for x in (32, 12, -12):  # back to origin 0: columns -3 and -4 come back
        p.update(x)
    assert p.om.size() == 5000
    assert p.dropped()[0] == 0


def test_pool_exhaustion_keeps_the_stored_part_and_counts_the_rest(pair):
    """a full tile leaves and comes back again and again until the pool cannot hold it: the part that fit is re-inserted,
    the rest is counted in sb_get_statistics()[12] and reported by sb_last_error"""
    p = pair(partial_extraction=0)
    p.upload(tile_surfels(EXTRACT_CAP, -4, 0, 5))
    used = 0
    while used + EXTRACT_CAP <= POOL_CAP:  # every cycle caches the whole tile
        for x in (12, 12, -12):
            p.update(x, check=False)
        used += EXTRACT_CAP
        assert p.gm.size() == p.om.size() == EXTRACT_CAP
    assert p.dropped()[0] == 0
    p.check("before the pool is full")
    stored = POOL_CAP - used
    p.update(12)
    p.update(12)
    p.update(-12, check=False)
    assert p.gm.size() == stored and p.om.size() == EXTRACT_CAP
    surfel_fields_equal(p.gm.getAllSurfels(), p.om.download()[:stored], "the stored part of the tile")
    dropped, err = p.dropped()
    assert dropped == EXTRACT_CAP - stored
    assert "submap tile pool exhausted: %d surfels" % dropped in err, err
    for x in (12, 12, -12):  # the pool is full: the stored part is lost too
        p.gm.update(pose_at(x), p.f)
    assert p.gm.size() == 0
    assert p.dropped()[0] == EXTRACT_CAP
