"""The kernels that move surfels between slots, at their block, group, round and capacity boundaries: the ordered
compaction of k_extract_flags + k_compact (a tile leaving the active window, the map after the update pass drops it, and
a map with dead slots), the extraction cut at 500 000 surfels or at the pool's end, and the managed tile cache's reclaim
(k_pool_reclaim, moved through the scratch set in rounds of at most 4 194 304 surfels).

Every case runs the oracle's map and the library's in lockstep with frames that measure nothing (Pair of
test_gpu_paging.py), next to a plain numpy model of the map's slots and of the tile pool that shares no code with either:
the model holds the uploaded records in upload order, extracts a tile as records[mask] cut at the extract cap and at the
pool's end, and appends re-inserted tiles in the loop order of SurfelMap.cpp:769-780. Both compact sequentially, so a
comparison with them is exact and independent of the CUDA code's block and group arithmetic. The profiler's per-kernel
launch counts show that each case reached the regime it was built for."""
import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api, synth
from helpers import both_params, scans, sized, surfel_fields_equal
from test_gpu_paging import EXTRACT_CAP, POOL_CAP, Pair, pose_at

pytestmark = pytest.mark.gpu

MAX_SURFELS = 2048 * 2048  # map capacity, and the surfels one reclaim round moves at most
BLOCK = 256                # threads of a compaction block
GROUP = 64 * BLOCK         # surfels behind one group total
EXT = 10.0                 # default submap extent (tiles of 20 m)
DIM = 4                    # default submap dimension (a window of 9 x 9 tiles)
F = np.float32
# the colour the update pass gives a surfel it does not see, pack_rgb(0.3, 0.3, 0.3): with it, such an update leaves
# every bit of the record as it was
UNSEEN_COLOR = np.array([0x4a9a9a9a], np.uint32).view(np.float32)[0]


def cusim(request):
    return getattr(request.config, "_cusim", False)


def surfels_at(tiles, seed):
    """one surfel per row of `tiles` (tile indices (i, j)), inside that tile, created at time 0 (identity pose) and
    confident enough to survive updates that measure nothing; field r holds the surfel's upload slot"""
    tiles = np.asarray(tiles).reshape(-1, 2)
    n = tiles.shape[0]
    rng = np.random.default_rng(seed)
    s = np.zeros(n, O.SURFEL_DTYPE)
    s["x"] = 2 * EXT * tiles[:, 0] + rng.uniform(-0.8 * EXT, 0.8 * EXT, n)
    s["y"] = 2 * EXT * tiles[:, 1] + rng.uniform(-0.8 * EXT, 0.8 * EXT, n)
    s["z"] = rng.uniform(-1.0, 2.0, n)
    s["nz"] = 1.0
    s["radius"] = rng.uniform(0.05, 0.5, n)
    s["confidence"] = 10.0
    s["weight"] = 1.0
    s["color"] = UNSEEN_COLOR
    s["r"] = np.arange(n)
    return s


def same_records(a, b, what):
    """surfel_fields_equal, with the comparison of whole records first (the records here hold no NaN)"""
    if a.shape != b.shape or a.tobytes() != b.tobytes():
        surfel_fields_equal(a, b, what)


class SlotModel:
    """The map's slots and the submap tile pool as plain lists, for walks with partial_extraction = 0 whose surfels all
    carry the identity pose (entry 0 of the pose table), so that the fp32 tile predicate of extract_surfels.vert is exact.
    The pool is a list of copies [tile, size, live] in pool order; a managed cache reclaims it by the rule of
    DESIGN.md section 10 (an upper bound of the used end that grows by a whole tile per extraction, read back and
    reclaimed when a whole tile might not fit)."""

    def __init__(self, pool_cap=POOL_CAP, managed=False):
        self.map = np.zeros(0, O.SURFEL_DTYPE)
        self.oi = self.oj = 0
        self.cache = {}
        self.pool = []
        self.pool_cap, self.managed = pool_cap, managed
        self.bound = self.known = 0
        self.reclaims = self.moved = self.dropped = self.reclaim_launches = 0
        self.last_reclaim = None

    @staticmethod
    def center(i):  # submapIndex2center, in fp32 from the double product
        return F(2.0 * i * EXT)

    @classmethod
    def inside(cls, s, ci, cj, e):  # !(|x - cx| > e || |y - cy| > e)
        return ~((np.abs(s["x"] - cls.center(ci)) > e) | (np.abs(s["y"] - cls.center(cj)) > e))

    def in_tile(self, s, t):
        return self.inside(s, t[0], t[1], F(EXT))

    def upload(self, s):
        self.map = s.copy()

    def end(self):
        return sum(c[1] for c in self.pool)

    def info(self):
        return dict(tiles_in_pool=sum(c[2] for c in self.pool), pool_used=self.end(),
                    pool_referenced=sum(c[1] for c in self.pool if c[2]), reclaims=self.reclaims,
                    reclaim_moved=self.moved, dropped=self.dropped)

    def update(self, x, y=0.0):
        # the update pass keeps the active window
        e = F(F(2.0 * DIM) * F(EXT)) + F(EXT)
        self.map = self.map[self.inside(self.map, self.oi, self.oj, e)]
        # paging, SurfelMap.cpp:744-824: both shifts are measured from the old centre; every leaving tile is extracted
        thr = F(1.1) * F(EXT)
        chx, chy = F(x) - self.center(self.oi), F(y) - self.center(self.oj)
        leaving = []
        if abs(chx) > thr:
            d = -1 if chx < 0 else 1
            leaving += [(self.oi - d * DIM, self.oj + k) for k in range(-DIM, DIM + 1)]
            self.oi += d
            self.append([(self.oi + d * DIM, self.oj + k) for k in range(-DIM, DIM + 1)])
        if abs(chy) > thr:
            d = -1 if chy < 0 else 1
            leaving += [(self.oi + k, self.oj - d * DIM) for k in range(-DIM, DIM + 1)]
            self.oj += d
            self.append([(self.oi + k, self.oj + d * DIM) for k in range(-DIM, DIM + 1)])
        for t in reversed(leaving):  # the extraction queue is taken from its back
            self.extract(t)

    def refresh(self):  # the records are read back: the bound becomes the used end
        self.bound, self.known = self.end(), len(self.pool)

    def append(self, tiles):
        for t in tiles:
            if any(c[0] == t and c[2] for c in self.pool[self.known:]):  # a tile whose record is not read back yet
                self.refresh()
            if t in self.cache:
                room = MAX_SURFELS - self.map.shape[0]
                self.map = np.concatenate([self.map, self.cache[t][:room]])

    def extract(self, t):
        for c in self.pool:  # the tile's earlier copy is abandoned
            if c[0] == t:
                c[2] = False
        if self.managed:
            if self.bound + EXTRACT_CAP > self.pool_cap:  # read back, then reclaim (no host tier to evict to)
                self.refresh()
                self.reclaim()
            self.bound += EXTRACT_CAP
        recs = self.map[self.in_tile(self.map, t)]
        want = min(recs.shape[0], EXTRACT_CAP)
        n = max(0, min(want, self.pool_cap - self.end()))
        self.dropped += want - n
        self.cache[t] = recs[:n].copy()
        self.pool.append([t, n, True])

    def reclaim(self):
        if all(c[2] for c in self.pool):
            return
        runs, src, dst = [], 0, 0  # [source, destination, surfels] of the moves, adjacent tiles merged
        for t, n, live in self.pool:
            if live:
                if n and src != dst:
                    if runs and runs[-1][0] + runs[-1][2] == src and runs[-1][1] + runs[-1][2] == dst:
                        runs[-1][2] += n
                    else:
                        runs.append([src, dst, n])
                dst += n
            src += n
        moved = sum(r[2] for r in runs)
        self.last_reclaim = dict(runs=runs, moved=moved, rounds=-(-moved // MAX_SURFELS))
        self.pool = [c for c in self.pool if c[2]]
        self.bound, self.known = dst, len(self.pool)
        self.reclaims += 1
        self.moved += moved
        self.reclaim_launches += 2 * self.last_reclaim["rounds"]  # gather into the scratch set, write back


class Moves:
    """a Pair (oracle map + library map) and the slot model, stepped together and compared after every step"""

    def __init__(self, pool=None, host=0, **kw):
        self.p = Pair(partial_extraction=0, **kw)
        if pool is not None:
            self.p.ctx.set_tile_cache(pool, host)
        self.model = SlotModel(POOL_CAP if pool is None else pool, managed=pool is not None)
        self.p.ctx.profile(True)
        self.p.ctx.profile_collect()

    def upload(self, s):
        # (timestamp >= 1: the first update then sets pose entry 1, and entry 0 stays the identity the surfels use)
        self.p.upload(s, max(1, self.p.om.timestamp()))
        self.model.upload(s)

    def step(self, x, y=0.0, upload=None, oracle=True):
        """an upload (if given) and one update at (x, y) on all three, compared; the launches of the moving kernels"""
        if upload is not None:
            self.upload(upload)
        launches = self.model.reclaim_launches
        self.p.om.update(pose_at(x, y), self.p.ov)
        self.p.gm.update(pose_at(x, y), self.p.f)
        self.model.update(x, y)
        c = self.launches()
        assert c["pool_reclaim"] == self.model.reclaim_launches - launches, c
        self.check("(%g, %g)" % (x, y), oracle)
        return c

    def launches(self):
        prof = self.p.ctx.profile_collect()
        return {k: prof.get(k, (0, 0))[1] for k in ("extract_flags", "compact_scatter", "pool_reclaim")}

    def check(self, what, oracle=True):
        """(oracle = False: a cache that cut a tile, which the oracle's unbounded host-side cache never does)"""
        m = self.model
        assert self.p.om.submap_origin() == (m.oi, m.oj, 0), what + ": oracle origin"
        assert self.p.gm.submap_origin() == (m.oi, m.oj, 0), what + ": library origin"
        g = self.p.gm.getAllSurfels()
        if oracle:
            same_records(g, self.p.om.download(), what + ": library vs oracle")
        same_records(g, m.map, what + ": library vs slot model")
        info = self.p.ctx.tile_cache_info()
        for k, v in m.info().items():
            assert info[k] == v, "%s: tile_cache_info %s = %d, the model has %d" % (what, k, info[k], v)


@pytest.fixture
def moves():
    made = []

    def make(**kw):
        made.append(Moves(**kw))
        return made[-1]

    yield make
    for m in made:
        m.p.ctx.close()


# ---- 1. ordered extraction under chosen masks
SIZES = [1, 31, 32, 33, 255, 256, 257, GROUP - 1, GROUP, GROUP + 1, 2 * GROUP - 1, 2 * GROUP + 1,
         MAX_SURFELS - 1, MAX_SURFELS]
PATTERNS = ["none", "all", "alternating", "lane0", "lane31", "block_first", "block_last", "group_last", "slot0",
            "slot_last", "random1e-4", "random0.5", "random0.9999"]


def pattern(name, n):
    k = np.arange(n)
    if name.startswith("random"):
        return np.random.default_rng(n).random(n) < float(name[6:])
    return {"none": k < 0, "all": k >= 0, "alternating": k % 2 == 1, "lane0": k % 32 == 0, "lane31": k % 32 == 31,
            "block_first": k % BLOCK == 0, "block_last": k % BLOCK == BLOCK - 1, "group_last": k % GROUP == GROUP - 1,
            "slot0": k == 0, "slot_last": k == n - 1}[name]


def shift_out_and_back(m, n_tile, n_rest):
    """origin 0 -> 1 (column -4 is extracted from the whole map), the next update pass drops the column, origin 1 -> 0
    (the column comes back behind the rest and column 5 is extracted); the launches of each step"""
    c1 = m.step(12)
    assert c1 == {"extract_flags": 9 if n_tile + n_rest else 0, "compact_scatter": 10, "pool_reclaim": 0}, c1
    c2 = m.step(12)
    assert c2 == {"extract_flags": 0, "compact_scatter": 1, "pool_reclaim": 0}, c2
    assert m.model.map.shape[0] == n_rest
    c3 = m.step(-12)
    back = min(n_tile, EXTRACT_CAP)
    assert c3 == {"extract_flags": 9 if back + n_rest else 0, "compact_scatter": 10, "pool_reclaim": 0}, c3
    assert m.model.map.shape[0] == n_rest + back


@pytest.mark.parametrize("name", PATTERNS)
@pytest.mark.parametrize("n", SIZES)
def test_ordered_extraction_under_a_mask(moves, n, name, request):
    """the surfels of the pattern lie in tile (-4, 0), which leaves the window, the others in tile (0, 0), which stays:
    the pool copy and the map after the update pass are both compactions under the mask, at sizes around a warp, a
    block, one and two groups and the full capacity (whose last group, 255, sums 255 group totals)"""
    if n >= MAX_SURFELS - 1 and cusim(request):
        pytest.skip("a full-capacity map: too slow for the CPU executor (the one- and two-group sizes run there)")
    keep = pattern(name, n)
    tiles = np.zeros((n, 2), np.int64)
    tiles[keep, 0] = -4
    s = surfels_at(tiles, n)
    m = moves()
    assert np.array_equal(m.model.in_tile(s, (-4, 0)), keep), "the model's tile predicate must give the pattern"
    m.upload(s)
    shift_out_and_back(m, int(keep.sum()), n - int(keep.sum()))
    # (the model's map: the kept surfels in slot order, then the tile's first 500 000 in slot order)
    assert np.array_equal(m.model.map["r"], np.concatenate([np.flatnonzero(~keep), np.flatnonzero(keep)[:EXTRACT_CAP]]))


# ---- 2. the extraction cut
@pytest.mark.parametrize("count", [EXTRACT_CAP - 1, EXTRACT_CAP, EXTRACT_CAP + 1])
def test_the_extract_cap_keeps_the_first_surfels_in_map_order(moves, count):
    """a tile of count surfels spread at random through a map with 200 000 that stay: the pool holds the first 500 000
    of the tile in map order (the cap is not a drop), the remaining map is unchanged"""
    n = count + 200_000
    keep = np.zeros(n, bool)
    keep[np.random.default_rng(count).choice(n, count, replace=False)] = True
    tiles = np.zeros((n, 2), np.int64)
    tiles[keep, 0] = -4
    s = surfels_at(tiles, count)
    m = moves()
    m.upload(s)
    shift_out_and_back(m, count, n - count)
    assert m.model.cache[(-4, 0)].shape[0] == min(count, EXTRACT_CAP)
    assert m.p.dropped()[0] == 0 and m.model.dropped == 0


def test_a_managed_pool_short_of_room_cuts_the_tile_at_its_end(moves):
    """pool of 500 000 and no host tier: tile (-4, 1) takes 300 000, and tile (-4, 0), extracted next, finds 200 000
    of room (cap - base < the extract cap): it keeps its first 200 000 in map order and the rest is counted as dropped;
    both tiles are interleaved with each other and with a tile that stays"""
    n1, n0, stay = 300_000, 300_000, 100_000
    which = np.random.default_rng(7).permutation(np.repeat([1, 0, 2], [n1, n0, stay]))
    tiles = np.zeros((which.size, 2), np.int64)
    tiles[which < 2, 0] = -4
    tiles[which == 1, 1] = 1
    s = surfels_at(tiles, 8)
    m = moves(pool=EXTRACT_CAP, host=0)
    m.upload(s)
    c = m.step(12)
    assert c["extract_flags"] == 9 and m.p.ctx.tile_cache_info()["reclaims"] == 0, c
    assert m.model.cache[(-4, 1)].shape[0] == n1 and m.model.cache[(-4, 0)].shape[0] == EXTRACT_CAP - n1
    m.step(12)
    m.step(-12, oracle=False)  # (the oracle's cache is unbounded: it brings the whole tile back)
    o, g = m.p.om.download(), m.p.gm.getAllSurfels()
    cut = n0 - (EXTRACT_CAP - n1)
    surfel_fields_equal(g, np.concatenate([o[:stay + EXTRACT_CAP - n1], o[stay + n0:]]), "the oracle's map without the cut")
    dropped, err = m.p.dropped()
    assert dropped == m.model.dropped == cut
    assert "submap tile pool exhausted: %d surfels" % dropped in err, err


# ---- 5. group totals across passes
def test_passes_that_shrink_and_grow_across_groups_in_one_context(moves):
    """one context, maps of 3 groups + 5, a group - 3, 3 groups + 5 again, 2 groups, 1 surfel and 2 groups + 7, each
    with half its surfels in the leaving tile: no extraction or update pass reads the block or group totals of a pass
    over a larger map before it"""
    m = moves()
    for r, n in enumerate([3 * GROUP + 5, GROUP - 3, 3 * GROUP + 5, 2 * GROUP, 1, 2 * GROUP + 7]):
        keep = np.random.default_rng(100 + r).random(n) < 0.5
        tiles = np.zeros((n, 2), np.int64)
        tiles[keep, 0] = -4
        m.upload(surfels_at(tiles, 100 + r))
        shift_out_and_back(m, int(keep.sum()), n - int(keep.sum()))


# ---- 4. multi-round pool reclaim
def column(i, sizes, j0):
    """tile indices of a column: sizes[k] surfels in tile (i, j0 + k)"""
    return [(i, j0 + k) for k, n in enumerate(sizes) for _ in range(n)]


def row(j, sizes, i0):
    return [(i0 + k, j) for k, n in enumerate(sizes) for _ in range(n)]


B = EXTRACT_CAP


@pytest.mark.parametrize("moved", ["two_rounds", "one_full_round"])
def test_a_reclaim_that_moves_more_than_one_round(moves, moved, request):
    """Full 16 M pool, no host tier. The walk builds this pool, in pool order (each column is extracted from its last
    tile to its first):
      column -4 (oj 0): tiles with surfels and empty ones, never extracted again: the prefix that stays in place
      column -3 (oj 0): (-3, 0) 100 000 and (-3, -4) 400 000; (-3, 0) is extracted again later (a 100 000 hole right
                        behind the prefix), (-3, -4) lies outside the column then: it moves down 100 000 together with
      row -4    (oj 1): tiles (3..6, -4) with 500 000 each -- one run of 2.4 M whose destination overlaps its source
      column -2 (oj 1): (-2, 5) 300 000 and (-2, 1) 200 000, extracted again later: a hole between moved tiles
      column 7, column 6 (and the copies extracted again): the second run, across the round boundary at 4 194 304.
    The read-back before column -2's re-extraction leaves the bound so that the reclaim comes at its 8th tile, once both
    holes exist. one_full_round: column 6 holds less and column -4 more, so that exactly 4 194 304 surfels move: one
    round, ending at the round's last slot. Then the window walks back over every tile, compared with the oracle and
    the model at every step (in one_full_round the map reaches its capacity on the way, so some re-insertions are cut:
    the same cut in all three)."""
    if cusim(request):
        pytest.skip("a 16 M-surfel pool with more than 4 M surfels moved per reclaim: too slow for the CPU executor (the "
                    "small-pool reclaims of test_gpu_tile_cache.py run there)")
    m = moves(pool=POOL_CAP, host=0)
    c6 = [B] * 5 if moved == "two_rounds" else [B, MAX_SURFELS - 4_000_000]
    # column -4 takes what column 6 lacks: the used end is the same when column 6 leaves, and so is the tile at which
    # the bound reaches the pool's end
    extra = 4_000_000 - sum(c6)
    p = [300_000] + [B] * (extra // B) + [extra % B] + [0] * (6 - extra // B) + [200_000]
    steps = [((12, 0), column(-4, p, -4)),
             ((32, 0), column(-3, [400_000, 0, 0, 0, 100_000, 0, 0, 0, 0], -4)),
             ((40, 12), row(-4, [0, 0, 0, 0, 0, B, B, B, B], -2)),
             ((52, 20), column(-2, [0, 0, 0, 0, 200_000, 0, 0, 0, 300_000], -3)),
             ((32, 20), column(7, [B, B, 0, 0, 0, 0, 0, 0, 0], -3)),
             ((12, 20), column(6, c6 + [0] * (9 - len(c6)), -3)),
             ((32, 20), None),   # column -3 again: the hole at (-3, 0)
             ((52, 20), None)]   # column -2 again: the hole between moved tiles, and the reclaim
    for k, ((x, y), tiles) in enumerate(steps):
        c = m.step(x, y, upload=None if tiles is None else surfels_at(tiles, 200 + k))
        if k < len(steps) - 1:
            assert m.p.ctx.tile_cache_info()["reclaims"] == 0, "step %d: no reclaim before the last step" % k
    r = m.model.last_reclaim
    assert m.model.reclaims == 1 and r is not None
    runs = r["runs"]
    assert r["moved"] == m.p.ctx.tile_cache_info()["reclaim_moved"]
    assert runs[0][1] == sum(p) and runs[0][0] == runs[0][1] + 100_000, runs  # behind the prefix, over a small hole
    assert runs[0][2] > runs[0][0] - runs[0][1], "the first run overlaps its destination"
    assert len(runs) >= 2 and runs[1][0] - runs[1][1] > runs[0][0] - runs[0][1], "a second hole starts a second run"
    if moved == "two_rounds":
        assert r["rounds"] == 2 and c["pool_reclaim"] == 4, (r, c)
        assert runs[0][2] < MAX_SURFELS < runs[0][2] + runs[1][2], "a run crosses the round boundary"
    else:
        assert r["moved"] == MAX_SURFELS and r["rounds"] == 1 and c["pool_reclaim"] == 2, (r, c)
    info = m.p.ctx.tile_cache_info()
    assert info["pool_used"] == info["pool_referenced"] and info["dropped"] == 0, info
    # every tile comes back: to origin (0, 0), whose window holds columns -4..-2 and row -4, then to (3, 0) for 6 and 7
    for x, y in ((32, 20), (12, 20), (-8, 20), (0, 0), (12, 0), (32, 0), (52, 0)):
        m.step(x, y)


# ---- 3. compaction of a map with dead slots
def hidden_surfels(dies, seed, extent=60.0):
    """surfels below the field of view of every scan here (never rendered, matched or fused, kept by the submap
    window); those marked in `dies` are unconfident, and the first update after their upload removes them (the
    unstable-surfel rule)"""
    n = dies.size
    rng = np.random.default_rng(seed)
    s = np.zeros(n, O.SURFEL_DTYPE)
    s["x"] = rng.uniform(-extent, extent, n)
    s["y"] = rng.uniform(-extent, extent, n)
    s["z"] = -60.0
    s["nz"] = 1.0
    s["radius"] = 0.2
    s["confidence"] = np.where(dies, -1.0, 10.0)
    s["weight"] = 1.0
    s["color"] = UNSEEN_COLOR
    s["r"] = np.arange(n)
    return s


def scan_launches(gsl):
    """the moving kernels' launches since the last call; 'dense': the compactions of a dense update (every tile
    extraction and map compaction pairs one compact_scatter with an extract_flags)"""
    cnt = {k: v[1] for k, v in gsl.ctx.profile_collect().items()}
    c = {k: cnt.get(k, 0) for k in ("extract_flags", "compact_scatter", "update_surfels")}
    c["dense"] = c["compact_scatter"] - c["extract_flags"]
    return c


# patterns at 1/8 of the slots or more make the next scan dense; the sparse ones leave the map to a download
DEAD_ROUTES = [("alternating", "dense_scan"), ("random0.5", "dense_scan"), ("lane31", "download"),
               ("block_first", "download"), ("group_last", "download")]


@pytest.mark.parametrize("name,route", DEAD_ROUTES)
def test_compaction_of_dead_slots_across_map_sizes(name, route):
    """One context. Three times a map is uploaded, of 3 groups + 5, a group - 3 and again 3 groups + 5 hidden surfels
    (so the map shrinks and grows across group boundaries between passes), whose pattern's surfels are unstable: the in-place update of the next scan leaves them behind as dead slots. Then either the following scan
    runs dense (k_update_surfels<false> + k_compact) or a download compacts the map (k_extract_flags over the liveness
    bytes + k_compact). The map equals the oracle's, and its first surfels are the hidden ones that live, in slot
    order."""
    po, pp = both_params(**sized(900))
    sc, _ = scans(900, n=9)
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    t = 0
    try:
        gsl.ctx.profile(True)
        for r, n in enumerate([3 * GROUP + 5, GROUP - 3, 3 * GROUP + 5]):
            dies = pattern(name, n)
            s = hidden_surfels(dies, 300 + r)
            live = s[~dies]
            ts = osl.map.timestamp()
            osl.map.upload(s, ts)
            gsl.getMap().upload(s, ts)
            gsl.ctx.profile_collect()
            for k in range(2 if route == "dense_scan" else 1):
                osl.process_scan(*sc[t])
                gsl.processScan(*sc[t])
                t += 1
                c = scan_launches(gsl)
                assert gsl.getMap().size() == osl.map.size(), "round %d scan %d" % (r, k)
                if k == 0:
                    assert c["dense"] == 0 and c["update_surfels"] == 1, "round %d: in place first: %s" % (r, c)
                else:
                    assert c["dense"] == 1, "round %d: at 1/8 dead slots the next scan is dense: %s" % (r, c)
            g = gsl.getMap().getAllSurfels()
            c = scan_launches(gsl)
            # (after a dense scan there is nothing left to compact; a map of less than a group has no group's last)
            want = int(route == "download" and dies.any())
            assert c["extract_flags"] == c["compact_scatter"] == want, "round %d download: %s" % (r, c)
            what = "round %d (%d hidden)" % (r, n)
            same_records(g, osl.map.download(), what + ": library vs oracle")
            same_records(g[:live.size], live, what + ": the hidden surfels that live, in slot order")
    finally:
        gsl.ctx.close()


@pytest.mark.parametrize("name", ["lane31", "block_first"])
def test_a_reinserted_tile_that_fits_only_after_compacting_dead_slots(name, request):
    """Paging near the capacity while interleaved dead slots exist (tiles of 6 m, partial_extraction = 0). A map
    uploaded 250 000 surfels below the capacity: 1 000 surfels in tile (-1, -1), 300 000 in tile (-1, 0) and a fill
    around the origin whose pattern's surfels die in the first update. Moving the pose to x = 4 extracts column -1,
    and the in-place updates that follow leave it behind as dead slots too; moving back re-inserts (-1, -1), which
    fits behind the physical end, and then (-1, 0), which fits only after the map is compacted (append_tiles ->
    compact_map over the host's physical end, which the first re-insertion raised)."""
    if cusim(request):
        pytest.skip("a map at the surfel capacity: too slow for the CPU executor (the dead-slot compactions above run "
                    "there)")
    from test_gpu_lazy_map import _hidden_block, _set_current_pose
    po, pp = both_params(**sized(900, submap_extent=3.0, submap_dimension=1, partial_extraction=0))
    scene = synth.Scene(width=900, height=64)
    home = synth.trajectory(1)[0]
    sc = [scene.scan(i, home) for i in range(8)]
    a1 = _hidden_block(1000, -8.5, -3.5, -8.5, -3.5, 21)
    a2 = _hidden_block(300_000, -8.5, -3.5, -2.5, 2.5, 22)
    n = MAX_SURFELS - 250_000 - a1.size - a2.size
    dies = pattern(name, n)
    fill = hidden_surfels(dies, 23, extent=2.5)
    s = np.concatenate([fill, a1, a2])
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    try:
        osl.map.upload(s, 0)
        gsl.getMap().upload(s, 0)
        gsl.ctx.profile(True)
        gsl.ctx.profile_collect()
        launches = []
        for part, x in ((sc[0:3], None), (sc[3:6], 4.0), (sc[6:8], 0.0)):
            if x is not None:
                _set_current_pose(osl, gsl, x)
            for pts, lab, prb in part:
                osl.process_scan(pts, lab, prb)
                gsl.processScan(pts, lab, prb)
                launches.append(scan_launches(gsl))
                assert gsl.getMap().size() == osl.map.size(), "scan %d" % (len(launches) - 1)
            assert gsl.getMap().submap_origin() == osl.map.submap_origin()
        assert all(c["dense"] == 0 for c in launches), launches  # in place throughout: the dead slots stay
        assert all(c["update_surfels"] == 1 for c in launches[1:]), launches
        ext = [c["extract_flags"] for c in launches]
        assert ext[3] == 3, ext  # column -1 leaves
        assert ext[6] == 4, ext  # column 2 leaves, column -1 comes back: one compaction
        g = gsl.getMap().getAllSurfels()
        same_records(g, osl.map.download(), "surfels after re-insertion")
        live = fill[~dies]
        same_records(g[:live.size], live, "the fill that lives, in slot order")
    finally:
        gsl.ctx.close()


# ---- the extraction cut at the physical end of the default pool
def test_a_tile_cut_at_the_end_of_the_default_pool(moves, request):
    """Default cache: tile (-4, 4), the first extraction, sits in slot 0 at the pool's start. Four columns of 4 163 190
    surfels fill the pool to 123 456 short of its 16 777 216-surfel allocation, and a 500 000-surfel tile is then cut
    at that end: the first 123 456 in map order are kept, the rest counted as dropped, and no lane is written past the
    allocation (one lane's end is the next lane's start, where slot 0 lies). Then tile (-4, 4) comes back unchanged."""
    if cusim(request):
        pytest.skip("fills the 16 M-surfel pool: too slow for the CPU executor (the managed pool's cut at its end runs "
                    "there)")
    m = moves()
    short = 123_456
    fill = (POOL_CAP - short - 1000) // 4
    assert 4 * fill + 1000 + short == POOL_CAP and fill <= MAX_SURFELS
    col = lambda i, n: column(i, [B] * 8 + [n - 8 * B], -4)  # noqa: E731
    m.step(12, upload=surfels_at([(-4, 4)] * 1000, 400))  # origin 1: column -4 leaves, (-4, 4) to slot 0
    for k in range(4):  # column -3 and column 6 leave in turn (origins 1 <-> 2)
        x, i = (32, -3) if k % 2 == 0 else (12, 6)
        m.step(x, upload=surfels_at(col(i, fill), 401 + k))
    assert m.model.end() == POOL_CAP - short
    m.step(32, upload=surfels_at(column(-3, [0] * 8 + [B], -4), 405), oracle=False)  # (-3, 4) leaves first
    assert m.model.end() == POOL_CAP and m.model.cache[(-3, 4)].shape[0] == short
    assert m.p.ctx.tile_cache_info()["dropped"] == B - short
    m.upload(np.zeros(0, O.SURFEL_DTYPE))
    m.step(12, oracle=False)  # origin 1
    m.upload(np.zeros(0, O.SURFEL_DTYPE))
    m.step(-12)  # origin 0: column -4 comes back, and the oracle's map is the library's again
    assert m.model.map.shape[0] == 1000
