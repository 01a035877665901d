"""Designed inputs of the map update at its thresholds, shared by tests/test_gpu_update_edges.py (CUDA, oracle, model) and
tests/test_update_edges_ref.py (the reference's shaders, oracle, model), so that the two cannot drift.

A case is a surfel list, a data frame uploaded as it is, a pose, a map timestamp and parameter overrides, plus the
branches tests/update_reference.py must report for given surfels and pixels. Surfels are placed by the pixel they
must land on (at least update_reference.PIXEL_MARGIN from its edges), and the quantity under test is placed exactly:
  * radius map / generation pass: a vertex (-L, 0, 0) has the view direction (1, -0, -0) exactly, so the angle
    dot3(n, view_dir) is the normal's x component, bit for bit;
  * update distance and angle: the surfel sits in the top row at z = 0.25 with normal (0, 0, -1), so the distance is
    |v.z - 0.25| (exact by Sterbenz for the data z used) and the angle |cross| is the x component of the normalised data
    normal, searched over fp32 inputs until it equals the target.
"""
import math

import numpy as np

import update_reference as M

f32 = np.float32
TS = 5  # map timestamp of every case
SHAPES = [(16, 96), (13, 77)]
BASE = dict(max_depth=60.0, model_max_depth=60.0)  # (max_depth - min_depth) = 58 makes z = 1 - 2^-24 reachable


def nxt(x, n=1):
    x = f32(x)
    for _ in range(abs(n)):
        x = np.nextafter(x, f32(np.inf) if n > 0 else f32(-np.inf))
    return x


class Case:
    def __init__(self, name, H, W, kw=None):
        self.name, self.H, self.W = name, H, W
        self.kw = dict(BASE, **(kw or {}))
        self.surfels = []
        self.V = np.zeros((H, W, 4), f32)
        self.N = np.zeros((H, W, 4), f32)
        self.S = np.zeros((H, W, 4), f32)
        self.pose = np.eye(4, dtype=f32)
        self.poses = {}
        self.expect = []        # (surfel index, tag)
        self.expect_pix = []    # ((row, col), tag) of the radius / generation passes

    def params(self, P):
        return P.default_params(data_width=self.W, model_width=self.W, data_height=self.H, model_height=self.H, **self.kw)

    def frame(self):
        return self.V, self.N, self.S

    def add(self, rec, *tags):
        self.surfels.append(rec)
        for t in tags:
            self.expect.append((len(self.surfels) - 1, t))
        return len(self.surfels) - 1

    def records(self):
        a = np.zeros(len(self.surfels), M.SURFEL_DTYPE)
        for i, r in enumerate(self.surfels):
            a[i] = r
        return a


# ---- placement -----------------------------------------------------------------------------------------------------
def direction(H, W, row, col, fx=0.5, fy=0.5):
    """unit direction (fp64) through (col + fx, row + fy) of the data image (fov 3 / -25 degrees)"""
    yaw = -math.pi * (2.0 * (col + fx) / W - 1.0)
    pitch = (1.0 - (row + fy) / H) * 28.0 - 3.0
    el = math.radians(-pitch)
    return np.array([math.cos(el) * math.cos(yaw), math.cos(el) * math.sin(yaw), math.sin(el)])


def at_depth(H, W, row, col, r):
    return (direction(H, W, row, col) * r).astype(f32)


def at_z(H, W, row, col, z):
    """a point of the pixel's centre beam whose z component is exactly z (rows with positive elevation)"""
    d = direction(H, W, row, col)
    p = (d * (z / d[2])).astype(f32)
    p[2] = f32(z)
    return p


def with_z01(c, p, row, col, target):
    """a point near the pixel's centre beam whose normalised depth (fp32, model) is exactly `target`"""
    d = direction(c.H, c.W, row, col)
    rng = np.arange(-40, 41)
    prm = c.params(_Params)
    lo, hi = f32(prm.min_depth), f32(prm.max_depth)
    for r in np.linspace(float(lo + target * (hi - lo)) - 1e-4, float(lo + target * (hi - lo)) + 1e-4, 9):
        base = (d * r).astype(f32)
        for k in rng:
            q = base.copy()
            q[0] = nxt(q[0], int(k))
            if M.depth01(prm, M.v3(*q)) == f32(target):
                return q
    raise AssertionError("no point at z = %r" % target)


def surfel(pos, nrm, **kw):
    r = np.zeros((), M.SURFEL_DTYPE)
    r["x"], r["y"], r["z"] = pos
    r["nx"], r["ny"], r["nz"] = nrm
    r["radius"], r["confidence"], r["timestamp"], r["weight"], r["count"] = 0.01, 1.0, TS - 1, 1.0, 0.0
    r["w"] = 0.5
    for k, v in kw.items():
        r[k] = v
    return r


def measure(c, row, col, v, n, w=(1.0, 1.0), sem=(0.0, 0.0, 0.0, 0.5)):
    c.V[row, col] = (*v, w[0])
    c.N[row, col] = (*n, w[1])
    c.S[row, col] = sem


def facing(c, row, col, depth, **kw):
    """a surfel at depth `depth` on the pixel's beam, its normal towards the sensor, and a measurement on top of it"""
    p = at_depth(c.H, c.W, row, col, depth)
    n = (-p / np.linalg.norm(p)).astype(f32)
    measure(c, row, col, p, n)
    return surfel(p, n, **kw)


UP = (f32(0), f32(0), f32(-1.0))


def top(c, col, **kw):
    """a surfel in the top row at z = 0.25 with normal (0, 0, -1), measured at distance 0 with the same normal"""
    p = at_z(c.H, c.W, c.H - 1, col, 0.25)
    measure(c, c.H - 1, col, p, UP)
    return surfel(p, UP, **kw)


def angle_normal(target):
    """a data normal (a, 0, -1) whose normalised x component, the update's angle against (0, 0, -1), is `target`"""
    t = float(target)
    a0 = t / math.sqrt(1.0 - t * t)
    a = np.array([nxt(a0, k) for k in range(-64, 65)], f32)
    ln = np.sqrt((a * a + f32(0.0) * f32(0.0)) + f32(1.0) * f32(1.0))
    hit = np.nonzero(a / ln == f32(target))[0]
    assert hit.size, "no normal at angle %r" % target
    return (a[hit[0]], f32(0.0), f32(-1.0))


def label_tie():
    """a semantic x whose label St.x * 255 is exactly k + 0.5"""
    for base in (10.5, 12.5, 40.5):
        x0 = f32(base / 255.0)
        for k in range(-8, 9):
            x = nxt(x0, k)
            if x * f32(255.0) == f32(base):
                return x
    raise AssertionError("no label tie")


class _Params:  # the model's default parameters (api / oracle take them from the library)
    @staticmethod
    def default_params(**kw):
        from oracle import oracle as O
        return O.default_params(**kw)


# ---- the cases -------------------------------------------------------------------------------------------------------
def radius_threshold(H, W):
    """K6b: angle > radconf_angle_thresh at equality and one ulp either side (max_angle 60)"""
    c = Case("radius_threshold", H, W, dict(max_angle=60.0))
    thr = M.derived(c.params(_Params))["radconf_angle_thresh"]
    for i, (a, tag) in enumerate(((nxt(thr, -1), "radius:angle_rejected"), (thr, "radius:angle_rejected"),
                                  (nxt(thr, 1), "radius:c_low"))):
        c.V[0, i] = (-4.0, 0.0, 0.0, 1.0)
        c.N[0, i] = (a, 0.0, 0.0, 1.0)
        c.expect_pix.append(((0, i), tag))
    return c


def radius_edges(H, W):
    """K6b clamps and validity, and the generation pass's own tests, on pixels with the exact-angle vertex (-L, 0, 0)"""
    c = Case("radius_edges", H, W)
    prm = c.params(_Params)
    ps = M.derived(prm)["pixel_size"]
    rad = lambda L: ((f32(1.41) * f32(L)) * ps) / f32(1.0)  # noqa: E731
    c.kw.update(min_radius=float(rad(4.0)), max_radius=float(rad(32.0)))
    px = iter((y, x) for x in range(W) for y in range(H))

    def pixel(L, n, w=(1.0, 1.0), sem=(0.0, 0.0, 0.0, 0.5), *tags):
        yx = next(px)
        c.V[yx] = (-f32(L), 0.0, 0.0, w[0])
        c.N[yx] = (*n, w[1])
        c.S[yx] = sem
        for t in tags:
            c.expect_pix.append((yx, t))
        return yx
    one = (1.0, 0.0, 0.0)
    # the c clamp at 0.5 and 1 (the rest of the normal off-axis: only n.x enters the angle)
    pixel(8.0, (nxt(0.5, -1), 0.8, 0.0), (1, 1), (0, 0, 0, .5), "radius:c_low")
    pixel(8.0, (f32(0.5), 0.8, 0.0), (1, 1), (0, 0, 0, .5), "radius:c_low")
    pixel(8.0, (nxt(0.5, 1), 0.8, 0.0), (1, 1), (0, 0, 0, .5), "radius:c_mid")
    pixel(8.0, (nxt(1.0, -1), 0.0, 0.0), (1, 1), (0, 0, 0, .5), "radius:c_mid")
    pixel(8.0, one, (1, 1), (0, 0, 0, .5), "radius:c_high")
    pixel(8.0, (nxt(1.0, 1), 0.0, 0.0), (1, 1), (0, 0, 0, .5), "radius:c_high")
    # min_radius / max_radius at equality and the depths one ulp either side
    for L in (nxt(4.0, -1), f32(4.0), nxt(4.0, 1)):
        pixel(L, one, (1, 1), (0, 0, 0, .5), "radius:min" if L <= 4.0 else "radius:c_high")
    for L in (nxt(32.0, -1), f32(32.0), nxt(32.0, 1)):
        pixel(L, one, (1, 1), (0, 0, 0, .5), "radius:max" if L >= 32.0 else "radius:c_high")
    # invalid vertex / normal: w = 0.5 and one ulp above; w in [0.5, 1) passes K6b but never generates
    h = nxt(0.5, 1)
    pixel(8.0, one, (0.5, 1.0), (0, 0, 0, .5), "radius:invalid", "gen:invalid")
    pixel(8.0, one, (1.0, 0.5), (0, 0, 0, .5), "radius:invalid", "gen:invalid")
    pixel(8.0, one, (h, 1.0), (0, 0, 0, .5), "radius:c_high", "gen:w_below_one")
    pixel(8.0, one, (1.0, h), (0, 0, 0, .5), "radius:c_high", "gen:w_below_one")
    pixel(8.0, one, (nxt(1.0, -1), 1.0), (0, 0, 0, .5), "gen:w_below_one")
    # the vertex at the origin: NaN view direction
    pixel(0.0, one, (1, 1), (0, 0, 0, .5), "radius:nan_angle", "gen:invalid_r")
    # R.w < 0.5: rejected by K6b with valid vertex and normal
    pixel(8.0, (-0.5, 0.0, 0.0), (1, 1), (0, 0, 0, .5), "radius:angle_rejected", "gen:invalid_r")
    # dot(n, view_dir) > 0.01 at equality and one ulp either side
    for a, t in ((nxt(0.01, -1), "gen:dot_rejected"), (f32(0.01), "gen:dot_rejected"), (nxt(0.01, 1), "gen:new")):
        pixel(8.0, (a, 0.0, 0.99), (1, 1), (0, 0, 0, .5), t)
    # movable labels (log_prior - 0.5), a label whose round trip is not exact, a non-movable one
    for lab in (10.0, 11.0, 13.0, 15.0, 18.0, 20.0, 30.0, 31.0, 32.0, 40.0):
        x = f32(f32(lab) / f32(255.0))
        mv = M.is_movable(x * f32(255.0))
        pixel(8.0, one, (1, 1), (x, 0.25, 0.75, 0.5), "gen:new:movable" if mv else "gen:new")
    return c


def stability(H, W):
    """old_conf < confidence_threshold and surfel_age < unstable_age at equality, and a timestamp in the future, on
    surfels that face away (no measurement decides for them)"""
    c = Case("stability", H, W)
    away = lambda col, **kw: surfel(at_depth(H, W, 2, col, 10.0), -facing_n(H, W, 2, col), **kw)  # noqa: E731
    c.add(away(1, confidence=0.0, timestamp=0), "stable", "not_visible")
    c.add(away(3, confidence=nxt(0.0, -1), timestamp=TS - 3), "unstable:old", "not_visible")
    c.add(away(5, confidence=nxt(0.0, -1), timestamp=TS - 2), "unstable:young")
    c.add(away(7, confidence=-0.25, timestamp=TS + 4), "unstable:future", "unstable:young")
    return c


def facing_n(H, W, row, col):
    d = direction(H, W, row, col)
    return (-d).astype(f32)


def visibility(H, W):
    """visible with a dot of exactly +-0, inside at the last column / row, z = 1 and the largest z below it, a surfel
    nearer than min_depth, and the measurement's w at 0.5 and one ulp above"""
    c = Case("visibility", H, W)
    r0 = _zero_row(H)
    # (x > 0 and y > 0: every term of the dot is a signed zero, and the normal's z gives the sign of the last)
    for col, nz, t in ((W // 2 - 3, 1.0, "visible:zero_dot_neg"), (W // 2 - 5, -1.0, "visible:zero_dot_pos")):
        p = at_depth(H, W, r0, col, 10.0)
        p[2] = 0.0
        measure(c, r0, col, p, (0.0, 0.0, nz))
        c.add(surfel(p, (0.0, 0.0, nz)), t, "not_visible")
    c.add(facing(c, H - 1, W - 1, 10.0), "match", "marks_pixel")
    c.add(facing(c, H - 2, W - 1, 10.0), "match", "marks_pixel")
    c.add(facing(c, H - 1, W - 3, 10.0), "match", "marks_pixel")
    for col, z, tags in ((6, 1.0, ("outside:z",)), (8, nxt(1.0, -1), ("match", "marks_pixel", "depth24:top"))):
        p = with_z01(c, None, 3, col, z)
        n = (-p / np.linalg.norm(p)).astype(f32)
        measure(c, 3, col, p, n)
        c.add(surfel(p, n), *tags)
    c.add(facing(c, 4, 10, 1.5), "inside:nearer_than_min_depth", "match")
    h = nxt(0.5, 1)
    for col, w, tags in ((12, (0.5, 1.0), ("measurement_invalid",)), (14, (1.0, 0.5), ("measurement_invalid",)),
                         (16, (h, 1.0), ("match",)), (18, (1.0, h), ("match",))):
        s = facing(c, 5, col, 12.0)
        c.V[5, col, 3], c.N[5, col, 3] = w
        c.add(s, *tags)
    return c


def _zero_row(H):
    """the row whose pixel holds elevation 0 (at least the margin from its edges)"""
    py = (1.0 - 3.0 / 28.0) * H
    assert abs(py - round(py)) > 1e-2
    return int(math.floor(py))


def compatibility(H, W):
    """distance < map_max_distance and angle < update_angle_thresh at equality and one ulp either side"""
    c = Case("compatibility", H, W)
    dthr = f32(c.params(_Params).map_max_distance)
    athr = M.derived(c.params(_Params))["update_angle_thresh"]
    col = 1
    for D, t in ((nxt(dthr, -1), "match"), (dthr, "no_match:distance"), (nxt(dthr, 1), "no_match:distance")):
        s = top(c, col)
        vz = f32(0.25 - float(D))
        assert abs(f32(0.25) - vz) == D
        c.V[H - 1, col, 2] = vz
        c.add(s, t)
        col += 3
    for A, t in ((nxt(athr, -1), "match"), (athr, "no_match:angle"), (nxt(athr, 1), "no_match:angle")):
        s = top(c, col)
        c.N[H - 1, col, :3] = angle_normal(A)
        c.add(s, t)
        col += 3
    return c


def semantics(H, W):
    """label_diff with a rounding tie, is_movable on labels with exact and inexact round trips, the penalty and its
    removal of a surfel that matched (which must not mark its pixel)"""
    c = Case("semantics", H, W)
    tie = label_tie()
    s = facing(c, 2, 3, 10.0, r=f32(f32(10.0) / f32(255.0)))
    c.S[2, 3] = (tie, 0, 0, 0.75)
    c.add(s, "label:round_tie", "match")
    col = 5
    for lab in (10.0, 11.0, 13.0, 15.0, 18.0, 20.0, 30.0, 31.0, 32.0):
        x = f32(f32(lab) / f32(255.0))
        exact = x * f32(255.0) == f32(lab)
        s = facing(c, 3, col, 10.0, r=x, confidence=5.0)
        c.S[3, col] = (f32(40.0) / f32(255.0), 0, 0, 0.25)
        c.add(s, "penalty" if exact else "match")
        col += 2
    # the penalty removes a surfel that matched: its pixel stays unmarked and generates a new surfel
    s = facing(c, 4, 40, 10.0, r=f32(f32(10.0) / f32(255.0)), confidence=0.0)
    c.S[4, 40] = (f32(40.0) / f32(255.0), 0, 0, 0.25)
    c.add(s, "penalty", "removed:log_unstable", "matched_but_removed")
    return c


def confidence(H, W, mode):
    c = Case("confidence_mode_%d" % mode, H, W, dict(confidence_mode=mode))
    c.add(facing(c, 2, 2, 10.0), "confidence_mode:%d" % mode, "match")
    return c


def p_clamps(H, W):
    """p clamped at p_unstable (sigma_distance tiny) and at 1 (p_stable = 1: log(p / (1 - p)) = inf, held at 20)"""
    a = Case("p_unstable", H, W, dict(confidence_mode=2, sigma_distance=1e-3))
    s = top(a, 2)
    a.V[H - 1, 2, 2] = f32(0.25 - 0.125)
    a.add(s, "p:unstable", "match")
    b = Case("p_one", H, W, dict(confidence_mode=0, p_stable=1.0))
    b.add(facing(b, 2, 2, 10.0), "p:one", "clamp20")
    return [a, b]


def nonmatching(H, W):
    """the non-matching branch: the index-map winner, a surfel behind it, an equal-depth tie (the lower index wins), and
    the clamp at 20 / `< log_unstable` at equality on surfels that take log_prior"""
    c = Case("nonmatching", H, W, dict(p_prior=0.5))
    d = M.derived(c.params(_Params))
    col = 2

    def pair(conf_behind, front_tags, behind_tags, tie=False):
        nonlocal col
        front = facing(c, 6, col, 10.0)
        back = surfel(at_depth(H, W, 6, col, 10.0 if tie else 14.0), (front["nx"], front["ny"], front["nz"]),
                      confidence=conf_behind)
        c.V[6, col, :3] = c.V[6, col, :3] * f32(0.5)  # the measurement 5 m in front of both: no match
        c.add(front, *front_tags)
        c.add(back, *behind_tags)
        col += 3
    pair(1.0, ("no_match:distance", "no_match:winner"), ("no_match:not_winner",))
    pair(1.0, ("no_match:winner",), ("no_match:not_winner",), tie=True)
    pair(f32(20.0), ("no_match:winner",), ("no_match:not_winner", "clamp20"))
    pair(nxt(20.0, 1), ("no_match:winner",), ("no_match:not_winner", "clamp20"))
    pair(nxt(20.0, -1), ("no_match:winner",), ("no_match:not_winner",))
    pair(d["log_unstable"], ("no_match:winner",), ("no_match:not_winner", "log_unstable:equal"))
    pair(nxt(d["log_unstable"], -1), ("no_match:winner",), ("no_match:not_winner", "removed:log_unstable"))
    return c


def averaging(H, W, kw, name, build):
    c = Case(name, H, W, kw)
    build(c)
    return c


def averaging_cases(H, W):
    out = []

    def radius_eq(c):
        rad = lambda row, col: M.radius_pixel(c.params(_Params), M.derived(c.params(_Params)), c.V[row, col],  # noqa
                                              c.N[row, col])[0][0]
        s = facing(c, 2, 2, 10.0)
        s["radius"] = rad(2, 2)
        c.add(s, "no_average")
        s = facing(c, 2, 4, 10.0)
        s["radius"] = nxt(rad(2, 4), 1)
        c.add(s, "average")
    out.append(averaging(H, W, {}, "new_radius_equal", radius_eq))

    def active(c):
        c.kw["active_timestamps"] = 3
        c.add(facing(c, 2, 2, 10.0, count=float(TS - 3), radius=2.0), "no_average")
        c.add(facing(c, 2, 4, 10.0, count=float(TS - 2), radius=2.0), "average")
    out.append(averaging(H, W, {}, "active_timestamps", active))
    out.append(averaging(H, W, dict(update_always=1), "update_always",
                         lambda c: c.add(_tilted(c, 2, 2), "average:always")))
    for ws in (0, 1, 2):
        out.append(averaging(H, W, dict(weighting_scheme=ws), "weighting_scheme_%d" % ws,
                             lambda c, ws=ws: c.add(_tilted(c, 2, 2, radius=2.0, weight=3.0), "weighting_scheme:%d" % ws)))

    def zero_sum(c):
        # w1 = old weight 0, w2 = dot(n, view_dir) = 0: the data normal (0, 0, -1) is perpendicular to a vertex at z = 0
        s = top(c, 3, weight=0.0, radius=2.0)
        c.V[H - 1, 3, 2] = 0.0
        c.add(s, "weights:zero_sum", "average")
    out.append(averaging(H, W, dict(weighting_scheme=2, map_max_distance=0.5), "weights_zero_sum", zero_sum))
    def max_weight(c):
        # w1 + w2 at max_weight and one ulp either side: min(max_weight, sum) is pinned by its neighbours
        c.add(_tilted(c, 2, 2, radius=2.0, weight=19.0), "max_weight:equal")
        c.add(_tilted(c, 2, 4, radius=2.0, weight=nxt(19.0, -1)), "weighting_scheme:1")
        c.add(_tilted(c, 2, 6, radius=2.0, weight=nxt(19.0, 1)), "weighting_scheme:1")
    out.append(averaging(H, W, dict(weighting_scheme=1, max_weight=20.0), "max_weight_equal", max_weight))
    out.append(averaging(H, W, dict(averaging_scheme=1), "averaging_scheme_1",
                         lambda c: c.add(_tilted(c, 2, 2, radius=2.0), "averaging_scheme:1")))
    # exactly parallel normals: slerp's 1 / sin(0) makes the normal NaN (DESIGN.md section 2)
    out.append(averaging(H, W, dict(update_always=1), "slerp_parallel",
                         lambda c: c.add(top(c, 2), "slerp:parallel", "average:always")))
    return out


def _tilted(c, row, col, **kw):
    """a matched surfel whose measured normal is 20 degrees off its own (a well-conditioned slerp)"""
    s = facing(c, row, col, 10.0, **kw)
    n = np.array([s["nx"], s["ny"], s["nz"]], np.float64)
    t = np.cross(n, [0.0, 0.0, 1.0])
    t /= np.linalg.norm(t)
    c.N[row, col, :3] = (math.cos(math.radians(20)) * n + math.sin(math.radians(20)) * t).astype(f32)
    return s


def submap(H, W):
    """copy_surfels: |w - c| == extent (kept) and one ulp beyond (dropped); a timestamp with bit 31 set (dropped); and
    records that only the update carries (fields it never writes keep their bits)"""
    c = Case("submap", H, W)
    prm = c.params(_Params)
    extent = f32(2.0) * f32(prm.submap_dimension) * f32(prm.submap_extent) + f32(prm.submap_extent)
    T = np.eye(4, dtype=f32)
    T[0, 3] = 64.0
    c.poses[1] = T  # the surfels' pose entry moves them out by a power of two
    for x, t in ((extent, "stable"), (nxt(extent, 1), "submap:dropped")):
        p = at_depth(H, W, 2, W // 2 - 3, 10.0)
        p[0] = x - f32(64.0)
        c.add(surfel(p, (1.0, 0.0, 0.0), count=1.0), t, "not_visible")
    c.add(surfel(at_depth(H, W, 2, 5, 10.0), (1.0, 0.0, 0.0), timestamp=0xFFFFFFFF), "submap:dropped")
    rng = np.random.default_rng(3)
    for col in (9, 11, 13):
        s = surfel(at_depth(H, W, 2, col, 10.0), -facing_n(H, W, 2, col), confidence=3.0)
        for f in ("radius", "weight", "r", "g", "b", "w"):
            s[f] = f32(rng.uniform(-1e3, 1e3))
        c.add(s, "not_visible")
    return c


def all_cases(H, W):
    cs = [radius_threshold(H, W), radius_edges(H, W), stability(H, W), visibility(H, W), compatibility(H, W),
          semantics(H, W), nonmatching(H, W), submap(H, W)]
    cs += [confidence(H, W, m) for m in range(4)]
    cs += p_clamps(H, W)
    cs += averaging_cases(H, W)
    return cs


def case_ids():
    return [c.name for c in all_cases(*SHAPES[0])]


def get(name, H, W):
    return next(c for c in all_cases(H, W) if c.name == name)


def check_tags(c, model):
    """the branches the case was built for are those the model reports"""
    for k, t in c.expect:
        assert t in model["tags"][k], "%s: surfel %d should take %s, the model says %s" % (c.name, k, t, sorted(model["tags"][k]))
    for yx, t in c.expect_pix:
        got = set(model["radius_tags"][yx].split(",")) | {model["gen_tags"].get(yx)}
        assert t in got, "%s: pixel %s should take %s, the model says %s" % (c.name, yx, t, got)


# every branch of update_reference's tags that the designed cases must reach
BRANCHES = {
    "radius:invalid", "radius:nan_angle", "radius:angle_rejected", "radius:c_low", "radius:c_mid", "radius:c_high",
    "radius:min", "radius:max",
    "stable", "unstable:young", "unstable:old", "unstable:future", "visible:zero_dot_neg", "visible:zero_dot_pos",
    "not_visible", "outside:z", "measurement_invalid", "inside:nearer_than_min_depth", "depth24:top", "match",
    "no_match:distance", "no_match:angle", "no_match:winner", "no_match:not_winner", "label:round_tie", "penalty",
    "confidence_mode:0", "confidence_mode:1", "confidence_mode:2", "confidence_mode:3", "p:unstable", "p:one",
    "clamp20", "removed:log_unstable", "log_unstable:equal", "average", "average:always", "no_average",
    "weighting_scheme:0", "weighting_scheme:1", "weighting_scheme:2", "weights:zero_sum", "max_weight:equal",
    "averaging_scheme:1", "slerp:parallel", "marks_pixel", "matched_but_removed", "submap:dropped",
    "gen:integrated", "gen:invalid", "gen:w_below_one", "gen:invalid_r", "gen:dot_rejected", "gen:new", "gen:new:movable",
}


def reached(model):
    got = set()
    for t in model["tags"]:
        got |= t
    for t in model["radius_tags"].values():
        got |= set(t.split(","))
    got |= set(model["gen_tags"].values())
    return got
