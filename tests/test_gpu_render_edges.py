"""The surfel render pass (k_render_scatter + k_render_resolve) at the points where its fast paths switch, bit for bit
against an exact reference rasteriser (tests/render_reference.py) and against the oracle.

The kernel rasterises a quad whose clamped pixel box is at most 12 x 5 and whose corners lie within 2^14 units (1/256 px)
of the box's first pixel centre with int32 edge functions, flattened over the block; every other quad takes a warp with
int64 set-up. Queue entries pack slot | di | dj | triangle, the orientation fix travels as a "swapped" bit, plain targets
take their own path (class-3 surfels fall back to emit_fragment), and depth ties are broken by the key's low bits. The
oracle and the reference have none of these paths; random clouds reach their edges only by chance. Every case here is
constructed numerically with the reference's own corner computation, asserts the regime it is built for (the log lists
the reference's classification per case), and goes through render / render_active / render_inactive / render_composed at
compose_rendering 0 and 1. On a mismatch the message names which of product, oracle and reference disagree. The
per-case classifications are written to the terminal also when the tests pass."""
import collections

import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api
from helpers import bits, both_params
import render_reference as RR

pytestmark = pytest.mark.gpu

F = np.float32
T_NOW = 150                  # map timestamp: timestamp_threshold = 50
OLD, NEW, BOTH = (10, 20), (120, 140), (10, 140)   # (creation = count, timestamp): old, new, old and re-observed
CONF = 0.5
SPAN = RR.SMALL_SPAN
EYE = np.eye(4)
SHIFT = np.eye(4)
SHIFT[:3, 3] = (0.25, -0.125, 0.0625)   # dyadic: inv(P) * pose[t] stays exact
# square-ish pixels: 1441 x 33 over 360 x 8 degrees; odd sizes put the image's middle row / column on pixel centres
BASE = dict(data_width=360, data_height=32, model_width=1441, model_height=33, model_fov_up=4.0, model_fov_down=-4.0)
SEEN = collections.Counter()  # regimes reached over the whole file
_REPORTER = []


@pytest.fixture(autouse=True)
def _terminal(request):
    pm = request.config.pluginmanager
    _REPORTER[:] = [pm.get_plugin("terminalreporter"), pm.get_plugin("capturemanager")]
    yield


def log(*parts):
    """a line in the test log also on a passing run (pytest captures print output)"""
    msg = " ".join(str(p) for p in parts)
    if _REPORTER and None not in _REPORTER:
        with _REPORTER[1].global_and_fixture_disabled():
            _REPORTER[0].write_line(msg)
    else:
        print(msg)


# ---------------------------------------------------------------------------------------------------------------
# surfels and geometry
# ---------------------------------------------------------------------------------------------------------------
def make_surfels(p, n, r, cls, seed=0):
    """surfel records: centres p [N, 3], normals n [N, 3], radii r [N], classes [(count, timestamp)]"""
    p, n = np.atleast_2d(p), np.atleast_2d(n)
    N = p.shape[0]
    S = np.zeros(N, O.SURFEL_DTYPE)
    S["x"], S["y"], S["z"] = p[:, 0], p[:, 1], p[:, 2]
    S["nx"], S["ny"], S["nz"] = n[:, 0], n[:, 1], n[:, 2]
    S["radius"] = r
    S["confidence"] = 1.0
    cls = np.broadcast_to(np.asarray(cls, np.int64).reshape(-1, 2), (N, 2))
    S["count"], S["timestamp"] = cls[:, 0], cls[:, 1]
    S["color"], S["weight"] = 3.0, 1.0
    rng = np.random.default_rng(seed)
    for f in "rgbw":
        S[f] = rng.uniform(0, 1, N).astype(F)   # the semantic lane tells the winners apart
    return S


def culled(N, seed=1):
    """surfels every draw call drops in stage A (confidence under the threshold)"""
    S = make_surfels(np.tile([10.0, 0.0, 0.0], (N, 1)), np.tile([-1.0, 0.0, 0.0], (N, 1)), 0.5, NEW, seed)
    S["confidence"] = -1.0
    return S


def direction(m, x, y):
    """unit direction (float64) of image coordinates x, y in [0, 1)"""
    yaw = np.pi * (1.0 - 2.0 * np.asarray(x, np.float64))
    pitch = np.deg2rad((1.0 - np.asarray(y, np.float64)) * float(m.fov) - float(m.fov_up))
    return np.stack([np.cos(pitch) * np.cos(yaw), np.cos(pitch) * np.sin(yaw), -np.sin(pitch)], -1)


def geometry(po, S, pose=EYE, old=False):
    R = RR.Renderer(po, S, T_NOW)
    return R.geometry(pose, CONF, R.t_thr, old)


def regimes(po, S):
    """the reference's classification of every surfel (drawn by the old or the new pass at the identity pose)"""
    R = RR.Renderer(po, S, T_NOW)
    go, gn = R.geometry(EYE, CONF, R.t_thr, True), R.geometry(EYE, CONF, R.t_thr, False)
    gn.alive = go.alive | gn.alive   # identity pose: both passes see the same quads
    return RR.classify(gn)


def boxes(g):
    """vectorised clamped boxes and corner spans: i0, i1, j0, j1, span (max |corner - first pixel centre|)"""
    W, H = g.m.W, g.m.H
    i0 = np.maximum(-((-(g.X.min(1) - 128)) // 256), 0)
    i1 = np.minimum((g.X.max(1) - 128) // 256, W - 1)
    j0 = np.maximum(-((-(g.Y.min(1) - 128)) // 256), 0)
    j1 = np.minimum((g.Y.max(1) - 128) // 256, H - 1)
    span = np.maximum(np.abs(g.X - (i0 * 256 + 128)[:, None]).max(1), np.abs(g.Y - (j0 * 256 + 128)[:, None]).max(1))
    return i0, i1, j0, j1, span


def random_quads(rng, po, N, x=(0.02, 0.98), y=(0.05, 0.95), d=(4.0, 40.0), rpx=(0.5, 8.0), tilt=1.5):
    """N random surfels facing the sensor more or less: centre at image coordinates in x / y, distance d, radius rpx
    azimuth pixels, normal tilted by up to `tilt` (float32 records)"""
    m = RR.Model(po)
    dirs = direction(m, rng.uniform(*x, N), rng.uniform(*y, N))
    dist = rng.uniform(*d, N)
    p = dirs * dist[:, None]
    nrm = -dirs + tilt * rng.uniform(0, 1, (N, 1)) * rng.normal(size=(N, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    r = dist * np.exp(rng.uniform(np.log(rpx[0]), np.log(rpx[1]), N)) * (2 * np.pi / m.W)
    return make_surfels(p, nrm, r, NEW)


def tri_areas(g, k):
    """signed snapped areas of the quad's two strip triangles (corners 0,1,2 and 1,2,3)"""
    X, Y = [int(v) for v in g.X[k]], [int(v) for v in g.Y[k]]
    return [(X[t + 1] - X[t]) * (Y[t + 2] - Y[t]) - (Y[t + 1] - Y[t]) * (X[t + 2] - X[t]) for t in range(2)]


def bisect(lo, hi, f, target):
    """a float32 value between lo and hi at which the integer-valued monotonic f equals target (None if skipped)"""
    lo, hi = F(lo), F(hi)
    flo = f(lo)
    for _ in range(200):
        mid = F((np.float64(lo) + np.float64(hi)) / 2)
        if mid == lo or mid == hi:
            return None
        fm = f(mid)
        if fm == target:
            return mid
        if (fm < target) == (flo < target):
            lo, flo = mid, fm
        else:
            hi = mid
    return None


# ---------------------------------------------------------------------------------------------------------------
# the comparison: product, oracle, reference
# ---------------------------------------------------------------------------------------------------------------
def _agree(what, got, ora, ref):
    for name, g, o, r in zip("vns", got, ora, ref):
        bg, bo, br = bits(np.asarray(g)), bits(np.asarray(o)), bits(np.asarray(r))
        if np.array_equal(bg, br) and np.array_equal(bo, br):
            continue
        px = lambda a, b: int(np.any(a != b, axis=-1).sum())   # noqa: E731
        first = np.argwhere(np.any(bg != br, axis=-1) | np.any(bo != br, axis=-1))[0]
        raise AssertionError("%s %s: pixels differing: product vs reference %d, oracle vs reference %d, product vs oracle "
                             "%d; first at %s: product %r oracle %r reference %r" %
                             (what, name, px(bg, br), px(bo, br), px(bg, bo), tuple(first), g[tuple(first)],
                              o[tuple(first)], r[tuple(first)]))


def check(name, kw, S, expect, poses=((EYE, EYE),), composes=(0, 1)):
    """S through the four render operators at compose_rendering 0 and 1, product = oracle = reference bit for bit;
    `expect`: the regimes (render_reference kinds) this case must reach"""
    kw = dict(BASE, **kw)
    po, _ = both_params(**kw)
    cls = regimes(po, S)
    counts = collections.Counter(c[0] for c in cls)
    small = collections.Counter((c[1], c[2]) for c in cls if c[0] == RR.SMALL)
    log("%s: %d surfels, regimes %s, small boxes (ni, nj) %s" % (name, len(S), dict(counts), dict(small)))
    for e in expect:
        assert counts[e] > 0, "%s: no surfel reaches %s (%s)" % (name, e, dict(counts))
    SEEN.update(counts)
    for compose in composes:
        po, pp = both_params(**dict(kw, compose_rendering=compose))
        R = RR.Renderer(po, S, T_NOW)
        ctx = api.Context(pp)
        try:
            gm, om = api.SurfelMap(ctx), O.Map(po)
            gm.upload(S, T_NOW)
            om.upload(S, T_NOW)
            out = api.Frame(ctx, po.model_width, po.model_height)
            for P_old, P_new in poses:
                tag = "%s compose=%d %s" % (name, compose, "same pose" if P_old is P_new else "two poses")
                ref = R.render(P_old, P_new, CONF)
                gm.render(P_old, P_new, out, CONF)
                _agree(tag + " render out", out.maps(), om.render(P_old, P_new, CONF), ref["out"])
                views = ("old", "new", "composed") if compose else ("old", "new")
                for w, key in enumerate(views):
                    _agree("%s %s frame" % (tag, key), getattr(gm, ("oldMapFrame", "newMapFrame", "composedFrame")[w])().maps(),
                           om.frame(w), ref[key])
                gm.render_active(P_new, CONF); om.render_active(P_new, CONF)
                _agree(tag + " render_active", gm.newMapFrame().maps()[:2], om.frame(1)[:2], R.render_active(P_new, CONF))
                gm.render_inactive(P_old, CONF); om.render_inactive(P_old, CONF)
                _agree(tag + " render_inactive", gm.oldMapFrame().maps()[:2], om.frame(0)[:2], R.render_inactive(P_old, CONF))
                gm.render_composed(P_old, P_new, CONF); om.render_composed(P_old, P_new, CONF)
                _agree(tag + " render_composed", gm.composedFrame().maps()[:2], om.frame(2)[:2],
                       R.render_composed(P_old, P_new, CONF))
        finally:
            ctx.close()
    return cls


# ---------------------------------------------------------------------------------------------------------------
# 1. box boundaries
# ---------------------------------------------------------------------------------------------------------------
def test_box_boundaries():
    """boxes of ni in {10..13} x nj in {3..6} (extent - 1): the 12 x 5 limit of the small path from both sides; one
    surfel per box, each class, laid out side by side"""
    po, _ = both_params(**BASE)
    rng = np.random.default_rng(7)
    C = random_quads(rng, po, 40000, rpx=(3.0, 12.0), tilt=1.2)
    g = geometry(po, C)
    i0, i1, j0, j1, span = boxes(g)
    chosen, used = [], np.zeros(po.model_width, bool)
    for ni in (10, 11, 12, 13):
        for nj in (3, 4, 5, 6):
            ok = g.alive & (i1 - i0 == ni) & (j1 - j0 == nj) & (span < SPAN)
            ok &= np.array([not used[a:b + 1].any() for a, b in zip(i0, i1)])
            k = int(np.nonzero(ok)[0][0])
            used[i0[k]:i1[k] + 1] = True
            chosen.append(k)
    S = C[chosen]
    S["count"], S["timestamp"] = np.array([OLD, NEW, BOTH] * 6)[:len(S)].T
    cls = check("box boundaries", {}, S, (RR.SMALL, RR.LARGE_BOX), poses=((EYE, EYE), (EYE, SHIFT)))
    want = [(RR.SMALL if ni < 12 and nj < 5 else RR.LARGE_BOX, ni, nj) for ni in (10, 11, 12, 13) for nj in (3, 4, 5, 6)]
    assert cls == want


# ---------------------------------------------------------------------------------------------------------------
# 2. corner span
# ---------------------------------------------------------------------------------------------------------------
SPAN_IMAGE = dict(model_width=12, model_height=5, model_fov_up=1.0, model_fov_down=-1.0)


def _span_case(po, row, offset, rng):
    """a quad facing the sensor, centred on the first or the last row of a 12 x 5 image (every clamped box is small), whose
    farthest corner lies exactly SPAN + offset units from the box's first pixel centre, beyond the top / bottom row"""
    m = RR.Model(po)
    for _ in range(20):
        dirv = direction(m, rng.uniform(0.3, 0.7), (row + 0.5 + rng.uniform(-0.3, 0.3)) / m.H)
        p, nrm = dirv * 5.0, -dirv

        def metric(r):
            g = geometry(po, make_surfels(p, nrm, r, NEW))
            if not g.alive[0]:
                return -10 ** 9
            dx0, dx1, dy0, dy1 = RR.corner_span(g, 0)
            return max(-dx0, dx1, -dy0, dy1)
        r = bisect(0.5, 5.0, metric, SPAN + offset)
        if r is not None:
            return make_surfels(p, nrm, r, NEW)
    raise AssertionError("no quad found for row %d, %+d" % (row, offset))


def test_corner_span():
    """clamped small boxes with the farthest corner at 2^14 - 1, 2^14 and 2^14 + 1 units from the box origin, hanging
    off the top and the bottom row (int32 edge functions are exact up to 2^14). The horizontal span cannot reach 2^14 on
    an image whose boxes are all small: the seam rule keeps every corner within half a turn of the centre."""
    po, _ = both_params(**dict(BASE, **SPAN_IMAGE))
    rng = np.random.default_rng(11)
    parts = []
    for row in (0, 4):
        for off in (-1, 0, 1):
            parts.append(_span_case(po, row, off, rng))
    S = np.concatenate(parts)
    S["count"], S["timestamp"] = np.array([OLD, NEW, BOTH] * 2).T
    cls = check("corner span", SPAN_IMAGE, S, (RR.SMALL, RR.LARGE_SPAN), poses=((EYE, EYE), (EYE, SHIFT)))
    for k, c in enumerate(cls):
        assert c[0] == (RR.SMALL if k % 3 == 0 else RR.LARGE_SPAN) and c[1] < 12 and c[2] < 5, (k, c)


# a wide image of five rows (every box is clamped to at most 5 rows) with a near plane close to the sensor
SPAN2_IMAGE = dict(model_width=1441, model_height=5, model_fov_up=1.0, model_fov_down=-1.0, model_min_depth=0.1)


def _int32_setup_peak(g, k):
    """the largest magnitude among the values tri_small_store would form in int32 for quad k (both triangles' area,
    edge functions at the box's first pixel centre), computed exactly"""
    i0, _, j0, _ = g.box(k)
    x = [int(v) - (i0 * 256 + 128) for v in g.X[k]]
    y = [int(v) - (j0 * 256 + 128) for v in g.Y[k]]
    peak = 0
    for t in range(2):
        A, B, C = (x[t], y[t]), (x[t + 1], y[t + 1]), (x[t + 2], y[t + 2])
        peak = max(peak, abs((B[0] - A[0]) * (C[1] - A[1]) - (B[1] - A[1]) * (C[0] - A[0])))
        for P, Q in ((B, C), (C, A), (A, B)):
            peak = max(peak, abs((Q[0] - P[0]) * (0 - P[1]) - (Q[1] - P[1]) * (0 - P[0])))
    return peak


def test_corner_span_on_both_axes():
    """clamped small boxes at the left and the right image edge whose corners lie between 2^14 and 2^16 units from the
    box origin on BOTH axes: a quad seen almost edge-on with one corner close to the sensor, whose projection swings far
    past the image edge and far above / below the five rows. Their int32 set-up would leave the int32 range (checked
    here exactly), so they pin the span limit itself: with a raised limit the small path would rasterise them with
    wrapped edge functions."""
    po, _ = both_params(**dict(BASE, **SPAN2_IMAGE))
    m = RR.Model(po)
    rng = np.random.default_rng(23)
    N = 60000
    parts = []
    for xs in ((0.5 / m.W, 8.0 / m.W), (1.0 - 8.0 / m.W, 1.0 - 0.5 / m.W)):
        c = direction(m, rng.uniform(*xs, N), rng.uniform(0.2, 0.8, N))
        d = rng.uniform(1.0, 6.0, N)
        q = rng.normal(size=(N, 3))
        q -= (q * c).sum(1, keepdims=True) * c
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        dot = rng.uniform(0.011, 0.06, N)   # just visible: the quad's plane nearly contains the line of sight
        C = make_surfels(c * d[:, None], -c * dot[:, None] + q * np.sqrt(1 - dot ** 2)[:, None], d * rng.uniform(0.4, 1.2, N),
                         NEW)
        g = geometry(po, C)
        i0, i1, j0, j1, _ = boxes(g)
        sx = np.abs(g.X - (i0 * 256 + 128)[:, None]).max(1)
        sy = np.abs(g.Y - (j0 * 256 + 128)[:, None]).max(1)
        sel = g.alive & (i0 <= i1) & (j0 <= j1) & (i1 - i0 < 12) & (j1 - j0 < 5)
        sel &= (np.minimum(sx, sy) >= SPAN) & (np.maximum(sx, sy) < 4 * SPAN)
        picked = [k for k in np.nonzero(sel)[0] if _int32_setup_peak(g, k) >= 2 ** 31][:4]
        assert len(picked) == 4, "too few quads at %s" % (xs,)
        parts.append(C[picked])
    S = np.concatenate(parts)
    S["count"][1::3], S["timestamp"][1::3] = OLD
    S["count"][2::3], S["timestamp"][2::3] = BOTH
    cls = check("corner span on both axes", SPAN2_IMAGE, S, (RR.LARGE_SPAN,), poses=((EYE, EYE), (EYE, SHIFT)))
    assert all(c[0] == RR.LARGE_SPAN and c[1] < 12 and c[2] < 5 for c in cls), cls


# ---------------------------------------------------------------------------------------------------------------
# 3. azimuth seam
# ---------------------------------------------------------------------------------------------------------------
def test_azimuth_seam():
    """centres within an ulp of x = 0 and of x -> 1 with corners pulled across the seam by +-1, and a quad whose corners
    spread over more than half the image width (the seam rule keeps them within half a turn of the centre)"""
    po, _ = both_params(**BASE)
    m = RR.Model(po)
    parts, info = [], []
    for side in (1.0, -1.0):   # +y: x just above 0; -y: x just below 1
        for rad in (0.002, 0.03, 0.3):
            for e in 10.0 ** np.arange(-8, -3.9, 0.25):
                p = np.array([-10.0, side * e, 0.0])
                S = make_surfels(p, -p / np.linalg.norm(p), rad, NEW)
                g = geometry(po, S)
                cx = RR.project01(g.pp, m.fov_up, m.fov, m.min_depth, m.max_depth)[0][0]
                if g.alive[0] and (cx < F(2.0 ** -18) or cx > F(1) - F(2.0 ** -18)):
                    parts.append(S)
                    info.append(float(cx))
    assert min(info) <= 2.0 ** -23 and max(info) >= 1 - 2.0 ** -23, info   # within an ulp of the seam on both sides
    # a horizontal quad under the sensor, reaching behind it: its corners spread over almost a whole turn of azimuth
    wide = make_surfels(np.array([2.5, 0.0, -0.1]), np.array([0.0, 0.0, 1.0]), 40.0, BOTH)
    S = np.concatenate(parts + [wide])
    S["count"][:-1:2], S["timestamp"][:-1:2] = OLD
    g = geometry(po, S)
    i0, i1, _, _, _ = boxes(g)
    assert g.alive[-1] and g.X[-1].max() - g.X[-1].min() > 0.5 * 256 * m.W, g.X[-1]
    crossed = [k for k in range(len(S) - 1) if g.X[k].min() < 0 or g.X[k].max() > 256 * m.W]
    assert crossed, "no corner pulled across the seam"
    check("azimuth seam", {}, S, (RR.SMALL, RR.LARGE_BOX), poses=((EYE, EYE), (EYE, SHIFT)))


# ---------------------------------------------------------------------------------------------------------------
# 4. degenerate geometry
# ---------------------------------------------------------------------------------------------------------------
def test_degenerate_geometry():
    """quads covering no pixel centre, quads whose snapped triangles have zero area (one or both), and quads whose
    projected corners cross so that the two triangles overlap"""
    po, _ = both_params(**BASE)
    m = RR.Model(po)
    rng = np.random.default_rng(5)
    N = 60000
    # tiny quads around pixel centres: the snapped corners are a few units apart
    i, j = rng.integers(10, m.W - 10, N), rng.integers(3, m.H - 3, N)
    jit = rng.uniform(-3, 3, (N, 2)) / 256
    dirs = direction(m, (i + 0.5 + jit[:, 0]) / m.W, (j + 0.5 + jit[:, 1]) / m.H)
    dist = rng.uniform(5, 30, N)
    nrm = -dirs + 0.8 * rng.normal(size=(N, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    C = make_surfels(dirs * dist[:, None], nrm, dist * rng.uniform(0.2, 6, N) / 256 * (2 * np.pi / m.W), NEW)
    g = geometry(po, C)
    i0, i1, j0, j1, _ = boxes(g)
    nonempty = g.alive & (i0 <= i1) & (j0 <= j1)
    picks = {"empty": np.nonzero(g.alive & ~((i0 <= i1) & (j0 <= j1)))[0][:4]}
    want = {"both zero": lambda a: a[0] == 0 and a[1] == 0, "first zero": lambda a: a[0] == 0 and a[1] != 0,
            "second zero": lambda a: a[0] != 0 and a[1] == 0}
    for key, pred in want.items():
        picks[key] = [k for k in np.nonzero(nonempty)[0][:20000] if pred(tri_areas(g, k))][:4]
    # crossed corners: same orientation of both strip triangles (an ordinary quad has opposite ones)
    B = random_quads(rng, po, 40000, d=(2.2, 6.0), rpx=(4.0, 300.0), tilt=3.0)
    gb = geometry(po, B)
    crossed = [k for k in np.nonzero(gb.alive)[0] if (lambda a: a[0] * a[1] > 0)(tri_areas(gb, k))][:6]
    log("degenerate picks:", {k: len(v) for k, v in picks.items()}, "crossed:", len(crossed))
    assert all(len(v) for v in picks.values()) and crossed, ({k: len(v) for k, v in picks.items()}, len(crossed))
    S = np.concatenate([C[np.concatenate([np.asarray(v, np.int64) for v in picks.values()])], B[crossed]])
    S["count"][1::3], S["timestamp"][1::3] = OLD
    S["count"][2::3], S["timestamp"][2::3] = BOTH
    check("degenerate geometry", {}, S, (RR.EMPTY, RR.SMALL))


# ---------------------------------------------------------------------------------------------------------------
# 5. tie rule
# ---------------------------------------------------------------------------------------------------------------
def _diamonds(po):
    """quads facing the sensor along +x / -x / +y / -y at pitch 0: the shared diagonal (corners 1, 2) runs along a row
    or a column of the image; along the x axes its two ends are tuned onto pixel centres 1..5 and 20 pixels apart"""
    m = RR.Model(po)
    out = []
    for axis in ([1.0, 0.0, 0.0], [-1.0, 0.0, 0.0]):
        p = np.array(axis) * 10.0
        n = -np.array(axis)
        g0 = geometry(po, make_surfels(p, n, 0.01, NEW))
        Xc = int(g0.X[0, 1] + g0.X[0, 2]) // 2
        for half in (1, 2, 3, 4, 5, 20):
            r = bisect(0.0005, 2.0, lambda r: abs(int(geometry(po, make_surfels(p, n, r, NEW)).X[0, 1]) - Xc), 256 * half)
            if r is not None:
                out.append(make_surfels(p, n, r, NEW))
    rng = np.random.default_rng(3)
    for axis in ([0.0, 1.0, 0.0], [0.0, -1.0, 0.0], [0.6, 0.8, 0.0], [-0.8, 0.6, 0.0]):
        for r in rng.uniform(0.02, 0.4, 6):
            out.append(make_surfels(np.array(axis) * 10.0, -np.array(axis), r, NEW))
    return np.concatenate(out)


def test_tie_rule():
    """snapped vertices on pixel centres and shared diagonals through pixel centres in several directions, both
    orientations of the strip triangles (the phase-2 corner mapping of the "swapped" bit). The property "every pixel centre
    strictly inside the shared diagonal is covered by exactly one of the two triangles" is checked on the reference's
    rasteriser, independently of any winner image; the kernel is held to the reference by the bit-exact comparison of
    every output that follows."""
    po, _ = both_params(**BASE)
    S = _diamonds(po)
    g = geometry(po, S)
    on_centres, tested, orient = 0, 0, set()
    for k in np.nonzero(g.alive)[0]:
        a = tri_areas(g, k)
        orient.update(np.sign(a).tolist())
        X, Y = [int(v) for v in g.X[k]], [int(v) for v in g.Y[k]]
        if X[1] % 256 == 128 and Y[1] % 256 == 128 and X[2] % 256 == 128 and Y[2] % 256 == 128:
            on_centres += 1
        corners = [(X[i], Y[i], g.Z[k, i], F(1), F(1)) for i in range(4)]
        cover = [RR.triangle(corners[t], corners[t + 1], corners[t + 2], g.m.W, g.m.H) for t in range(2)]
        cover = [set() if c is None else set(c[0].tolist()) for c in cover]
        # pixel centres strictly between corners 1 and 2 on the diagonal
        dx, dy = X[2] - X[1], Y[2] - Y[1]
        for ci in range(max(min(X[1], X[2]) // 256 - 1, 0), min(max(X[1], X[2]) // 256 + 2, g.m.W)):
            for cj in range(max(min(Y[1], Y[2]) // 256 - 1, 0), min(max(Y[1], Y[2]) // 256 + 2, g.m.H)):
                Xc, Yc = ci * 256 + 128, cj * 256 + 128
                if dx * (Yc - Y[1]) - dy * (Xc - X[1]) != 0 or (Xc, Yc) in ((X[1], Y[1]), (X[2], Y[2])):
                    continue
                if not (min(X[1], X[2]) <= Xc <= max(X[1], X[2]) and min(Y[1], Y[2]) <= Yc <= max(Y[1], Y[2])):
                    continue
                pix = cj * g.m.W + ci
                assert (pix in cover[0]) + (pix in cover[1]) == 1, (k, ci, cj)
                tested += 1
    log("tie rule: %d quads with both diagonal ends on pixel centres, %d diagonal centres tested, orientations %s" %
          (on_centres, tested, orient))
    assert on_centres >= 4 and tested >= 20 and orient >= {-1, 1}
    S["count"][1::3], S["timestamp"][1::3] = OLD
    S["count"][2::3], S["timestamp"][2::3] = BOTH
    check("tie rule", {}, S, (RR.SMALL, RR.LARGE_BOX), poses=((EYE, EYE), (EYE, SHIFT)))


# ---------------------------------------------------------------------------------------------------------------
# 6. depth ties
# ---------------------------------------------------------------------------------------------------------------
def test_depth_ties():
    """equal depth24 between different surfels in one warp, in two warps of one block, and in blocks 256 and 4096
    indices apart; every class pairing (old, new, old and re-observed), so that GL_LESS keys, the composed GL_LEQUAL keys,
    plain mode and its emit_fragment fall-back for class-3 surfels all resolve a tie"""
    po, _ = both_params(**BASE)
    m = RR.Model(po)
    base = np.array([10.0, 0.0, 0.0])
    pairs = [(3, 17), (40, 200), (300, 300 + 256), (600, 600 + 4096)]
    classes = [(OLD, OLD), (NEW, NEW), (BOTH, BOTH), (OLD, NEW), (NEW, BOTH), (BOTH, OLD)]
    S = culled(600 + 4096 + 300)
    ties = 0
    for q, (a, b) in enumerate(pairs):
        for c, (ca, cb) in enumerate(classes):
            x = (q * len(classes) + c + 0.5) / (len(pairs) * len(classes)) * 0.8 + 0.1
            dirv = direction(m, x, 0.5)
            p = dirv * 10.0
            n = -dirv
            off = a + 10 * c if a + 10 * c < b else a + c
            ka, kb = off, b + c if b != a else off + 1
            one = make_surfels(np.stack([p, p + np.array([0.0, 0.0, 4e-6])]), np.stack([n, n]), 0.06 if c % 2 else 0.3, NEW,
                               seed=ka)
            one["count"], one["timestamp"] = np.array([ca, cb]).T
            S[ka], S[kb] = one[0], one[1]
            g = geometry(po, one)
            fa, fb = (dict(zip(*[np.concatenate(v) for v in zip(*RR.quad_fragments(g, k))])) for k in (0, 1))
            ties += sum(1 for pix, d in fa.items() if fb.get(pix) == d)
    log("depth ties: %d pixels where a pair's depth24 values are equal" % ties)
    assert ties > 100
    check("depth ties", {}, S, (RR.SMALL, RR.LARGE_BOX, RR.CULLED), poses=((EYE, EYE), (EYE, SHIFT)))


# ---------------------------------------------------------------------------------------------------------------
# 7. z clip
# ---------------------------------------------------------------------------------------------------------------
def test_z_clip():
    """quads whose corners straddle model_min_depth and model_max_depth (the centre inside the range); facing quads
    whose four corners lie exactly at model_max_depth: fragments at z = 1 (GL_LEQUAL passes them against the cleared
    depth, GL_LESS does not) and just beyond; and a tiny quad centred on a pixel centre at exactly model_min_depth, whose
    corners' window depth rounds to exactly 0, so its fragment has z = 0 (kept by the near clip, depth24 = 0)"""
    po, _ = both_params(**BASE)
    m = RR.Model(po)
    parts = []
    for k, x in enumerate(np.linspace(0.1, 0.9, 8)):
        dirv = direction(m, x, 0.5)
        tilt = np.array([0.0, 0.0, 1.0]) if k % 2 else np.cross(dirv, [0.0, 0.0, 1.0])
        n = -dirv * 0.3 + tilt
        n /= np.linalg.norm(n)
        near, far = float(m.min_depth) + 0.004, float(m.max_depth) - 0.03
        r = (0.012 if k % 2 else 0.4) if k < 4 else (0.6 if k % 2 else 2.0)   # small and large quads at each end
        parts.append(make_surfels(dirv * (near if k < 4 else far), n, r, NEW))
    ones = 0
    for x in np.linspace(0.15, 0.85, 6):
        dirv = direction(m, x, 0.5 + 0.5 / m.H)
        r = 1.5

        def corner_depth(d):
            g = geometry(po, make_surfels(dirv * float(d), -dirv, r, NEW))
            return int(np.sign(float(g.Z[0].max()) - 1.0))
        d = bisect(70.0, 75.0, corner_depth, 0)
        if d is None:
            continue
        S = make_surfels(dirv * float(d), -dirv, r, NEW)
        g = geometry(po, S)
        z = [zz for k in (0,) for _, dd in RR.quad_fragments(g, k) for zz in dd]
        ones += sum(1 for v in z if v == RR.DEPTH_CLEAR)
        parts.append(S)
    # pitch 0 and yaw 0 fall on the centre of pixel (720, 16); 2 m is exactly model_min_depth, so the centre has z = 0
    zero = make_surfels(np.array([float(m.min_depth), 0.0, 0.0]), np.array([-1.0, 0.0, 0.0]), 1e-3, NEW)
    gz = geometry(po, zero)
    assert gz.alive[0] and (gz.Z[0] == 0).all(), gz.Z[0]
    zeros = sum(int((d == 0).sum()) for _, d in RR.quad_fragments(gz, 0))
    S = np.concatenate(parts + [zero])
    S["count"][1::3], S["timestamp"][1::3] = OLD
    S["count"][2::3], S["timestamp"][2::3] = BOTH
    g = geometry(po, S)
    zc = g.Z[:8]
    assert (zc.min(1)[:4] < 0).all() and (zc.max(1)[4:8] > 1).all(), zc
    log("z clip: %d fragments at z = 1 exactly, %d at z = 0 exactly" % (ones, zeros))
    assert ones > 0 and zeros > 0
    check("z clip", {}, S, (RR.SMALL, RR.LARGE_BOX), poses=((EYE, EYE), (EYE, SHIFT)))


# ---------------------------------------------------------------------------------------------------------------
# 8. block loads
# ---------------------------------------------------------------------------------------------------------------
def test_block_loads():
    """block 0: 256 large quads (32 per warp in the warp loop); block 1: 256 maximal small boxes (12 x 5 = 60 pixels,
    15 360 flattened pixels, a chunk of 60 per thread); block 2: one survivor among 255 culled surfels; block 3: nothing
    survives stage A"""
    po, _ = both_params(**BASE)
    rng = np.random.default_rng(13)
    C = random_quads(rng, po, 60000, rpx=(3.0, 14.0), tilt=1.2)
    g = geometry(po, C)
    i0, i1, j0, j1, span = boxes(g)
    big = np.nonzero(g.alive & (i1 - i0 >= 12) & (i1 - i0 <= 24) & (j1 - j0 <= 8))[0]
    maxi = np.nonzero(g.alive & (i1 - i0 == 11) & (j1 - j0 == 4) & (span < SPAN))[0]
    assert len(big) >= 256 and len(maxi) >= 16, (len(big), len(maxi))
    lone = culled(256)
    lone[137] = C[maxi[0]]
    S = np.concatenate([C[big[:256]], C[np.resize(maxi, 256)], lone, culled(256)])   # repeats tie in depth
    S["count"][1::3], S["timestamp"][1::3] = OLD
    S["count"][2::3], S["timestamp"][2::3] = BOTH
    cls = check("block loads", {}, S, (RR.SMALL, RR.LARGE_BOX, RR.CULLED))
    assert all(c[0] == RR.LARGE_BOX for c in cls[:256])
    assert all(c == (RR.SMALL, 11, 4) for c in cls[256:512])
    assert [k for k, c in enumerate(cls[512:768]) if c[0] != RR.CULLED] == [137]
    assert all(c[0] == RR.CULLED for c in cls[768:])


# ---------------------------------------------------------------------------------------------------------------
# 9. the model width limit
# ---------------------------------------------------------------------------------------------------------------
def test_model_width_65536():
    """model_width = 65536, the widest the 16-bit box packing addresses: small quads whose boxes start at column 65535
    (i0 = 0xffff) on the last row, large quads through column 65535 on the last row, small ones ending at column 65535
    on the first and the last row"""
    kw = dict(model_width=65536, model_height=4)
    po, _ = both_params(**dict(BASE, **kw))
    m = RR.Model(po)
    rng = np.random.default_rng(17)
    N = 40000
    found = {}
    for row in (m.H - 1, 0):   # centres within a thousandth of a row of the row's pixel centres
        C = random_quads(rng, po, N, x=(1.0 - 3.0 / m.W, 1.0 - 0.2 / m.W), y=((row + 0.499) / m.H, (row + 0.501) / m.H),
                         d=(5.0, 20.0), rpx=(0.3, 40.0), tilt=0.5)
        g = geometry(po, C)
        i0, i1, j0, j1, span = boxes(g)
        small = (i1 - i0 < 12) & (j1 - j0 < 5) & (span < SPAN)
        last = g.alive & (i0 <= i1) & (j0 <= j1) & (j1 == m.H - 1)
        first = g.alive & (i0 <= i1) & (j0 <= j1) & (j0 == 0)
        for key, sel in (("small at 65535, last row", last & (i0 == m.W - 1) & small),
                         ("large through 65535, last row", last & (i1 == m.W - 1) & ~small),
                         ("small ending at 65535, last row", last & (i1 == m.W - 1) & (i0 < m.W - 1) & small),
                         ("small ending at 65535, first row", first & (i1 == m.W - 1) & small)):
            idx = np.nonzero(sel)[0]
            if len(idx) and key not in found:
                found[key] = C[idx[:3]]
    log("model width 65536:", {k: len(v) for k, v in found.items()})
    assert "small at 65535, last row" in found and "large through 65535, last row" in found, list(found)
    S = np.concatenate(list(found.values()))
    S["count"][1::3], S["timestamp"][1::3] = OLD
    S["count"][2::3], S["timestamp"][2::3] = BOTH
    check("model width 65536", kw, S, (RR.SMALL, RR.LARGE_BOX))


def test_every_regime_was_reached():
    """the cases above together reach every regime of the kernel (runs last in this file)"""
    if not SEEN:
        pytest.skip("needs the cases above in the same run")
    for kind in (RR.CULLED, RR.EMPTY, RR.SMALL, RR.LARGE_BOX, RR.LARGE_SPAN):
        assert SEEN[kind] > 0, (kind, dict(SEEN))


# ---------------------------------------------------------------------------------------------------------------
# the model-side rule
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h,ok", [(65537, 1, False), (1, 65537, False), (65536, 1, True), (1, 65536, True)])
def test_model_side_over_65536_is_refused(w, h, ok):
    """sb_create and the oracle refuse a model image with a side over 65536 (the render pass packs pixel boxes in 16
    bits per axis) and accept 65536"""
    po, pp = both_params(data_width=360, data_height=32, model_width=w, model_height=h)
    why = "model image side > 65536 (the render pass packs pixel boxes in 16 bits)"
    assert O.check_params(po) == (None if ok else why)
    if ok:
        api.Context(pp).close()
        return
    with pytest.raises(api.SumaError, match="INVALID"):
        api.Context(pp)
    with pytest.raises(ValueError, match="16 bits"):
        O.Map(po)
