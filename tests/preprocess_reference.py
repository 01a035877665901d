"""An exact numpy model of the preprocessing pass K1-K3 (gen_vertexmap.vert/.frag, gen_normalmap.frag, floodfill.frag),
written from the shaders' rules and the GL table of DESIGN.md section 2. It shares no code with the oracle or the library.

* Every +, *, /, sqrt is one numpy float32 operation in the kernels' order, no FMA: len3 = sqrt((x*x + y*y) + z*z),
  normalize3 divides each component by it, cross3 as in csrc/sb_math.cuh.
* The pixel a point lands on is computed in fp64 from its fp32 coordinates. The pinned atan2f_ / asinf_ polynomials err
  by a few ulps, so every designed point lies at least PIXEL_MARGIN pixels from a pixel edge and the model asserts it.
  One exception is exact: the azimuth seam. The pinned atan2 tests `y < 0`, so it ignores the sign of zero, and a
  quotient |y| / |x| below half an ulp of pi leaves yaw = +-pi in fp32: a point with x < 0 and y = +-0 (or y = +1 ulp)
  lands in column 0, one with y = -1 ulp gives x = 1 and fx = W, and is clipped. IEEE atan2(-0, x < 0) = -pi would clip
  the y = -0 point too.
* The normalised depth z, 0.5 z + 0.5 and depth24 (fp64 product, rounded half to even) are exact; the z-buffer is
  GL_LESS in buffer order: the lowest point index wins a tie.
* The radius map of the pipeline instance is update_reference.radius_pixel, applied to the model's own maps.
"""
import math

import numpy as np

import update_reference as UR

f32 = np.float32
PIXEL_MARGIN = 1e-3
DEPTH_CLEAR = 0xFFFFFF
MOVABLE = UR.MOVABLE
SEAM_RATIO = 2.0 ** -30  # |y| / |x| below this: atan_poly(t) = t < ulp(pi) / 2, yaw = +-pi exactly
LEN_EPS = f32(0.0000001)
FILL_THR = f32(0.007)
ONE, ZERO = f32(1.0), f32(0.0)
LEN_ABOVE = np.nextafter(LEN_EPS, ONE) * f32(16)  # "normal:len_above": 1e-7 < len <= this
# every branch tag the model can report (a _Tags set refuses any other)
TAGS = frozenset([
    "point:won", "point:won_tie", "point:lost_tie", "point:lost_nearer", "point:clipped", "point:z_below",
    "point:z_above", "point:z_minus_one", "point:d24_clear", "point:d24_top", "seam:col0", "seam:clipped",
    "point:movable_removed", "point:movable_kept", "q1:label_past_n", "q1:prob_past_n",
    "normal:no_vertex", "normal:uv_both", "normal:st_both", "normal:u_or_v", "normal:only_v_missing", "normal:valid",
    "normal:len_nan", "normal:len_zero", "normal:len_eq", "normal:len_below", "normal:len_above", "normal:across_seam",
    "erode:by_u", "erode:by_v", "erode:by_s", "erode:by_t", "erode:zero_neighbour", "erode:kept", "erode:eroded",
    "erode:across_seam",
    "fill:labelled", "fill:none", "fill:no_vertex", "fill:equal_rejected", "fill:priority", "fill:across_seam"] +
    ["fill:o%d_%s" % (o, d) for o in (1, 2) for d in ("+x", "+y", "-x", "-y")])


class _Tags(set):
    def add(self, t):
        assert t in TAGS, "tag %r is not in TAGS" % t
        set.add(self, t)


def len3(a):
    return np.sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2])


def sub3(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def normalize3(a):
    n = len3(a)
    return (a[0] / n, a[1] / n, a[2] / n)


def cross3(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def v3(*a):
    return tuple(f32(x) for x in a)


def depth24(zw):
    return int(np.rint(np.float64(zw) * 16777215.0))


def is_movable(label):
    return float(label) in MOVABLE


def fovs(p):
    up = f32(abs(f32(p.data_fov_up)))
    return up, f32(up + f32(abs(f32(p.data_fov_down))))


def pixel_coords(p, v):
    """(px, py) in fp64 pixel units, (None, None) for a point at the origin"""
    x, y, z = (float(c) for c in v)
    d = math.sqrt(x * x + y * y + z * z)
    if not (math.isfinite(d) and d > 0.0):
        return None, None
    up, fov = fovs(p)
    if x < 0.0 and abs(y) <= abs(x) * SEAM_RATIO:  # the seam rule (module docstring)
        px = float(p.data_width) if y < 0.0 else 0.5
    else:
        px = 0.5 * (-math.atan2(y, x) / math.pi + 1.0) * p.data_width
    py = (1.0 - (math.degrees(-math.asin(z / d)) + float(up)) / float(fov)) * p.data_height
    return px, py


def pixel_of(p, v):
    """(column, row) of point v, the margin to the nearest pixel edge asserted; None if clipped. The second value tags
    the seam rule ("seam:col0", "seam:clipped") or is None."""
    px, py = pixel_coords(p, v)
    if px is None:
        return None, None
    seam = None
    x, y = float(v[0]), float(v[1])
    if x < 0.0 and abs(y) <= abs(x) * SEAM_RATIO:
        seam = "seam:clipped" if y < 0.0 else "seam:col0"
    else:
        assert abs(px - round(px)) >= PIXEL_MARGIN, "point %s lies within %g px of a column edge" % (v, PIXEL_MARGIN)
    assert abs(py - round(py)) >= PIXEL_MARGIN, "point %s lies within %g px of a row edge" % (v, PIXEL_MARGIN)
    fx, fy = math.floor(px), math.floor(py)
    if not (0 <= fx < p.data_width and 0 <= fy < p.data_height):
        return None, seam
    return (fx, fy), seam


def depth_z(p, v):
    """the kernel's z = 2 ((d - min) / (max - min)) - 1, fp32"""
    d = len3(v3(*v))
    return f32(2.0) * ((d - f32(p.min_depth)) / (f32(p.max_depth) - f32(p.min_depth))) - ONE


def point_d24(p, v):
    """(d24 or None if the depth test or the clip drops it, tag)"""
    z = depth_z(p, v)
    if not (z >= f32(-1.0) and z <= ONE):
        return None, "point:z_below" if z < f32(-1.0) else "point:z_above"
    d24 = depth24(f32(0.5) * z + f32(0.5))
    if d24 >= DEPTH_CLEAR:
        return None, "point:d24_clear"
    tag = "point:z_minus_one" if z == f32(-1.0) else ("point:d24_top" if d24 == DEPTH_CLEAR - 1 else None)
    return d24, tag


def preprocess(p, pts, labels=None, probs=None, timestamp=100):
    """K1-K3 of one scan. pts: float32 [n, 4]. Returns dict(vertex, normal, semantic, radius (float32 [H, W, 4]),
    point_tags (a set per point), pixel_tags ({(row, col): set}))."""
    with np.errstate(all="ignore"):
        return _preprocess(p, np.asarray(pts, f32).reshape(-1, 4), labels, probs, timestamp)


def _preprocess(p, pts, labels, probs, timestamp):
    H, W = p.data_height, p.data_width
    n = len(pts)
    isfirst = timestamp < 10
    ptags = [_Tags() for _ in range(n)]
    # ---- K1: projection and z-buffer (GL_LESS, buffer order) ----
    best = {}
    for i in range(n):
        v = v3(*pts[i, :3])
        pix, seam = pixel_of(p, v)
        if seam:
            ptags[i].add(seam)
        if pix is None:
            ptags[i].add("point:clipped")
            continue
        d24, tag = point_d24(p, v)
        if tag:
            ptags[i].add(tag)
        if d24 is None:
            continue
        key = (pix[1], pix[0])
        if key not in best or d24 < best[key][0]:
            if key in best:
                ptags[best[key][1]].add("point:lost_nearer")
            best[key] = (d24, i)
        else:
            ptags[i].add("point:lost_tie" if d24 == best[key][0] else "point:lost_nearer")
            if d24 == best[key][0]:
                ptags[best[key][1]].add("point:won_tie")
    V = np.zeros((H, W, 4), f32)
    raw = np.zeros((H, W, 2), f32)  # (label / 255, prob)
    ql = 4 if p.label_offset_quirk else 0
    for (y, x), (_, i) in best.items():
        ptags[i].add("point:won")
        lab = prob = ZERO
        if labels is not None:
            li = i + ql
            if li < n:
                lab = f32(labels[li])
            elif ql:
                ptags[i].add("q1:label_past_n")
        if probs is not None:
            pi = i + (ql + 1 if ql else 0)
            if pi < n:
                prob = f32(probs[pi])
            elif ql:
                ptags[i].add("q1:prob_past_n")
        if isfirst and is_movable(lab):
            ptags[i].add("point:movable_removed")
        else:
            V[y, x] = (pts[i, 0], pts[i, 1], pts[i, 2], 1.0)
            if is_movable(lab):
                ptags[i].add("point:movable_kept")
        raw[y, x] = (lab / f32(255.0), prob)

    tags = {(y, x): _Tags() for y in range(H) for x in range(W)}

    def at(img, y, x):  # rows outside: border 0; columns wrap once
        if y < 0 or y >= H:
            return np.zeros(img.shape[2], f32)
        return img[y, x % W]

    # ---- K2: normals and label erosion ----
    N = np.zeros((H, W, 4), f32)
    ero = np.zeros((H, W, 2), f32)
    for y in range(H):
        for x in range(W):
            t = tags[(y, x)]
            N[y, x] = (0, 0, 0, 1)
            ero[y, x] = (0, 1)
            P = V[y, x]
            if not P[3] > ZERO:
                t.add("normal:no_vertex")
                continue
            U, Vn, S, T = at(V, y, x + 1), at(V, y + 1, x), at(V, y, x - 1), at(V, y - 1, x)
            nw = True
            if U[3] < ONE and Vn[3] < ONE:
                nw = False
                t.add("normal:uv_both")
            if S[3] < ONE and T[3] < ONE:
                nw = False
                t.add("normal:st_both")
            if not (U[3] > f32(0.5)) or not (Vn[3] > f32(0.5)):
                nw = False
                t.add("normal:u_or_v")
                if U[3] > f32(0.5) and not (S[3] < ONE and T[3] < ONE):
                    t.add("normal:only_v_missing")
            if nw:
                pp = v3(*P[:3])
                u = normalize3(sub3(v3(*U[:3]), pp))
                v = normalize3(sub3(v3(*Vn[:3]), pp))
                w = cross3(u, v)
                ln = len3(w)
                N[y, x] = (w[0] / ln, w[1] / ln, w[2] / ln, ONE if ln > LEN_EPS else ZERO)
                if ln != ln:
                    t.add("normal:len_nan")
                elif ln == ZERO:
                    t.add("normal:len_zero")
                elif ln == LEN_EPS:
                    t.add("normal:len_eq")
                elif ln < LEN_EPS:
                    t.add("normal:len_below")
                elif ln <= LEN_ABOVE:
                    t.add("normal:len_above")
                else:
                    t.add("normal:valid")
                if x == W - 1:
                    t.add("normal:across_seam")
            else:
                N[y, x] = (0, 0, 0, 0)
            # erosion: only where a vertex exists; a neighbour whose label is 0 never erodes
            pl = raw[y, x, 0]
            ero[y, x] = raw[y, x]
            for name, (yy, xx) in (("u", (y, x + 1)), ("v", (y + 1, x)), ("s", (y, x - 1)), ("t", (y - 1, x))):
                q = at(raw, yy, xx)[0]
                if pl != q and q != ZERO:
                    ero[y, x] = (0, 1)
                    t.add("erode:by_" + name)
                    if not 0 <= xx < W:
                        t.add("erode:across_seam")
                elif pl != q:
                    t.add("erode:zero_neighbour")
            if ero[y, x, 0] == ZERO and raw[y, x, 0] != ZERO:
                t.add("erode:eroded")
            elif raw[y, x, 0] != ZERO:
                t.add("erode:kept")
    # ---- K3: flood fill (offset 1 then 2; +x, +y, -x, -y; the first hit wins) ----
    Sm = np.zeros((H, W, 4), f32)
    for y in range(H):
        for x in range(W):
            t = tags[(y, x)]
            e = ero[y, x]
            Sm[y, x] = (e[0], e[0], e[0], e[1])
            if e[0] != ZERO:
                t.add("fill:labelled")
                continue
            lp = len3(v3(*V[y, x, :3]))
            thr = FILL_THR * lp
            hits = []
            for off in (1, 2):
                for k, (dy, dx) in enumerate(((0, 1), (1, 0), (0, -1), (-1, 0))):
                    q = at(ero, y + dy * off, x + dx * off)
                    if q[0] == ZERO:
                        continue
                    lq = len3(v3(*at(V, y + dy * off, x + dx * off)[:3]))
                    diff = abs(lp - lq)
                    if diff < thr:
                        hits.append((off, k, q))
                    elif diff == thr:
                        t.add("fill:equal_rejected")
            if not hits:
                t.add("fill:none" if V[y, x, 3] > ZERO else "fill:no_vertex")
                continue
            off, k, q = hits[0]
            if len(hits) > 1:
                t.add("fill:priority")
            t.add("fill:o%d_%s" % (off, "+x +y -x -y".split()[k]))
            if not 0 <= x + (off if k == 0 else (-off if k == 2 else 0)) < W:
                t.add("fill:across_seam")
            Sm[y, x] = (q[0], q[0], q[0], q[1] / f32(off + 1))
    d = UR.derived(p)
    R = np.zeros((H, W, 4), f32)
    for y in range(H):
        for x in range(W):
            R[y, x] = UR.radius_pixel(p, d, V[y, x], N[y, x])[0]
    return dict(vertex=V, normal=N, semantic=Sm, radius=R, point_tags=ptags, pixel_tags=tags)
