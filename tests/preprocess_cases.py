"""Designed inputs of the preprocessing pass (K1-K3) at its thresholds, shared by tests/test_gpu_preprocess_edges.py
(CUDA, oracle, model) and tests/test_preprocess_edges_ref.py (the reference's shaders, oracle, model), so that the two
cannot drift.

A case is a point list with labels and probabilities, a timestamp and parameter overrides, plus the branches
tests/preprocess_reference.py must report for given points and pixels. Points are placed on beam centres (the
direction through a pixel's centre, as test_gpu_shapes._beam_centres) or, where a case needs it, at a stated
fractional position inside the pixel, always at least preprocess_reference.PIXEL_MARGIN from its edges. Each threshold
is put at equality and one step either side in the quantity the kernel compares, found by searching over fp32 scales
along the beam:
  * the depth test: len3 of the point, hence z and depth24;
  * the flood fill: |lp - lq| against 0.007 lp. lp - lq is exact, so equality needs 0.007 lp to be a multiple of
    ulp(lp): the search scales P until it is, then puts lq at lp + 0.007 lp exactly. One step either side is one ulp of
    lq, which moves |lp - lq| by ulp(lp), the finest step the difference has;
  * the normal's len > 1e-7: len = 0 exactly (normals_collinear), 0 < len < 1e-7 (normals_len_below) and the smallest
    len above 1e-7 a search reaches (normals_len_above, between 1.2e-7 and 6.3e-7). len = 1e-7f itself is not built
    (see normals_len_above).
"""
import functools
import math

import numpy as np

import preprocess_reference as M

f32 = np.float32
SHAPES = [(40, 96), (37, 77), (16, 4), (16, 5)]
FOV_UP, FOV_DOWN = 3.0, -25.0


def nxt(x, n=1):
    x = f32(x)
    for _ in range(abs(n)):
        x = np.nextafter(x, f32(np.inf) if n > 0 else f32(-np.inf))
    return x


def direction(H, W, row, col):
    """unit direction (fp64) through the image position (col, row), both fractional: col + 0.5, row + 0.5 is a pixel's
    beam centre (test_gpu_shapes._beam_centres)"""
    fov = FOV_UP - FOV_DOWN
    az = math.pi * (1.0 - 2.0 * col / W)
    el = math.radians(FOV_UP - fov * (1.0 - row / H))
    return np.array([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)])


def point(H, W, row, col, depth, fx=0.5, fy=0.5):
    return (direction(H, W, row + fy, col + fx) * depth).astype(f32)


def with_len(d, L):
    """an fp32 point near the ray d whose len3 is exactly L (searched over ulps of two components)"""
    base = (d * float(L)).astype(f32)
    k = np.arange(-48, 49)
    i, j = np.meshgrid(k, k, indexing="ij")
    ax = np.argsort(-np.abs(d))[:2]
    q = np.broadcast_to(base, i.shape + (3,)).copy()
    for a, kk in zip(ax, (i, j)):
        step = np.spacing(np.abs(base[a]))
        q[..., a] = (base[a].astype(np.float64) + kk * float(step)).astype(f32)
    ln = np.sqrt((q[..., 0] * q[..., 0] + q[..., 1] * q[..., 1]) + q[..., 2] * q[..., 2])
    hit = np.argwhere(ln == f32(L))
    assert len(hit), "no point of length %r on the ray" % L
    return q[tuple(hit[len(hit) // 2])]


class Case:
    def __init__(self, name, H, W, timestamp=100, kw=None):
        self.name, self.H, self.W, self.timestamp = name, H, W, timestamp
        self.kw = dict(dict(label_offset_quirk=0), **(kw or {}))  # labels pair with their points unless a case says
        self.pts, self.labels, self.probs = [], [], []
        self.expect_pt, self.expect_pix = [], []

    def params(self, P):
        return P.default_params(data_width=self.W, model_width=self.W, data_height=self.H, model_height=self.H,
                                **self.kw)

    def add(self, p, label=0.0, prob=0.0, *tags):
        self.pts.append((float(p[0]), float(p[1]), float(p[2]), 1.0))
        self.labels.append(label)
        self.probs.append(prob)
        for t in tags:
            self.expect_pt.append((len(self.pts) - 1, t))
        return len(self.pts) - 1

    def at(self, row, col, depth, label=0.0, prob=0.0, *tags, fx=0.5, fy=0.5):
        return self.add(point(self.H, self.W, row, col, depth, fx, fy), label, prob, *tags)

    def pad_to(self, n):
        """filler points above fov_up (clipped) up to index n - 1"""
        while len(self.pts) < n:
            self.add(point(self.H, self.W, self.H + 3, len(self.pts) % self.W, 10.0), 0.0, 0.0, "point:clipped")

    def expect(self, row, col, *tags):
        for t in tags:
            self.expect_pix.append(((row % self.H, col % self.W), t))

    def arrays(self):
        pts = np.array(self.pts, f32).reshape(-1, 4)
        return pts, np.array(self.labels, f32), np.array(self.probs, f32)


def _params(c):
    from oracle import oracle as O
    return c.params(O)


# ---- K1: the depth test ------------------------------------------------------------------------------------------------
def _d24(c, q):
    return M.point_d24(_params(c), q)[0]


def depth_ties(H, W):
    """equal d24 from equal and from different depths, a later point one d24 nearer, and three-way ties across a warp
    (31 / 32 / 64) and a block (255 / 256 / 257) of the scatter"""
    c = Case("depth_ties", H, W)
    r = H // 2
    d = direction(H, W, r + 0.5, 0.5)
    p = (d * 10.0).astype(f32)
    c.add(p, 0, 0, "point:won", "point:won_tie")
    c.add(p, 0, 0, "point:lost_tie")                                  # the same bits
    # different lengths, one d24: scale until len3 changes and d24 does not
    base = _d24(c, p)
    s = next(nxt(10.0, k) for k in range(1, 64) if M.len3(tuple((d * float(nxt(10.0, k))).astype(f32))) != M.len3(tuple(p))
             and _d24(c, (d * float(nxt(10.0, k))).astype(f32)) == base)
    c.add((d * float(s)).astype(f32), 0, 0, "point:lost_tie")
    # a later point one d24 nearer wins (pixel r + 1)
    d2 = direction(H, W, r + 1.5, 0.5)
    q = (d2 * 10.0).astype(f32)
    c.add(q, 0, 0, "point:lost_nearer")
    k = next(k for k in range(1, 64) if _d24(c, (d2 * float(nxt(10.0, -k))).astype(f32)) == _d24(c, q) - 1)
    c.add((d2 * float(nxt(10.0, -k))).astype(f32), 0, 0, "point:won")
    # three-way ties across a warp and a block: rows r - 2, r - 3
    for row, idx in ((r - 2, (31, 32, 64)), (r - 3, (255, 256, 257))):
        for i in idx:
            c.pad_to(i)
            c.at(row, 0, 12.0, 0, 0, "point:won" if i == idx[0] else "point:lost_tie")
    # a later point one d24 nearer across the block: 258 loses to 259
    dd = direction(H, W, r - 4 + 0.5, 0.5)
    c.pad_to(258)
    c.add((dd * 12.0).astype(f32), 0, 0, "point:lost_nearer")
    k = next(k for k in range(1, 64) if _d24(c, (dd * float(nxt(12.0, -k))).astype(f32)) == _d24(c, (dd * 12.0).astype(f32)) - 1)
    c.add((dd * float(nxt(12.0, -k))).astype(f32), 0, 0, "point:won")
    return c


def depth_range(H, W, max_depth=None):
    """z at +-1 at the default depths 2 and 75 m on the beam at elevation -11.3 deg: len 75 gives d24 = 0xFFFFFF
    (dropped), one ulp under it is kept, one ulp over it and a point whose depth24 would wrap under the clear value are
    clipped by z > 1; len down to 18 ulps under 2 m rounds z to -1 (kept), 19 ulps under is the
    first dropped. At 75 m the largest d24 a length reaches is 0xFFFFFD (one ulp of len moves z by two of its ulps);
    with max_depth 60 (a range of 58 m) one ulp under 60 m gives the largest d24 under the clear value, 0xFFFFFE."""
    c = Case("depth_range" if max_depth is None else "depth_range_%d" % max_depth, H, W,
             kw={} if max_depth is None else dict(max_depth=max_depth))
    row = int(math.floor((1.0 - (FOV_UP + 11.3) / (FOV_UP - FOV_DOWN)) * H))
    cols = iter(range(W * 8))

    def put(L, *tags):
        k = next(cols)
        r, col = row - (k // W) * 2, k % W
        c.add(with_len(direction(H, W, r + 0.5, col + 0.5), L), 0, 0, *tags)
    far = f32(max_depth or 75.0)
    put(far, "point:d24_clear")
    put(nxt(far, -1), "point:won", *(("point:d24_top",) if max_depth else ()))
    if max_depth is None:
        put(nxt(far, 1), "point:z_above")
        # far beyond max_depth: z = 511.8, and depth24's cast to 32 bits would wrap to a d24 under the clear value, so
        # only the clip z <= 1 keeps this point out of its pixel
        L = f32(18720.0)
        z = M.depth_z(_params(c), (L, 0.0, 0.0))
        assert (int(np.rint(np.float64(f32(0.5) * z + f32(0.5)) * 16777215.0)) & 0xFFFFFFFF) < M.DEPTH_CLEAR
        put(L, "point:z_above")
        put(f32(2.0), "point:z_minus_one")
        put(nxt(2.0, -18), "point:z_minus_one", "point:won")
        put(nxt(2.0, -19), "point:z_below")
        put(nxt(2.0, 1), "point:won")
    return c


# ---- K1: the image bounds and the seam ---------------------------------------------------------------------------------
def bounds(H, W):
    """rows 0 and H - 1 and the rows outside, fov_down and fov_up just inside / outside, columns 0 and W - 1 at their
    outer edge, and the seam: x < 0 with y = +0, -0, +1 ulp (column 0) and -1 ulp (fx = W, clipped). No azimuth lies
    outside [0, W): the only clipped column is the seam's y = -1 ulp."""
    c = Case("bounds", H, W)
    c.at(0, 1, 9.0, 0, 0, "point:won")
    c.at(H - 1, 1, 9.0, 0, 0, "point:won")
    c.at(-1, 1, 9.0, 0, 0, "point:clipped")
    c.at(H, 1, 9.0, 0, 0, "point:clipped")
    c.at(0, 2 % W, 9.0, 0, 0, "point:won", fy=0.01)       # just inside fov_down
    c.at(-1, 2 % W, 9.0, 0, 0, "point:clipped", fy=0.99)  # just outside
    c.at(H - 1, 2 % W, 9.0, 0, 0, "point:won", fy=0.99)   # just inside fov_up
    c.at(H, 2 % W, 9.0, 0, 0, "point:clipped", fy=0.01)
    c.at(1, 0, 9.0, 0, 0, "point:won", fx=0.01)
    c.at(2, W - 1, 9.0, 0, 0, "point:won", fx=0.99)
    c.at(3, 0, 9.0, 0, 0, "point:won")
    c.at(4, W - 1, 9.0, 0, 0, "point:won")
    tiny = nxt(0.0, 1)
    for k, (y, tag) in enumerate(((f32(0.0), "seam:col0"), (f32(-0.0), "seam:col0"), (tiny, "seam:col0"),
                                  (-tiny, "seam:clipped"))):
        row = H // 2 + k
        el = math.radians(FOV_UP - (FOV_UP - FOV_DOWN) * (1.0 - (row + 0.5) / H))
        i = c.add((f32(-5.0), y, f32(5.0 * math.tan(el))), 0, 0, tag)
        if tag == "seam:col0":
            c.expect_pt.append((i, "point:won"))
    return c


# ---- K2 / K3: tiles, halo and the seam --------------------------------------------------------------------------------
def tiles(H, W):
    """a dense scene: a point on every beam centre but a sparse set of holes, depth smooth with steps, labels in blocks
    whose borders lie on the tile borders x = 31|32, 63|64 and y = 15|16, 31|32 and on the seam. Winners, normals,
    erosion and flood fill all reach across tile and halo borders and into the partial last tile row and column."""
    c = Case("tiles", H, W)
    for y in range(H):
        for x in range(W):
            if (7 * x + 3 * y) % 23 == 0:
                continue  # a hole
            depth = 8.0 + 0.03 * x + 0.05 * y + (2.0 if x >= 48 else 0.0) + 0.004 * ((x * y) % 5)
            lab = 40 + (x >= 32) + 2 * (x >= 64) + 4 * (y >= 16) + 8 * (y >= 32) + (16 if x == 0 else 0)
            if (x + 2 * y) % 13 == 0:
                lab = 0
            c.at(y, x, depth, float(lab), 0.25 + 0.5 * ((x + y) % 2))
    if H > 16:
        c.expect(15, 5, "erode:by_v")
        c.expect(16, 5, "erode:by_t")
    return c


def seam_stencils(H, W):
    """normals, erosion and the +-1 / +-2 flood fill reaching across column 0 <-> W - 1"""
    c = Case("seam_stencils", H, W)
    # a normal at column W - 1 from U = column 0 (rows 1, 2)
    c.at(1, W - 1, 10.0, 50.0, 0.5)
    c.at(1, 0, 10.02, 50.0, 0.5)
    c.at(2, W - 1, 10.04, 50.0, 0.5)
    c.at(0, W - 1, 9.98, 50.0, 0.5)
    c.expect(1, W - 1, "normal:valid", "normal:across_seam", "erode:kept")
    # erosion across the seam (row 5): column 0 label 60, column W - 1 label 61
    c.at(5, 0, 10.0, 60.0, 0.5)
    c.at(5, W - 1, 10.0, 61.0, 0.5)
    c.expect(5, 0, "erode:by_s", "erode:across_seam")
    c.expect(5, W - 1, "erode:by_u", "erode:across_seam")
    # flood fill at offset 2 across the seam (row 9): pixel W - 1 unlabelled, column 1 labelled, nothing else near
    c.at(9, W - 1, 10.0, 0.0, 0.0)
    c.at(9, 1, 10.01, 70.0, 0.9)
    c.expect(9, W - 1, "fill:o2_+x", "fill:across_seam")
    # flood fill at offset 1 across the seam (row 13): pixel 0 unlabelled, column W - 1 labelled
    c.at(13, 0, 10.0, 0.0, 0.0)
    c.at(13, W - 1, 10.01, 71.0, 0.9)
    c.expect(13, 0, "fill:o1_-x", "fill:across_seam")
    return c


# ---- K2: normals -------------------------------------------------------------------------------------------------------
def normals(H, W):
    """each validity rule, a neighbour row outside the image, and collinear neighbours with len = 0"""
    c = Case("normals", H, W)
    # all four neighbours: valid (row 2, column 1)
    for (r, x) in ((2, 1), (2, 2), (3, 1), (1, 1), (2, 0)):
        c.at(r, x, 10.0 + 0.01 * x + 0.02 * r)
    c.expect(2, 1, "normal:valid")
    # S and T missing (row 6, column 1): U, V present
    for (r, x) in ((6, 1), (6, 2), (7, 1)):
        c.at(r, x, 10.0 + 0.01 * x + 0.02 * r)
    c.expect(6, 1, "normal:st_both")
    # only V missing (row 10, column 1): U, S, T present
    for (r, x) in ((10, 1), (10, 2), (10, 0), (9, 1)):
        c.at(r, x, 10.0 + 0.01 * x + 0.02 * r)
    c.expect(10, 1, "normal:only_v_missing")
    # U and V missing, S present; the top row's V is the border (row H - 1)
    for (r, x) in ((H - 1, 1), (H - 1, 0)):
        c.at(r, x, 10.0 + 0.01 * x)
    c.expect(H - 1, 1, "normal:uv_both")
    c.expect(H - 1, 0, "normal:u_or_v")
    # only U missing (row 13): V, S present
    for (r, x) in ((13, 1), (14, 1), (13, 0)):
        c.at(r, x, 10.0 + 0.01 * x + 0.02 * r)
    c.expect(13, 1, "normal:u_or_v")
    return c


def _normal_len(P, U, V):
    """len3 of the kernel's cross product for the stencil P, U (x + 1), V (y + 1)"""
    pp = M.v3(*P)
    with np.errstate(all="ignore"):
        return M.len3(M.cross3(M.normalize3(M.sub3(M.v3(*U), pp)), M.normalize3(M.sub3(M.v3(*V), pp))))


def _triples(c, ks=(4.0,), spread=0):
    """(row, col, depth, P, e, k) with P and P + e on a 2^-12 grid, P near its pixel's upper right corner, P + e in the
    next column and P - k e in the next row, every point at least 0.02 px from its pixel's edges; e also moved by up to
    `spread` grid steps per component"""
    H, W = c.H, c.W
    q = 2.0 ** -12
    grid = lambda a: (np.round(np.asarray(a, np.float64) / q) * q).astype(f32)  # noqa: E731
    prm = _params(c)

    def inside(X, col, row):
        px, py = M.pixel_coords(prm, X)
        return min(abs(px - round(px)), abs(py - round(py))) > 0.02 and \
            (math.floor(px) % W, math.floor(py)) == (col % W, row)
    steps = range(-spread, spread + 1)
    for r in range(3, H - 3):
        for col in range(W):
            for depth in (4.0, 8.0, 16.0, 32.0):
                P = grid(direction(H, W, r + 0.9, col + 0.9) * depth)
                e0 = grid(direction(H, W, r + 0.8, col + 1.05) * depth - P)
                if not inside(P, col, r):
                    continue
                for dx in steps:
                    for dy in steps:
                        for dz in steps:
                            e = e0 + f32(q) * np.array([dx, dy, dz], f32)
                            if not inside(P + e, col + 1, r):
                                continue
                            for k in ks:
                                if inside(P - f32(k) * e, col, r + 1):
                                    yield r, col, depth, P, e, k


def _normal_case(c, r, col, depth, P, U, V, tag):
    c.add(P)
    c.add(U)
    c.add(V)
    c.at(r - 1, col, depth)  # T: the S / T rule passes
    c.expect(r, col, tag)
    return c


def normals_collinear(H, W):
    """U - P = s e and V - P = -4 s e exactly (e on a 2^-12 grid): the normalised u and v are exactly opposite, the cross
    product is exactly 0, len = 0, the normal's components 0 / 0 = NaN and its w 0. P sits near its pixel's upper right
    corner so that U falls in the next column and V in the next row."""
    c = Case("normals_collinear", H, W)
    r, col, depth, P, e, _ = next(_triples(c))
    return _normal_case(c, r, col, depth, P, P + e, P - f32(4.0) * e, "normal:len_zero")


def normals_len_below(H, W):
    """V - P = -k (U - P) with k not a power of two: the normalisations round differently, u and v are almost but not
    exactly opposite, and 0 < len < 1e-7 (w = 0, finite components). Searched over k and over grid steps of e."""
    c = Case("normals_len_below", H, W)
    for r, col, depth, P, e, k in _triples(c, (3.0, 5.0, 6.0, 7.0), 2):
        ln = _normal_len(P, P + e, P - f32(k) * e)
        if f32(0.0) < ln < M.LEN_EPS:
            return _normal_case(c, r, col, depth, P, P + e, P - f32(k) * e, "normal:len_below")
    raise AssertionError("no stencil with 0 < len < 1e-7 at %dx%d" % (H, W))


def normals_len_above(H, W):
    """the stencils of normals_collinear / normals_len_below with V moved by up to 3 ulps of one coordinate: the smallest
    len above 1e-7 that such a move reaches (w = 1). len itself cannot be put at 1e-7f: the cross product's components
    are differences of products of unit-vector components, quantised at about 3e-8, and no search over these stencils
    landed a len3 of them on 1e-7f exactly"""
    c = Case("normals_len_above", H, W)
    best = None
    for n, (r, col, depth, P, e, k) in enumerate(_triples(c, (3.0, 4.0, 5.0, 6.0, 7.0), 1)):
        if n >= 64:
            break
        V0 = P - f32(k) * e
        for a in range(3):
            for k in (-3, -2, -1, 1, 2, 3):
                V = V0.copy()
                V[a] = nxt(V[a], k)
                ln = _normal_len(P, P + e, V)
                if ln > M.LEN_EPS and (best is None or ln < best[0]):
                    best = (ln, r, col, depth, P, P + e, V)
    assert best is not None, "no stencil with len above 1e-7 at %dx%d" % (H, W)
    return _normal_case(c, *best[1:], "normal:len_above")


# ---- K1 / K2: labels ---------------------------------------------------------------------------------------------------
def erosion_directions(H, W):
    """erosion by each of the four neighbours"""
    c = Case("erosion_directions", H, W)
    rows = iter(range(1, H - 1, 3))
    for name, (dy, dx) in (("u", (0, 1)), ("v", (1, 0)), ("s", (0, -1)), ("t", (-1, 0))):
        r = next(rows)
        c.at(r, 1, 10.0, 40.0, 0.5)
        c.at(r + dy, 1 + dx, 10.01, 41.0, 0.5)
        c.expect(r, 1, "erode:by_" + name)
    return c


def erosion(H, W, timestamp=100):
    """a neighbour with label 0, a movable-removed neighbour (its label still counts), two raw labels whose
    label / 255 are equal and two whose values differ by one ulp"""
    c = Case("erosion" if timestamp >= 10 else "erosion_early", H, W, timestamp)
    A = 40.0
    rows = iter(range(1, H - 1, 3))
    r = next(rows)
    c.at(r, 1, 10.0, A, 0.5)
    c.at(r, 2, 10.0, 0.0, 0.5)
    c.expect(r, 1, "erode:zero_neighbour", "erode:kept")
    r = next(rows)
    c.at(r, 1, 10.0, A, 0.5)
    i = c.at(r, 2, 10.0, 10.0, 0.5)  # a car
    c.expect(r, 1, "erode:by_u", "erode:eroded")
    c.expect_pt.append((i, "point:movable_removed" if timestamp < 10 else "point:movable_kept"))
    # labels whose / 255 collide: adjacent floats just above 63.75 (label / 255 just above 0.25); and 40 vs nxt(40)
    r = next(rows)
    l1 = next(nxt(63.8, k) for k in range(0, 64) if nxt(63.8, k) / f32(255.0) == nxt(63.8, k + 1) / f32(255.0))
    c.at(r, 1, 10.0, float(l1), 0.5)
    c.at(r, 2, 10.0, float(nxt(l1, 1)), 0.5)
    c.expect(r, 1, "erode:kept")
    r = next(rows)
    c.at(r, 1, 10.0, A, 0.5)
    c.at(r, 2, 10.0, float(nxt(A, 1)), 0.5)
    c.expect(r, 1, "erode:by_u")
    return c


def movable(H, W, timestamp):
    """movable classes at timestamp 9 (removed: no vertex, the label written) and 10 (kept); non-integers next to a
    movable class are never movable"""
    c = Case("movable_t%d" % timestamp, H, W, timestamp)
    labs = list(M.MOVABLE) + [float(nxt(10.0, -1)), float(nxt(10.0, 1)), 12.0, 40.0]
    for k, lab in enumerate(labs):
        row, col = 1 + 2 * (k // W), k % W
        mv = M.is_movable(lab)
        c.at(row, col, 10.0, lab, 0.75, "point:won",
             ("point:movable_removed" if timestamp < 10 else "point:movable_kept") if mv else "point:won")
    return c


def q1_tail(H, W):
    """label_offset_quirk: points i read labels[i + 4] and probs[i + 5]; at i = n - 6 ... n - 1 the reads at or past n
    give 0"""
    c = Case("q1_tail", H, W, kw=dict(label_offset_quirk=1))
    n = 10
    for i in range(n):
        row, col = 1 + 2 * (i // W), i % W
        c.at(row, col, 10.0 + 0.5 * i, 40.0 + i, 0.05 * (i + 1), "point:won")
    for i in range(n - 6, n):
        if i + 4 >= n:
            c.expect_pt.append((i, "q1:label_past_n"))
        if i + 5 >= n:
            c.expect_pt.append((i, "q1:prob_past_n"))
    return c


# ---- K3: the flood fill ------------------------------------------------------------------------------------------------
def _fill_pair(P_dir, sign):
    """P near P_dir with 0.007 lp a multiple of ulp(lp), and three lengths lq = lp + sign 0.007 lp + {-1, 0, +1} ulp"""
    for k in range(0, 4000):
        L = nxt(10.0, k)
        thr = M.FILL_THR * L
        if float(thr) % float(np.spacing(L)) == 0.0:
            P = with_len(P_dir, L)
            lp = M.len3(tuple(P))
            thr = M.FILL_THR * lp
            tgt = lp + thr if sign > 0 else lp - thr
            if float(tgt) != float(lp) + sign * float(thr):
                continue
            return P, thr, tgt
    raise AssertionError("no P")


def fill_threshold(H, W, step, sign):
    """|lp - lq| < 0.007 lp with lq at equality (rejected), one ulp nearer lp (accepted) or farther (rejected); the
    labelled neighbour at +x, offset 1 (sign > 0: farther than P, sign < 0: nearer)"""
    name = "fill_%s_%s" % ({-1: "below", 0: "equal", 1: "above"}[step], "far" if sign > 0 else "near")
    c = Case(name, H, W)
    r = H // 2
    P, thr, tgt = _fill_pair(direction(H, W, r + 0.5, 1.5), sign)
    lq = nxt(tgt, step * sign)
    c.add(P, 0.0, 0.0)
    c.add(with_len(direction(H, W, r + 0.5, 2.5), lq), 80.0, 0.6)
    c.expect(r, 1, "fill:o1_+x" if step < 0 else ("fill:equal_rejected" if step == 0 else "fill:none"))
    return c


def fill_directions(H, W, off, k):
    """one labelled neighbour at offset `off` in direction k (+x, +y, -x, -y): the probability divided by off + 1"""
    name = "fill_o%d_%s" % (off, "+x +y -x -y".split()[k])
    c = Case(name, H, W)
    r, x = H // 2, 2
    dy, dx = ((0, 1), (1, 0), (0, -1), (-1, 0))[k]
    c.at(r, x, 10.0, 0.0, 0.0)
    c.at(r + dy * off, x + dx * off, 10.02, 90.0, 0.9)
    if W == 4 and off == 2 and k == 2:  # x - 2 is the texel x + 2, and +x is searched first
        c.expect(r, x, "fill:o2_+x", "fill:across_seam")
    else:
        c.expect(r, x, "fill:%s" % name[5:])
    return c


def fill_priority(H, W):
    """several neighbours qualify: offset 1 before offset 2, and +x, +y, -x, -y in that order; a pixel without a
    vertex never fills"""
    c = Case("fill_priority", H, W)
    r = 3
    c.at(r, 2, 10.0, 0.0, 0.0)
    c.at(r + 1, 2, 10.01, 91.0, 0.9)    # +y offset 1
    c.at(r, 4 % W, 10.01, 92.0, 0.8)    # +x offset 2 (W = 4: the same texel as -x offset 2)
    c.at(r - 1, 2, 10.01, 93.0, 0.7)    # -y offset 1
    c.expect(r, 2, "fill:o1_+y", "fill:priority")
    r = 9
    c.at(r, 1, 10.0, 0.0, 0.0)
    c.at(r, 0, 10.01, 94.0, 0.9)        # -x offset 1
    c.at(r - 1, 1, 10.01, 95.0, 0.8)    # -y offset 1
    c.expect(r, 1, "fill:o1_-x", "fill:priority")
    # a labelled neighbour next to a pixel without a vertex (row 13, column 1 empty)
    c.at(13, 2, 10.0, 96.0, 0.9)
    c.expect(13, 1, "fill:no_vertex")
    return c


@functools.lru_cache(maxsize=None)
def all_cases(H, W):
    """every case at one shape, built once (the searches take a while); callers must not modify them"""
    cs = [depth_ties(H, W), depth_range(H, W), depth_range(H, W, 60), bounds(H, W), tiles(H, W), seam_stencils(H, W), normals(H, W),
          normals_collinear(H, W), normals_len_below(H, W), normals_len_above(H, W),
          erosion_directions(H, W), erosion(H, W), erosion(H, W, 5), movable(H, W, 9), movable(H, W, 10), q1_tail(H, W),
          fill_priority(H, W)]
    cs += [fill_threshold(H, W, s, sg) for sg in (1, -1) for s in (-1, 0, 1)]
    cs += [fill_directions(H, W, off, k) for off in (1, 2) for k in range(4)]
    return tuple(cs)


def case_ids():
    return [c.name for c in all_cases(*SHAPES[0])]


def get(name, H, W):
    return next(c for c in all_cases(H, W) if c.name == name)


def check_tags(c, model):
    """the branches the case was built for are those the model reports"""
    for i, t in c.expect_pt:
        assert t in model["point_tags"][i], "%s: point %d should take %s, the model says %s" % (
            c.name, i, t, sorted(model["point_tags"][i]))
    for yx, t in c.expect_pix:
        got = model["pixel_tags"][yx]
        assert t in got, "%s: pixel %s should take %s, the model says %s" % (c.name, yx, t, sorted(got))


# the model's branches no case reaches, and why
UNREACHED = {
    "normal:len_eq": "len = 1e-7f exactly is not built (normals_len_above)",
    "normal:len_nan": "needs U or V equal to P bit for bit, or an overflow, and neither can lie in another pixel within "
                      "max_depth",
}
BRANCHES = M.TAGS - set(UNREACHED)


def reached(model):
    got = set()
    for t in model["point_tags"]:
        got |= t
    for t in model["pixel_tags"].values():
        got |= t
    return got
