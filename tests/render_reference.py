"""An exact reference of the surfel render pass, numpy only, written from the shaders' rules (DESIGN.md section 2):
render_surfels.vert / .geom / .frag, the GL rasterisation rules the project fixes, and render_compose.frag.

It shares no code with the oracle or the CUDA sources and has none of the kernel's fast paths: every triangle is
rasterised over its whole bounding box (clamped only at the image) with exact integer edge functions, and the depth test
is a z-buffer walked in buffer order. The geometry is restated one correctly rounded float32 operation at a time in the
kernel's order (numpy float32 arithmetic is IEEE and never contracts a*b+c into an FMA, which matches -fmad=false).

Transforms are kept exact instead of restated: the pose-table entries and the render poses must be translations by
values for which inv(P) * pose[t] is exact in float32 (checked), so no restatement of the pose products is needed.

`classify` also reports, per surfel, the regime k_render_scatter puts it in: culled in stage A/B, empty box, small with
its box extent (ni, nj), large by box size, or large by corner span -- the tests use it to prove that a case reaches the
regime it is built for."""
import numpy as np

F = np.float32
K_PI, K_INV_PI, K_PI_O2, K_PI_O4 = F(3.14159265358979323846), F(0.31830988618379067154), F(1.57079632679489661923), \
    F(0.78539816339744830962)
K_RAD2DEG = F(57.29577951308232)
DEPTH_CLEAR = 0xFFFFFF          # 24-bit depth buffer cleared to 1.0
COMPOSE_AGE = 100               # SurfelMap.h:144: timestamp_threshold = map timestamp - 100
SMALL_W, SMALL_H, SMALL_SPAN = 12, 5, 1 << 14
MAX_POSES = 10000

CULLED, EMPTY, SMALL, LARGE_BOX, LARGE_SPAN = "culled", "empty", "small", "large_box", "large_span"


# ---- GLSL built-ins as the project fixes them: fixed fp32 polynomials ----------------------------------------------
def _atan_poly(t):
    z = t * t
    p = F(8.05374449538e-2)
    p = p * z - F(1.38776856032e-1)
    p = p * z + F(1.99777106478e-1)
    p = p * z - F(3.33329491539e-1)
    return (p * z) * t + t


def atan2f(y, x):
    """GLSL atan(y, x), atan(0, 0) = 0"""
    ax, ay = np.abs(x), np.abs(y)
    swap = ay > ax
    hi = np.where(swap, ay, ax)
    lo = np.where(swap, ax, ay)
    t = lo / np.where(hi == 0, F(1), hi)
    big = t > F(0.4142135623730950)
    r = np.where(big, K_PI_O4 + _atan_poly((t - F(1)) / (t + F(1))), _atan_poly(t))
    r = np.where(swap, K_PI_O2 - r, r)
    r = np.where(x < 0, K_PI - r, r)
    r = np.where(y < 0, -r, r)
    return np.where(hi == 0, F(0), r).astype(F)


def asinf(x):
    a = np.abs(x)
    flag = a > F(0.5)
    zf = F(0.5) * (F(1) - a)
    z = np.where(flag, zf, a * a)
    w = np.where(flag, np.sqrt(zf), a)
    p = F(4.2163199048e-2)
    p = p * z + F(2.4181311049e-2)
    p = p * z + F(4.5470025998e-2)
    p = p * z + F(7.4953002686e-2)
    p = p * z + F(1.6666752422e-1)
    r = (p * z) * w + w
    r = np.where(flag, K_PI_O2 - (r + r), r)
    r = np.where(x < 0, -r, r)
    return np.where(a < F(1.0e-4), x, r).astype(F)


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _len(a):
    return np.sqrt(_dot(a, a))


def _normalize(a):
    n = _len(a)
    return (a[0] / n, a[1] / n, a[2] / n)


def project01(p, fov_up, fov, min_depth, max_depth):
    """spherical projection of every pass: x, y in [0, 1) image coordinates, z normalised depth"""
    depth = _len(p)
    yaw = atan2f(p[1], p[0])
    pitch = -asinf(p[2] / depth)
    x = F(0.5) * ((-yaw * K_INV_PI) + F(1))
    y = F(1) - (K_RAD2DEG * pitch + fov_up) / fov
    z = (depth - min_depth) / (max_depth - min_depth)
    return x, y, z


def depth24(z):
    """24-bit window depth: rint(z * (2^24 - 1)), the product exact in float64"""
    return np.rint(np.asarray(z, np.float64) * 16777215.0).astype(np.int64)


# ---- parameters and exact transforms ----------------------------------------------------------------------------
class Model:
    """the model image's parameters as the render pass uses them"""

    def __init__(self, p):
        self.W, self.H = int(p.model_width), int(p.model_height)
        self.fov_up = F(abs(p.model_fov_up))
        self.fov = F(abs(p.model_fov_up)) + F(abs(p.model_fov_down))
        self.min_depth, self.max_depth = F(p.model_min_depth), F(p.model_max_depth)
        self.use_stability = bool(p.use_stability)
        self.max_loop_closure_distance = F(p.max_loop_closure_distance)


def _translation(T):
    T = np.asarray(T, np.float64)
    assert np.array_equal(T[:3, :3], np.eye(3)) and np.array_equal(T[3], [0, 0, 0, 1]), "not a translation"
    assert np.array_equal(T[:3, 3].astype(F).astype(np.float64), T[:3, 3]), "translation not exact in float32"
    return T[:3, 3]


def pose_matrices(surfels, render_pose, table=None):
    """per surfel: inv(render_pose) * pose[int(count)] as a float32 translation (exact), column-major order not needed"""
    tr = -_translation(render_pose)
    idx = np.clip(surfels["count"].astype(np.int64), 0, MAX_POSES - 1)   # int(count), clamped like the pose fetch
    t = np.zeros((len(surfels), 3))
    for k, i in enumerate(idx):
        t[k] = (_translation(table[i]) if table and i in table else 0.0) + tr
    assert np.array_equal(t.astype(F).astype(np.float64), t), "pose product not exact in float32"
    return t.astype(F)


def _xform(surfels, t):
    """xform_point / xform_dir with the identity rotation: ((M0 x + M4 y) + M8 z) + M12, in float32"""
    one, zero = F(1), F(0)
    px, py, pz = surfels["x"], surfels["y"], surfels["z"]
    nx, ny, nz = surfels["nx"], surfels["ny"], surfels["nz"]
    pp = (((one * px + zero * py) + zero * pz) + t[:, 0], ((zero * px + one * py) + zero * pz) + t[:, 1],
          ((zero * px + zero * py) + one * pz) + t[:, 2])
    nn = ((one * nx + zero * ny) + zero * nz, (zero * nx + one * ny) + zero * nz, (zero * nx + zero * ny) + one * nz)
    return pp, nn


# ---- geometry stage ---------------------------------------------------------------------------------------------
class Geometry:
    """render_surfels.vert + .geom for one draw call: which surfels emit a quad, and the quad's four snapped corners"""

    def __init__(self, surfels, m, t, conf_thr, t_thr, old):
        s = np.ascontiguousarray(surfels)
        self.n = len(s)
        pp, nn = _xform(s, t)
        self.pp, self.nn = pp, nn
        with np.errstate(all="ignore"):
            inv_len = _len(pp)
            visible = _dot(nn, (-pp[0] / inv_len, -pp[1] / inv_len, -pp[2] / inv_len)) > F(0.01)   # .geom:84
            cx, cy, cz = project01(pp, m.fov_up, m.fov, m.min_depth, m.max_depth)
            inside = (cx >= 0) & (cy >= 0) & (cz >= 0) & (cx < 1) & (cy < 1) & (cz < 1)
            conf = ~np.bool_(m.use_stability) | (s["confidence"] > F(conf_thr))                    # .geom:87
            creation = s["count"].astype(np.int32)           # int(float): truncation
            ts = s["timestamp"].astype(np.uint32).view(np.int32)
            cls = (creation < t_thr) if old else ((creation >= t_thr) | (ts >= t_thr))            # .geom:90-91
            self.alive = visible & inside & conf & cls
            # .geom:80-82 quad axes, .geom:100-118 corners (p -/+ ru) -/+ rv
            u = _normalize((nn[1] - nn[2], -nn[0], nn[0]))
            cr = (nn[1] * u[2] - nn[2] * u[1], nn[2] * u[0] - nn[0] * u[2], nn[0] * u[1] - nn[1] * u[0])
            v = _normalize(cr)
            r = s["radius"]
            ru = tuple(r * c for c in u)
            rv = tuple(r * c for c in v)
            self.X = np.zeros((self.n, 4), np.int64)
            self.Y = np.zeros((self.n, 4), np.int64)
            self.Z = np.zeros((self.n, 4), F)
            Wf, Hf = F(m.W), F(m.H)
            for i in range(4):
                h = tuple((a + b) if i & 1 else (a - b) for a, b in zip(pp, ru))
                c = tuple((a + b) if i & 2 else (a - b) for a, b in zip(h, rv))
                x, y, z = project01(c, m.fov_up, m.fov, m.min_depth, m.max_depth)
                x = np.where(cx - x > F(0.5), x + F(1), x)      # .geom:68
                x = np.where(x - cx > F(0.5), x - F(1), x)      # .geom:69
                xw = (F(0.5) * (F(2) * x - F(1)) + F(0.5)) * Wf
                yw = (F(0.5) * (F(2) * y - F(1)) + F(0.5)) * Hf
                self.Z[:, i] = F(0.5) * (F(2) * z - F(1)) + F(0.5)
                xs, ys = np.rint(xw * F(256)), np.rint(yw * F(256))   # snapped to 1/256 px, ties to even
                ok = np.isfinite(xs) & np.isfinite(ys) & (np.abs(xs) < 2.0 ** 40) & (np.abs(ys) < 2.0 ** 40)
                assert np.all(ok[self.alive])
                self.X[:, i] = np.where(ok, xs, 0).astype(np.int64)
                self.Y[:, i] = np.where(ok, ys, 0).astype(np.int64)
        self.m = m

    def box(self, k):
        """pixel bounding box of quad k clamped to the image: (i0, i1, j0, j1), empty when i0 > i1 or j0 > j1"""
        return _box(self.X[k], self.Y[k], self.m.W, self.m.H)


def _ceil256(a):
    return -((-a) // 256)


def _box(X, Y, W, H):
    i0, i1 = max(_ceil256(int(min(X)) - 128), 0), min((int(max(X)) - 128) // 256, W - 1)
    j0, j1 = max(_ceil256(int(min(Y)) - 128), 0), min((int(max(Y)) - 128) // 256, H - 1)
    return i0, i1, j0, j1


def classify(g):
    """the regime of every surfel in k_render_scatter: (kind, ni, nj) with ni / nj the clamped box extent - 1"""
    out = []
    for k in range(g.n):
        if not g.alive[k]:
            out.append((CULLED, -1, -1))
            continue
        i0, i1, j0, j1 = g.box(k)
        if i0 > i1 or j0 > j1:
            out.append((EMPTY, -1, -1))
            continue
        ni, nj = i1 - i0, j1 - j0
        if not (ni < SMALL_W and nj < SMALL_H):
            out.append((LARGE_BOX, ni, nj))
            continue
        X0, Y0 = i0 * 256 + 128, j0 * 256 + 128
        span = max(max(abs(int(x) - X0) for x in g.X[k]), max(abs(int(y) - Y0) for y in g.Y[k]))
        out.append((SMALL if span < SMALL_SPAN else LARGE_SPAN, ni, nj))
    return out


def corner_span(g, k):
    """largest |corner - first pixel centre of the box| in 1/256 px, per axis sign: (min dx, max dx, min dy, max dy)"""
    i0, _, j0, _ = g.box(k)
    X0, Y0 = i0 * 256 + 128, j0 * 256 + 128
    return (int(min(g.X[k])) - X0, int(max(g.X[k])) - X0, int(min(g.Y[k])) - Y0, int(max(g.Y[k])) - Y0)


# ---- rasterisation ----------------------------------------------------------------------------------------------
def _tie(P, Q):
    dx, dy = Q[0] - P[0], Q[1] - P[1]
    return dy > 0 or (dy == 0 and dx > 0)


def _edge(P, Q, X, Y):
    return (Q[0] - P[0]) * (Y - P[1]) - (Q[1] - P[1]) * (X - P[0])


def triangle(A, B, C, W, H):
    """pixel centres covered by triangle (A, B, C), corners (X, Y, z, tx, ty) with integer X, Y in 1/256 px.
    Returns (pixel indices, barycentric weights fA, fB, fC, the corners after the orientation fix) or None."""
    area = (B[0] - A[0]) * (C[1] - A[1]) - (B[1] - A[1]) * (C[0] - A[0])
    if area == 0:
        return None
    if area < 0:    # orientation fix: B and C exchanged
        B, C = C, B
        area = -area
    i0, i1, j0, j1 = _box([A[0], B[0], C[0]], [A[1], B[1], C[1]], W, H)
    if i0 > i1 or j0 > j1:
        return None
    jj, ii = np.meshgrid(np.arange(j0, j1 + 1, dtype=np.int64), np.arange(i0, i1 + 1, dtype=np.int64), indexing="ij")
    X, Y = ii.ravel() * 256 + 128, jj.ravel() * 256 + 128
    w = []
    for P, Q in ((B, C), (C, A), (A, B)):
        assert max(abs(P[0]), abs(P[1]), abs(Q[0]), abs(Q[1]), W * 256, H * 256) < 2 ** 29   # products exact in int64
        e = _edge(P, Q, X, Y)
        w.append((e, (e > 0) | ((e == 0) & _tie(P, Q))))
    inside = w[0][1] & w[1][1] & w[2][1]
    assert abs(area) < 2 ** 53 and np.all(np.abs(w[1][0]) < 2 ** 53)     # int -> float32 rounds once
    fa = F(area)
    fB = w[1][0][inside].astype(F) / fa
    fC = w[2][0][inside].astype(F) / fa
    fA = (F(1) - fB) - fC
    pix = Y[inside] // 256 * W + X[inside] // 256
    return pix, fA, fB, fC, (A, B, C)


def quad_fragments(g, k):
    """fragments of quad k in primitive order (triangle 0, then 1) that pass the disc test and the z clip:
    list of (pixel indices, depth24)"""
    m = g.m
    corners = [(int(g.X[k, i]), int(g.Y[k, i]), g.Z[k, i], F(1 if i & 1 else -1), F(1 if i & 2 else -1)) for i in range(4)]
    out = []
    for t in range(2):
        r = triangle(corners[t], corners[t + 1], corners[t + 2], m.W, m.H)
        if r is None:
            continue
        pix, fA, fB, fC, (A, B, C) = r
        tx = (fA * A[3] + fB * B[3]) + fC * C[3]
        ty = (fA * A[4] + fB * B[4]) + fC * C[4]
        z = (fA * A[2] + fB * B[2]) + fC * C[2]
        keep = ~(tx * tx + ty * ty > F(1)) & (z >= 0) & (z <= 1)     # render_surfels.frag:22-28, near / far clip
        out.append((pix[keep], depth24(z[keep])))
    return out


class ZBuffer:
    """one render target: 24-bit depth cleared to 1.0 and the winning surfel per pixel (-1: none)"""

    def __init__(self, m):
        self.depth = np.full(m.W * m.H, DEPTH_CLEAR, np.int64)
        self.winner = np.full(m.W * m.H, -1, np.int64)
        self.passes = np.full(m.W * m.H, -1, np.int64)

    def draw(self, g, lequal, pass_id):
        """one glDrawArrays over the whole buffer: GL_LESS keeps the earliest of equal depths, GL_LEQUAL the last"""
        for k in np.nonzero(g.alive)[0]:
            for pix, d in quad_fragments(g, k):
                win = d <= self.depth[pix] if lequal else d < self.depth[pix]
                self.depth[pix[win]] = d[win]
                self.winner[pix[win]] = k
                self.passes[pix[win]] = pass_id


# ---- the operators ------------------------------------------------------------------------------------------------
def _frame(m, surfels, zb, geoms):
    """vertex / normal / semantic image of a z-buffer's winners (the winner's centre and normal under its pass's pose,
    w = 1; the semantic vec4 of the surfel); zeros where nothing was drawn"""
    P = m.W * m.H
    v, n, s = (np.zeros((P, 4), F) for _ in range(3))
    hit = zb.winner >= 0
    for pid, g in enumerate(geoms):
        sel = hit & (zb.passes == pid)
        k = zb.winner[sel]
        v[sel, 0], v[sel, 1], v[sel, 2], v[sel, 3] = g.pp[0][k], g.pp[1][k], g.pp[2][k], F(1)
        n[sel, 0], n[sel, 1], n[sel, 2], n[sel, 3] = g.nn[0][k], g.nn[1][k], g.nn[2][k], F(1)
        for c, f in enumerate("rgbw"):
            s[sel, c] = surfels[f][k]
    return tuple(a.reshape(m.H, m.W, 4) for a in (v, n, s))


def compose(m, old, new):
    """render_compose.frag:26-48: the new view's pixel unless it is invalid and the old one valid and (the new one empty
    or its vertex within max_loop_closure_distance of the old one)"""
    ov, on, os_ = old
    nv, nn, ns = new
    valid = (ov[..., 3] > F(0.5)) & (on[..., 3] > F(0.5))
    new_valid = (nv[..., 3] > F(0.5)) & (nn[..., 3] > F(0.5))
    d = nv[..., :3] - ov[..., :3]
    dist = np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
    take_old = ~new_valid & valid & ((nv[..., 3] < F(0.5)) | (dist < m.max_loop_closure_distance))
    return tuple(np.where(take_old[..., None], o, nw) for o, nw in zip(old, new))


class Renderer:
    """SurfelMap::render / render_active / render_inactive / render_composed over an uploaded surfel array"""

    def __init__(self, params, surfels, timestamp, pose_table=None):
        self.m = Model(params)
        self.compose_rendering = bool(params.compose_rendering)
        self.s = np.ascontiguousarray(surfels)
        self.t_thr = int(timestamp) - COMPOSE_AGE
        self.table = pose_table or {}

    def geometry(self, pose, conf_thr, t_thr, old):
        return Geometry(self.s, self.m, pose_matrices(self.s, pose, self.table), conf_thr, t_thr, old)

    def _view(self, draws, lequal):
        zb = ZBuffer(self.m)
        for pid, g in enumerate(draws):
            zb.draw(g, lequal, pid)
        return zb

    def render(self, pose_old, pose_new, conf_thr):
        """{"old", "new", "composed", "out"}: (vertex, normal, semantic) images and "winners": the winner images"""
        m = self.m
        if not self.compose_rendering:   # one view of everything created at or after timestamp 0, copied to old and new
            g = self.geometry(pose_old, conf_thr, 0, False)
            zb = self._view([g], False)
            f = _frame(m, self.s, zb, [g])
            return dict(old=f, new=f, out=f, winners=dict(new=zb.winner))
        go = self.geometry(pose_old, conf_thr, self.t_thr, True)
        gn = self.geometry(pose_new, conf_thr, self.t_thr, False)
        zo, zn, zc = self._view([go], False), self._view([gn], False), self._view([go, gn], False)
        old, new = _frame(m, self.s, zo, [go]), _frame(m, self.s, zn, [gn])
        return dict(old=old, new=new, composed=_frame(m, self.s, zc, [go, gn]), out=compose(m, old, new),
                    winners=dict(old=zo.winner, new=zn.winner, composed=zc.winner))

    def render_active(self, pose, conf_thr):
        """new surfels into the new frame: (vertex, normal)"""
        g = self.geometry(pose, conf_thr, self.t_thr, False)
        return _frame(self.m, self.s, self._view([g], False), [g])[:2]

    def render_inactive(self, pose, conf_thr):
        g = self.geometry(pose, conf_thr, self.t_thr, True)
        return _frame(self.m, self.s, self._view([g], False), [g])[:2]

    def render_composed(self, pose_old, pose_new, conf_thr):
        """GL_LEQUAL, old pass then new pass into one target: (vertex, normal)"""
        go = self.geometry(pose_old, conf_thr, self.t_thr, True)
        gn = self.geometry(pose_new, conf_thr, self.t_thr, False)
        return _frame(self.m, self.s, self._view([go, gn], True), [go, gn])[:2]
