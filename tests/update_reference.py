"""An exact numpy model of the map update K6a-K6e (gen_indexmap, init_radiusConf, update_surfels, gen_surfels,
copy_surfels), written from the shader rules of DESIGN.md section 2 and the operation order documented in
csrc/sb_math.cuh. It shares no code with the oracle or the library.

* Every +, *, /, sqrt is one numpy float32 operation, strictly left to right in the kernels' order, no FMA: dot3, len3,
  normalize3, cross3, xform_point, xform_dir, mat4_mul, pack_rgb and depth24 (fp64 product, rounded half to even) are
  restated below.
* The pixel a surfel lands on is computed in fp64. The pinned atan2f_ / asinf_ polynomials err by a few ulps, so every
  designed surfel lies at least PIXEL_MARGIN pixels from a pixel edge and the model asserts it. The normalised depth z
  needs no transcendental and is exact.
* The transcendentals of the update (acosf_ / sinf_ in slerp, expf_ / logf_ in the confidence) are evaluated in fp64 and
  rounded once. The outputs that depend on them (the `approx` mask of the returned records) agree within TOL_CONF and
  TOL_NORMAL; every decision the designed cases test is arranged not to depend on them.
"""
import math

import numpy as np

f32 = np.float32
PIXEL_MARGIN = 1e-3
DEPTH_CLEAR = 0xFFFFFF
# logf_ / expf_ are within 2 ulps of fp64. The update's log-odds log(p / (1 - p)) is taken at p <= 0.61 in every case whose
# confidence is compared (p = 1 gives +inf and the exact clamp at 20): its condition number is at most 1 / (1 - p) < 3, and
# the confidence adds two more roundings. 16 ulps of max(|c|, 1) covers this with margin.
TOL_CONF_ULPS = 16
# slerp: acos is taken only at dots <= cos(10 deg) or at exactly 1 (NaN); its weights carry a few ulps each, the
# normalisation one more
TOL_NORMAL = 2e-6
SURFEL_DTYPE = np.dtype([
    ("x", "f4"), ("y", "f4"), ("z", "f4"), ("radius", "f4"),
    ("nx", "f4"), ("ny", "f4"), ("nz", "f4"), ("confidence", "f4"),
    ("timestamp", "u4"), ("color", "f4"), ("weight", "f4"), ("count", "f4"),
    ("r", "f4"), ("g", "f4"), ("b", "f4"), ("w", "f4"),
])
MOVABLE = (10.0, 11.0, 13.0, 15.0, 18.0, 20.0, 30.0, 31.0, 32.0)


# ---- fp32 vector arithmetic in the kernels' order ---------------------------------------------------------------------
def dot3(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def len3(a):
    return np.sqrt(dot3(a, a))


def sub3(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def add3(a, b):
    return (a[0] + b[0], a[1] + b[1], a[2] + b[2])


def scale3(s, a):
    return (s * a[0], s * a[1], s * a[2])


def divs3(a, s):
    return (a[0] / s, a[1] / s, a[2] / s)


def neg3(a):
    return (-a[0], -a[1], -a[2])


def cross3(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def normalize3(a):
    return divs3(a, len3(a))


def xform_point(M, p):  # M: numpy (row-major) 4x4 float32
    return tuple(((M[r, 0] * p[0] + M[r, 1] * p[1]) + M[r, 2] * p[2]) + M[r, 3] for r in range(3))


def xform_dir(M, p):
    return tuple((M[r, 0] * p[0] + M[r, 1] * p[1]) + M[r, 2] * p[2] for r in range(3))


def mat4_mul(A, B):
    C = np.zeros((4, 4), f32)
    for c in range(4):
        for r in range(4):
            C[r, c] = ((A[r, 0] * B[0, c] + A[r, 1] * B[1, c]) + A[r, 2] * B[2, c]) + A[r, 3] * B[3, c]
    return C


def rigid_inverse(T):
    """[R^T | -R^T t] in fp64, rounded once (DESIGN.md section 2)"""
    T = np.asarray(T, np.float64)
    R = np.eye(4)
    R[:3, :3] = T[:3, :3].T
    R[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return R.astype(f32)


def round_away(x):
    """GLSL round(): ties away from zero"""
    x = float(x)
    return math.copysign(math.floor(abs(x) + 0.5), x)


def pack_rgb(r, g, b):
    v = int(round_away(f32(r) * f32(255.0)))
    v = (v << 8) + int(round_away(f32(g) * f32(255.0)))
    v = (v << 8) + int(round_away(f32(b) * f32(255.0)))
    return f32(v)


def depth24(zw):
    return int(np.rint(np.float64(zw) * 16777215.0))


def is_movable(label):
    return float(label) in MOVABLE


def v3(*a):
    return tuple(f32(x) for x in a)


# ---- derived uniforms (SurfelMap::setParameters), fp64 of the fp32 parameters, rounded once ---------------------------
def _log(x):
    return math.log(x) if x > 0.0 else -math.inf


def derived(p):
    vfov = f32(abs(f32(p.data_fov_up)) + abs(f32(p.data_fov_down)))
    vpix = f32(math.tan(float(f32(0.5)) * (float(vfov) * math.pi / 180.0) / p.data_height))
    hpix = f32(math.tan(float(f32(0.5)) * (360.0 * math.pi / 180.0) / p.data_width))
    p_unstable = f32(1.0) - f32(p.p_stable)
    rad = lambda d: f32(f32(d) * f32(math.pi / 180.0))  # noqa: E731
    return dict(pixel_size=max(vpix, hpix), p_unstable=p_unstable,
                log_prior=f32(_log(float(f32(p.p_prior)) / (1.0 - float(f32(p.p_prior))))),
                log_unstable=f32(_log(float(p_unstable) / (1.0 - float(p_unstable)))),
                radconf_angle_thresh=f32(math.cos(float(rad(p.max_angle)))),
                update_angle_thresh=f32(math.sin(float(rad(p.map_max_angle)))))


def derived_exact(p):
    """the same six quantities in fp64 (each derived value must lie within 1 ulp of it); the angles are those of the
    reference's fp32 radians(), deg * (float)(pi / 180)"""
    vfov = abs(p.data_fov_up) + abs(p.data_fov_down)
    pu = 1.0 - float(f32(p.p_stable))
    rad = lambda d: float(f32(f32(d) * f32(math.pi / 180.0)))  # noqa: E731
    return dict(pixel_size=max(math.tan(0.5 * math.radians(vfov) / p.data_height), math.tan(math.pi / p.data_width)),
                p_unstable=pu, log_prior=_log(float(f32(p.p_prior)) / (1.0 - float(f32(p.p_prior)))),
                log_unstable=_log(pu / (1.0 - pu)), radconf_angle_thresh=math.cos(rad(p.max_angle)),
                update_angle_thresh=math.sin(rad(p.map_max_angle)))


# ---- projection ---------------------------------------------------------------------------------------------------------
def fovs(p):
    up = f32(abs(f32(p.data_fov_up)))
    return up, f32(up + f32(abs(f32(p.data_fov_down))))


def pixel_of(p, v, check=True):
    """(column, row) of the point v (sensor frame) in fp64, the margin to the nearest pixel edge asserted; None if not
    finite"""
    x, y, z = (float(c) for c in v)
    d = math.sqrt(x * x + y * y + z * z)
    if not (math.isfinite(d) and d > 0.0):
        return None
    up, fov = fovs(p)
    yaw = math.atan2(y, x)
    pitch = -math.asin(z / d)
    px = 0.5 * (-yaw / math.pi + 1.0) * p.data_width
    py = (1.0 - (math.degrees(pitch) + float(up)) / float(fov)) * p.data_height
    if check:
        for q in (px, py):
            assert abs(q - round(q)) >= PIXEL_MARGIN, "designed point %s lies within %g px of a pixel edge" % (v, PIXEL_MARGIN)
    return math.floor(px), math.floor(py)


def depth01(p, v):
    """the normalised depth z of project01, fp32"""
    return (len3(v) - f32(p.min_depth)) / (f32(p.max_depth) - f32(p.min_depth))


def pose_index(count, cap=10000):
    c = int(count) if math.isfinite(float(count)) else 0
    return min(max(c, 0), cap - 1)


# ---- the update -----------------------------------------------------------------------------------------------------
def radius_pixel(p, d, V, N):
    """K6b for one pixel: (radius map texel, branch tag)"""
    with np.errstate(all="ignore"):
        return _radius_pixel(p, d, V, N)


def _radius_pixel(p, d, V, N):
    v, n = v3(*V[:3]), v3(*N[:3])
    dist = len3(v)
    view_dir = divs3(neg3(v), dist)
    angle = dot3(n, view_dir)
    o = np.zeros(4, f32)
    if not (V[3] > f32(0.5) and N[3] > f32(0.5)):
        return o, "radius:invalid"
    if not angle > d["radconf_angle_thresh"]:
        return o, "radius:nan_angle" if angle != angle else "radius:angle_rejected"
    c = f32(0.5) if angle < f32(0.5) else (f32(1.0) if angle > f32(1.0) else angle)
    radius = ((f32(1.41) * dist) * d["pixel_size"]) / c
    lo = radius if radius > f32(p.min_radius) else f32(p.min_radius)
    radius = lo if lo < f32(p.max_radius) else f32(p.max_radius)
    o[0], o[3] = radius, 1.0
    tag = "radius:c_low" if angle <= f32(0.5) else ("radius:c_high" if angle >= f32(1.0) else "radius:c_mid")
    if lo == f32(p.min_radius):
        tag += ",radius:min"
    if radius == f32(p.max_radius):
        tag += ",radius:max"
    return o, tag


def update(p, surfels, frame, pose, timestamp, poses=None, origin=(0, 0), pending_extraction=0):
    """One SurfelMap::update of the surfel list `surfels` (SURFEL_DTYPE, map order) at map timestamp `timestamp` with the
    current pose `pose` (4x4) and the data frame (vertex, normal, semantic float32 [H, W, 4]). poses: {entry: 4x4} of the
    pose table (others identity). Returns a dict with the index map (surfel index + 1, 0 = none), the radius map, the
    integrated flags, n_updated, n_new, the resulting map, the mask `approx` of its fields that went through a
    transcendental, and the branch tags of every surfel and of every pixel of the radius and generation passes."""
    np.seterr(all="ignore")
    H, W = p.data_height, p.data_width
    d = derived(p)
    V, N, S = (np.asarray(a, f32) for a in frame)
    pose = np.asarray(pose, f32)
    table = {k: np.asarray(v, f32) for k, v in (poses or {}).items()}
    table[timestamp] = pose  # SurfelMap.cpp:494-495
    eye = np.eye(4, dtype=f32)
    SP = lambda k: table.get(k, eye)  # noqa: E731
    SPI = lambda k: rigid_inverse(table[k]) if k in table else eye  # noqa: E731
    inv_pose = rigid_inverse(pose)
    up, fov = fovs(p)
    n_s = len(surfels)

    # K6a: nearest visible surfel per data pixel, GL_LESS in map order
    index = np.zeros((H, W), np.uint32)
    best = np.full((H, W), DEPTH_CLEAR, np.int64)
    for k in range(n_s):
        s = surfels[k]
        T = mat4_mul(inv_pose, SP(pose_index(s["count"])))
        v = xform_point(T, v3(s["x"], s["y"], s["z"]))
        n = xform_dir(T, v3(s["nx"], s["ny"], s["nz"]))
        if not dot3(n, divs3(neg3(v), len3(v))) > f32(0.01):
            continue
        pix = pixel_of(p, v)
        if pix is None or not (0 <= pix[0] < W and 0 <= pix[1] < H):
            continue
        zn = f32(2.0) * depth01(p, v) - f32(1.0)
        if not (zn >= f32(-1.0) and zn <= f32(1.0)):
            continue
        d24 = depth24(f32(0.5) * zn + f32(0.5))
        if d24 < best[pix[1], pix[0]]:
            best[pix[1], pix[0]] = d24
            index[pix[1], pix[0]] = k + 1

    # K6b
    radius = np.zeros((H, W, 4), f32)
    radius_tags = {}
    for y in range(H):
        for x in range(W):
            radius[y, x], radius_tags[(y, x)] = radius_pixel(p, d, V[y, x], N[y, x])

    # K6c
    integrated = np.zeros((H, W), np.uint8)
    out, out_approx, valid_list, tags = [], [], [], []
    for k in range(n_s):
        s = surfels[k]
        tag = set()
        o = s.copy()
        approx = set()
        ts_i = int(np.int32(np.uint32(s["timestamp"]).view(np.int32)))
        surfel_age = timestamp - ts_i
        creation = int(s["count"])
        ci = pose_index(s["count"])
        old_position = xform_point(SP(ci), v3(s["x"], s["y"], s["z"]))
        old_normal = xform_dir(SP(ci), v3(s["nx"], s["ny"], s["nz"]))
        old_radius, old_conf, old_weight = s["radius"], s["confidence"], s["weight"]
        valid_out = True
        if old_conf < f32(p.confidence_threshold) and p.use_stability:
            valid_out = surfel_age < p.unstable_age
            tag.add("unstable:young" if valid_out else "unstable:old")
            if surfel_age < 0:
                tag.add("unstable:future")
        else:
            tag.add("stable")
        o["color"] = pack_rgb(0.3, 0.3, 0.3)
        vertex = xform_point(inv_pose, old_position)
        normal = normalize3(xform_dir(inv_pose, old_normal))
        vis_dot = dot3(normal, divs3(neg3(vertex), len3(vertex)))
        visible = vis_dot > f32(0.0)
        if vis_dot == 0.0:
            tag.add("visible:zero_dot_%s" % ("neg" if math.copysign(1.0, float(vis_dot)) < 0 else "pos"))
        z = depth01(p, vertex)
        pix = pixel_of(p, vertex)
        ix, iy = (pix[0] + 0.5, pix[1] + 0.5) if pix is not None else (float("nan"), float("nan"))
        inside = (ix < W and iy < H and z < f32(1.0)) and not (ix < 0.0 and iy < 0.0 and z < f32(0.0))
        in_img = pix is not None and 0 <= pix[0] < W and 0 <= pix[1] < H
        Vt = V[pix[1], pix[0]] if in_img else np.zeros(4, f32)
        Nt = N[pix[1], pix[0]] if in_img else np.zeros(4, f32)
        valid = Vt[3] > f32(0.5) and Nt[3] > f32(0.5)
        if not visible:
            tag.add("not_visible")
        if not inside:
            tag.add("outside:z" if z >= f32(1.0) else "outside")
        if visible and inside and not valid:
            tag.add("measurement_invalid")
        penalty = f32(0.0)
        update_conf = d["log_prior"]
        conf_approx = False
        mark = None
        avg_prob = None
        if valid and inside and visible:
            if z < f32(0.0):
                tag.add("inside:nearer_than_min_depth")
            St = S[pix[1], pix[0]]
            Rt = radius[pix[1], pix[0]]
            data_label, data_prob = St[0] * f32(255.0), St[3]
            model_label, model_prob = s["r"] * f32(255.0), s["w"]
            if data_label - math.floor(data_label) == 0.5:
                tag.add("label:round_tie")
            label_diff = round_away(data_label) != round_away(model_label)
            if label_diff and is_movable(model_label):
                penalty = f32(1.0)
                tag.add("penalty")
            v = v3(*Vt[:3])
            n = v3(*Nt[:3])
            v_global = xform_point(pose, v)
            n_global = normalize3(xform_dir(pose, n))
            view_dir = divs3(neg3(v), len3(v))
            distance = abs(dot3(old_normal, sub3(v_global, old_position)))
            angle = len3(cross3(n_global, old_normal))
            new_radius, new_conf = Rt[0], Rt[1]
            dpix = (pix[1], pix[0])
            if distance < f32(p.map_max_distance) and angle < d["update_angle_thresh"]:
                tag.add("match")
                zn = f32(2.0) * z - f32(1.0)
                if zn >= f32(-1.0) and zn <= f32(1.0):
                    assert depth24(f32(0.5) * zn + f32(0.5)) < DEPTH_CLEAR  # unreachable for z < 1 (see the test)
                    mark = dpix
                    if depth24(f32(0.5) * zn + f32(0.5)) == DEPTH_CLEAR - 1:
                        tag.add("depth24:top")
                confidence = old_conf + new_conf
                o["confidence"] = confidence
                o["timestamp"] = np.uint32(timestamp & 0xFFFFFFFF)
                avg_radius = new_radius if new_radius < old_radius else old_radius
                avg_radius = avg_radius if avg_radius > f32(0.0) else f32(0.0)
                o["radius"] = avg_radius
                valid_out = True
                o["color"] = pack_rgb(0.0, 0.7, 0.0)
                o["count"] = f32(creation)
                a, dd = float(angle), float(distance)
                pr = float(f32(p.p_stable))
                if p.confidence_mode in (1, 3):
                    pr = float(f32(pr) * f32(math.exp(float((-f32(a)) * f32(a) / (f32(p.sigma_angle) * f32(p.sigma_angle))))))
                if p.confidence_mode in (2, 3):
                    pr = float(f32(pr) * f32(math.exp(float((-f32(dd)) * f32(dd) / (f32(p.sigma_distance) * f32(p.sigma_distance))))))
                pr = f32(pr)
                pr = pr if pr > d["p_unstable"] else d["p_unstable"]
                if pr >= f32(1.0):
                    tag.add("p:one")
                if pr <= d["p_unstable"]:
                    tag.add("p:unstable")
                pr = pr if pr < f32(1.0) else f32(1.0)
                q = float(pr / (f32(1.0) - pr))
                update_conf = f32(math.log(q)) if q != math.inf else f32(np.inf)
                conf_approx = q != math.inf
                tag.add("confidence_mode:%d" % p.confidence_mode)
                if (new_radius < old_radius and timestamp - creation < p.active_timestamps) or p.update_always:
                    tag.add("average" + (":always" if p.update_always else ""))
                    w1, w2 = f32(0.9), f32(0.1)
                    if p.weighting_scheme > 0:
                        w1 = old_weight
                        w2 = f32(1.0)
                        if p.weighting_scheme == 2:
                            w2 = dot3(n, view_dir)
                        sw = w1 + w2
                        o["weight"] = f32(p.max_weight) if f32(p.max_weight) < sw else sw
                        if sw == f32(p.max_weight):
                            tag.add("max_weight:equal")
                        if sw == 0.0:
                            tag.add("weights:zero_sum")
                        ssum = w1 + w2
                        w1 = w1 / ssum
                        w2 = w2 / ssum
                    tag.add("weighting_scheme:%d" % p.weighting_scheme)
                    avg_position = add3(scale3(w1, old_position), scale3(w2, v_global))
                    avg_normal, par = _slerp(old_normal, n_global, w1)
                    if par:
                        tag.add("slerp:parallel")
                    avg_prob = (w1 * model_prob + w2 * (f32(1.0) - data_prob)) if label_diff else (w1 * model_prob + w2 * data_prob)
                    if p.averaging_scheme == 1:
                        avg_position = add3(old_position, scale3(w2 * distance, old_normal))
                        tag.add("averaging_scheme:1")
                    avg_normal = normalize3(avg_normal)
                    spi = SPI(ci)
                    avg_position = xform_point(spi, avg_position)
                    avg_normal = xform_dir(spi, avg_normal)
                    o["x"], o["y"], o["z"], o["radius"] = (*avg_position, avg_radius)
                    o["nx"], o["ny"], o["nz"] = avg_normal
                    approx |= {"nx", "ny", "nz"}
                    o["color"] = pack_rgb(1.0, 0.0, 1.0)
                else:
                    tag.add("no_average")
            else:
                tag.add("no_match:" + ("distance" if not distance < f32(p.map_max_distance) else "angle"))
                if index[dpix] == k + 1:
                    update_conf = f32(math.log(float(d["p_unstable"]) / float(f32(1.0) - d["p_unstable"])))
                    conf_approx = True
                    o["color"] = pack_rgb(0.0, 1.0, 1.0)
                    tag.add("no_match:winner")
                else:
                    tag.add("no_match:not_winner")
        update_conf = update_conf - penalty
        if p.use_stability:
            c = (old_conf + update_conf) - d["log_prior"]
            if conf_approx:
                approx.add("confidence")
            elif c >= f32(20.0):
                tag.add("clamp20")
            o["confidence"] = c if c < f32(20.0) else f32(20.0)
        else:
            o["confidence"] = old_conf
        if o["confidence"] < d["log_unstable"] and p.use_stability:
            valid_out = False
            tag.add("removed:log_unstable")
        if not conf_approx and o["confidence"] == d["log_unstable"]:
            tag.add("log_unstable:equal")
        if mark is not None:
            if valid_out:
                integrated[mark] = 1
                tag.add("marks_pixel")
            else:
                tag.add("matched_but_removed")
        if avg_prob is not None:
            o["w"] = avg_prob
        if valid_out:
            valid_list.append(k)
            out.append(o)
            out_approx.append(approx)
        tags.append(tag)

    # K6d: new surfels, x-major pixel order
    new, gen_tags = [], {}
    for x in range(W):
        for y in range(H):
            Vp, Np, Rp = V[y, x], N[y, x], radius[y, x]
            invalid = (Vp[3] < f32(1.0)) or (Np[3] < f32(1.0)) or (Rp[3] < f32(0.5))
            v, n = v3(*Vp[:3]), v3(*Np[:3])
            dt = dot3(n, divs3(neg3(v), len3(v)))
            if integrated[y, x]:
                gen_tags[(y, x)] = "gen:integrated"
                continue
            if invalid:
                gen_tags[(y, x)] = "gen:invalid_r" if (Vp[3] >= 1 and Np[3] >= 1) else (
                    "gen:w_below_one" if (Vp[3] > 0.5 and Np[3] > 0.5) else "gen:invalid")
                continue
            if not dt > f32(0.01):
                gen_tags[(y, x)] = "gen:dot_rejected"
                continue
            ng = normalize3(n)
            o = np.zeros((), SURFEL_DTYPE)
            o["x"], o["y"], o["z"], o["radius"] = v[0], v[1], v[2], Rp[0]
            o["nx"], o["ny"], o["nz"] = ng
            mv = is_movable(S[y, x, 0] * f32(255.0))
            o["confidence"] = d["log_prior"] - f32(0.5) if mv else d["log_prior"]
            o["timestamp"] = np.uint32(timestamp)
            o["color"], o["weight"], o["count"] = pack_rgb(0.0, 0.0, 1.0), 1.0, f32(timestamp)
            o["r"], o["g"], o["b"], o["w"] = S[y, x]
            new.append(o)
            gen_tags[(y, x)] = "gen:new" + (":movable" if mv else "")

    # K6e: the submap window
    ext = f32(p.submap_extent)
    cx, cy = f32(2.0 * origin[0] * float(ext)), f32(2.0 * origin[1] * float(ext))
    extent = f32(2.0) * f32(p.submap_dimension) * ext + ext
    if p.partial_extraction and pending_extraction > 0:
        extent = extent + f32(2.0) * ext

    def keep(o):
        w = xform_point(SP(pose_index(o["count"])), v3(o["x"], o["y"], o["z"]))
        return not (int(np.uint32(o["timestamp"])) >> 31 or abs(w[0] - cx) > extent or abs(w[1] - cy) > extent)

    kept, kept_approx = [], []
    for i, (o, ap) in enumerate(zip(out, out_approx)):
        if keep(o):
            kept.append(o)
            kept_approx.append(ap)
        else:
            tags[valid_list[i]].add("submap:dropped")
    n_new_kept = 0
    for o in new:
        if keep(o):
            kept.append(o)
            kept_approx.append(set())
            n_new_kept += 1
    recs = np.array(kept, SURFEL_DTYPE) if kept else np.zeros(0, SURFEL_DTYPE)
    return dict(index=index, radius=radius, integrated=integrated, n_updated=len(out), n_new=len(new),
                n_updated_kept=len(kept) - n_new_kept, n_new_kept=n_new_kept, surfels=recs, approx=kept_approx, tags=tags, radius_tags=radius_tags,
                gen_tags=gen_tags, derived=d)


def _slerp(v0, v1, weight):
    """update_surfels.vert:113-124 in fp64, rounded once per output; parallel unit normals give acos 0, 1/sin inf and NaN
    weights, as the fp32 evaluation does"""
    c = float(dot3(normalize3(v0), normalize3(v1)))
    omega = math.acos(max(-1.0, min(1.0, c))) if c == c else float("nan")
    eta = 1.0 / math.sin(omega) if omega != 0.0 else math.inf
    w = float(weight)
    w0 = eta * math.sin(w * omega) if not (eta == math.inf and w * omega == 0.0) else float("nan")
    w1 = eta * math.sin((1.0 - w) * omega) if not (eta == math.inf and (1.0 - w) * omega == 0.0) else float("nan")
    out = add3(scale3(f32(w0), v0), scale3(f32(w1), v1))
    return out, omega == 0.0


def compare(model, surfels, what, tol=True):
    """the model's map against downloaded records: bits for exact fields (NaN as NaN), tolerances for the transcendental
    ones"""
    assert len(surfels) == len(model["surfels"]), "%s: %d surfels, model %d" % (what, len(surfels), len(model["surfels"]))
    for i, (a, b, ap) in enumerate(zip(surfels, model["surfels"], model["approx"])):
        for f in SURFEL_DTYPE.names:
            x, y = a[f], b[f]
            if f in ap:
                if f == "confidence":
                    ok = abs(float(x) - float(y)) <= TOL_CONF_ULPS * float(np.spacing(f32(max(abs(float(y)), 1.0))))
                else:
                    ok = (x != x and y != y) or abs(float(x) - float(y)) <= TOL_NORMAL
            elif f == "timestamp":
                ok = x == y
            else:
                ok = (x != x and y != y) or np.asarray(x, f32).view(np.uint32) == np.asarray(y, f32).view(np.uint32)
            assert ok, "%s: surfel %d field %s: %r vs model %r" % (what, i, f, x, y)
