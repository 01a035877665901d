"""TEST INFRASTRUCTURE: ctypes binding of the CPU oracle (oracle/*.c).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
The product (semantic_suma_b200/) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "build", "liborc.so")


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h", ".cpp")) or f == "Makefile"]
    srcs.append(os.path.join(_HERE, "..", "include", "suma_b200_loop.hpp"))
    stale = force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs)
    if stale:
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _LIB


class Params(C.Structure):
    _fields_ = [
        ("data_width", C.c_int32), ("data_height", C.c_int32),
        ("data_fov_up", C.c_float), ("data_fov_down", C.c_float),
        ("min_depth", C.c_float), ("max_depth", C.c_float),
        ("model_width", C.c_int32), ("model_height", C.c_int32),
        ("model_fov_up", C.c_float), ("model_fov_down", C.c_float),
        ("model_min_depth", C.c_float), ("model_max_depth", C.c_float),
        ("max_iterations", C.c_int32),
        ("stopping_threshold", C.c_double), ("delta", C.c_double),
        ("icp_max_distance", C.c_float), ("icp_max_angle", C.c_float),
        ("weighting", C.c_int32), ("factor", C.c_float),
        ("initialize_identity", C.c_int32), ("bilinear_sampling", C.c_int32),
        ("fallback_mode", C.c_int32),
        ("fallback_max_distance", C.c_float), ("fallback_max_angle", C.c_float),
        ("compose_rendering", C.c_int32), ("max_loop_closure_distance", C.c_float),
        ("min_radius", C.c_float), ("max_radius", C.c_float), ("max_angle", C.c_float),
        ("map_max_distance", C.c_float), ("map_max_angle", C.c_float),
        ("unstable_age", C.c_int32), ("confidence_mode", C.c_int32),
        ("confidence_threshold", C.c_float),
        ("p_stable", C.c_float), ("p_prior", C.c_float), ("sigma_angle", C.c_float), ("sigma_distance", C.c_float),
        ("use_stability", C.c_int32), ("active_timestamps", C.c_int32),
        ("max_weight", C.c_float),
        ("weighting_scheme", C.c_int32), ("averaging_scheme", C.c_int32), ("update_always", C.c_int32),
        ("submap_dimension", C.c_int32), ("submap_extent", C.c_float), ("partial_extraction", C.c_int32),
        ("label_offset_quirk", C.c_int32), ("render_after_update", C.c_int32),
    ]


SURFEL_DTYPE = np.dtype([
    ("x", "f4"), ("y", "f4"), ("z", "f4"), ("radius", "f4"),
    ("nx", "f4"), ("ny", "f4"), ("nz", "f4"), ("confidence", "f4"),
    ("timestamp", "u4"), ("color", "f4"), ("weight", "f4"), ("count", "f4"),
    ("r", "f4"), ("g", "f4"), ("b", "f4"), ("w", "f4"),
])
assert SURFEL_DTYPE.itemsize == 64

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        L = _lib
        for name in ("atan2f",):
            pass
        L.orc_t_atan2f.restype = C.c_float; L.orc_t_atan2f.argtypes = [C.c_float, C.c_float]
        for n in ("asinf", "acosf", "sinf", "expf", "logf"):
            f = getattr(L, "orc_t_" + n); f.restype = C.c_float; f.argtypes = [C.c_float]
        L.orc_t_sincos.argtypes = [C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.orc_check_params.restype = C.c_char_p
        L.orc_map_create.restype = C.c_void_p
        L.orc_slam_create.restype = C.c_void_p
        L.orc_slam_map.restype = C.c_void_p
        L.orc_map_size.restype = C.c_uint32
        L.orc_map_timestamp.restype = C.c_uint32
        L.orc_map_download.restype = C.c_uint32
        L.orc_slam_timestamp.restype = C.c_uint32
        L.orc_icp_minimize.restype = C.c_int
        L.orc_gn_step.restype = C.c_int
        L.orc_set_threads.restype = C.c_int; L.orc_set_threads.argtypes = [C.c_int]
        L.orc_loop_attach.restype = C.c_void_p
        L.orc_loop_edges.restype = C.c_uint32
        L.orc_loop_integrate.restype = C.c_uint32
    return _lib


def gl_sums(on):
    """sum the 48 ICP values the way the reference's GL path does (orc_core.c orc_set_gl_sums) instead of exactly; returns
    the previous mode. Only for comparisons with oracle/_ref/libsuma_ref_full.so."""
    return int(lib().orc_set_gl_sums(int(bool(on))))


def set_threads(n=0):
    """host threads for the oracle's loops (0 = all cores, capped at 64); results do not depend on it"""
    return int(lib().orc_set_threads(int(n)))


def _p(a, t=C.c_float):
    if a is None:
        return None
    return a.ctypes.data_as(C.POINTER(t))


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def default_params(**kw):
    p = Params()
    lib().orc_default_params(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise KeyError(k)
        setattr(p, k, v)
    return p


def check_params(p):
    """None if sb_create accepts these parameters, otherwise the reason it refuses them (orc_check_params)"""
    why = lib().orc_check_params(C.byref(p))
    return None if why is None else why.decode()


def _create(fn, p):
    why = check_params(p)
    if why is not None:
        raise ValueError("parameters refused: " + why)
    return C.c_void_p(fn(C.byref(p)))


def colmajor(T, dtype):
    """numpy (row-major) 4x4 -> 16 values in column-major order (Eigen .data())."""
    return np.ascontiguousarray(np.asarray(T, dtype=dtype).T).reshape(16)


def from_colmajor(a):
    return np.asarray(a).reshape(4, 4).T.copy()


def scalar(name, *args):
    return getattr(lib(), "orc_t_" + name)(*args)


def sincos(x):
    s, c = C.c_double(), C.c_double()
    lib().orc_t_sincos(x, C.byref(s), C.byref(c))
    return s.value, c.value


def preprocess(p, pts, labels=None, probs=None, timestamp=100):
    pts = _f32(pts); labels = _f32(labels); probs = _f32(probs)
    n = pts.shape[0]
    H, W = p.data_height, p.data_width
    v = np.empty((H, W, 4), np.float32); nm = np.empty_like(v); s = np.empty_like(v)
    lib().orc_preprocess(C.byref(p), _p(pts), _p(labels), _p(probs), C.c_uint32(n), C.c_uint32(timestamp), _p(v), _p(nm),
                         _p(s))
    return v, nm, s


def icp_jacobian(p, data, model, pose, iteration=0, max_distance=None, max_angle=None, rows=None, semantic=True):
    dv, dn, ds = [_f32(a) for a in data]
    mv, mn, ms = [_f32(a) for a in model]
    if not semantic:
        ds = ms = None
    out48 = np.zeros(48, np.float64); raw = np.zeros(32, np.int64)
    r0, r1 = rows if rows is not None else (0, p.data_height)
    pose_cm = colmajor(pose, np.float64)
    lib().orc_icp_jacobian(C.byref(p), _p(dv), _p(dn), _p(ds), _p(mv), _p(mn), _p(ms), _p(pose_cm, C.c_double),
                           C.c_int32(iteration),
                           C.c_float(p.icp_max_distance if max_distance is None else max_distance),
                           C.c_float(p.icp_max_angle if max_angle is None else max_angle), C.c_int32(r0),
                           C.c_int32(r1), _p(out48, C.c_double), _p(raw, C.c_int64))
    return out48, raw


def icp_unpack(raw):
    raw = np.ascontiguousarray(raw, np.int64)
    out48 = np.zeros(48, np.float64)
    lib().orc_icp_unpack(_p(raw, C.c_int64), _p(out48, C.c_double))
    return out48


def icp_jacobian_fp32gl(p, data, model, pose, iteration=0):
    dv, dn, ds = [_f32(a) for a in data]
    mv, mn, ms = [_f32(a) for a in model]
    out48 = np.zeros(48, np.float32)
    pose_cm = colmajor(pose, np.float64)
    lib().orc_icp_jacobian_fp32gl(C.byref(p), _p(dv), _p(dn), _p(ds), _p(mv), _p(mn), _p(ms), _p(pose_cm, C.c_double),
                                  C.c_int32(iteration), C.c_float(p.icp_max_distance), C.c_float(p.icp_max_angle),
                                  _p(out48))
    return out48


def icp_minimize(p, data, model, T0, max_distance=None, max_angle=None):
    dv, dn, ds = [_f32(a) for a in data]
    mv, mn, ms = [_f32(a) for a in model]
    pose_out = np.zeros(16, np.float64); out48 = np.zeros(48, np.float64)
    hist = np.zeros((p.max_iterations + 2) * 16, np.float64); hl = C.c_int32(0)
    T0cm = colmajor(T0, np.float64)
    k = lib().orc_icp_minimize(C.byref(p), _p(dv), _p(dn), _p(ds), _p(mv), _p(mn), _p(ms), _p(T0cm, C.c_double),
                               C.c_float(p.icp_max_distance if max_distance is None else max_distance),
                               C.c_float(p.icp_max_angle if max_angle is None else max_angle),
                               _p(pose_out, C.c_double), _p(out48, C.c_double), _p(hist, C.c_double), C.byref(hl))
    history = [from_colmajor(hist[16 * i:16 * i + 16]) for i in range(hl.value)]
    return from_colmajor(pose_out), out48, k, history


def se3_exp(x):
    x = np.ascontiguousarray(x, np.float64); T = np.zeros(16, np.float64)
    lib().orc_se3_exp(_p(x, C.c_double), _p(T, C.c_double))
    return from_colmajor(T)


def se3_log(T):
    Tc = colmajor(T, np.float64); x = np.zeros(6, np.float64)
    lib().orc_se3_log(_p(Tc, C.c_double), _p(x, C.c_double))
    return x


def ldlt_solve6(A, b):
    A = np.ascontiguousarray(np.asarray(A, np.float64).T).reshape(36)
    b = np.ascontiguousarray(b, np.float64); x = np.zeros(6, np.float64)
    lib().orc_ldlt_solve6(_p(A, C.c_double), _p(b, C.c_double), _p(x, C.c_double))
    return x


class Map:
    def __init__(self, p, handle=None):
        self.p = p
        self._own = handle is None
        self.h = None
        self.h = _create(lib().orc_map_create, p) if handle is None else C.c_void_p(handle)

    def __del__(self):
        if getattr(self, "_own", False) and self.h:
            lib().orc_map_destroy(self.h); self.h = None

    def size(self):
        return lib().orc_map_size(self.h)

    def timestamp(self):
        return lib().orc_map_timestamp(self.h)

    def download(self):
        n = self.size()
        a = np.zeros(max(n, 1), SURFEL_DTYPE)
        k = lib().orc_map_download(self.h, a.ctypes.data_as(C.c_void_p), C.c_uint32(n))
        return a[:k]

    def upload(self, surfels, timestamp):
        a = np.ascontiguousarray(surfels, SURFEL_DTYPE)
        lib().orc_map_upload(self.h, a.ctypes.data_as(C.c_void_p), C.c_uint32(a.shape[0]), C.c_uint32(timestamp))

    def set_pose(self, t, pose):
        pc = colmajor(pose, np.float32)
        lib().orc_map_set_pose(self.h, C.c_uint32(t), _p(pc))

    def _mframe(self):
        H, W = self.p.model_height, self.p.model_width
        return [np.zeros((H, W, 4), np.float32) for _ in range(3)]

    def render(self, pose_old, pose_new, conf_thr):
        v, n, s = self._mframe()
        lib().orc_map_render(self.h, _p(colmajor(pose_old, np.float32)), _p(colmajor(pose_new, np.float32)),
                             C.c_float(conf_thr), _p(v), _p(n), _p(s))
        return v, n, s

    def render_active(self, pose, conf_thr):
        lib().orc_map_render_active(self.h, _p(colmajor(pose, np.float32)), C.c_float(conf_thr))

    def render_inactive(self, pose, conf_thr):
        lib().orc_map_render_inactive(self.h, _p(colmajor(pose, np.float32)), C.c_float(conf_thr))

    def render_composed(self, pose_old, pose_new, conf_thr):
        lib().orc_map_render_composed(self.h, _p(colmajor(pose_old, np.float32)), _p(colmajor(pose_new, np.float32)),
                                      C.c_float(conf_thr))

    def frame(self, which):
        v, n, s = self._mframe()
        lib().orc_map_get_frame(self.h, C.c_int(which), _p(v), _p(n), _p(s))
        return v, n, s

    def update(self, pose, frame):
        fv, fn, fs = [_f32(a) for a in frame]
        lib().orc_map_update(self.h, _p(colmajor(pose, np.float32)), _p(fv), _p(fn), _p(fs))

    def update_debug(self):
        H, W = self.p.data_height, self.p.data_width
        idx = np.zeros((H, W), np.uint32); rad = np.zeros((H, W, 4), np.float32); integ = np.zeros((H, W), np.uint8)
        nu, nn = C.c_uint32(0), C.c_uint32(0)
        lib().orc_map_get_update_debug(self.h, _p(idx, C.c_uint32), _p(rad), _p(integ, C.c_uint8), C.byref(nu),
                                       C.byref(nn))
        return idx, rad, integ, nu.value, nn.value

    def submap_origin(self):
        i, j, pend = C.c_int32(0), C.c_int32(0), C.c_uint32(0)
        lib().orc_map_get_submap_origin(self.h, C.byref(i), C.byref(j), C.byref(pend))
        return i.value, j.value, pend.value


class Slam:
    def __init__(self, p):
        self.p = p
        self.h = None
        self.h = _create(lib().orc_slam_create, p)
        self.map = Map(p, handle=lib().orc_slam_map(self.h))
        self.loop = None

    def enable_loop_closure(self, search_distance=50.0, min_trajectory_distance=200.0, min_verifications=5,
                            residual_threshold=1.15, outlier_threshold=1.1, valid_threshold=0.95):
        """SurfelMapping::checkLoopClosure between updatePose() and updateMap() (oracle/orc_loop.cpp)"""
        self.loop = C.c_void_p(lib().orc_loop_attach(self.h, C.c_float(search_distance), C.c_float(min_trajectory_distance),
                                                     C.c_int32(min_verifications), C.c_float(residual_threshold),
                                                     C.c_float(outlier_threshold), C.c_float(valid_threshold)))

    def loop_info(self):
        info = np.zeros(12, np.int64); ratios = np.zeros(5, np.float64); pose = np.zeros(16, np.float64)
        lib().orc_loop_info(self.loop, _p(info, C.c_int64), _p(ratios, C.c_double), _p(pose, C.c_double))
        keys = ("loop_count", "time_without_loop_closure", "candidates_tested", "loop_edges_added", "unverified",
                "already_verified", "found_candidate", "use_candidate", "optimisation_requested", "last_added_candidate",
                "n_edges", "n_poses")
        d = dict(zip(keys, (int(x) for x in info)))
        d.update(valid_ratio=np.float32(ratios[0]), outlier_ratio=np.float32(ratios[1]), rel_error=np.float32(ratios[2]),
                 residual_old=ratios[3], residual_new=ratios[4], current_pose_old=from_colmajor(pose))
        return d

    def integrate_loop_closures(self, poses=None):
        """SurfelMapping::integrateLoopClosures before the next scan; poses=None: the identity "optimiser" """
        if poses is None:
            return int(lib().orc_loop_integrate(self.loop, None, C.c_uint32(0)))
        a = np.ascontiguousarray([colmajor(P, np.float64) for P in poses], np.float64)
        return int(lib().orc_loop_integrate(self.loop, _p(a, C.c_double), C.c_uint32(a.shape[0])))

    def loop_edges(self):
        n = int(self.loop_info()["n_edges"])
        ft = np.zeros((max(n, 1), 2), np.int32); rel = np.zeros((max(n, 1), 16), np.float64)
        lib().orc_loop_edges(self.loop, _p(ft, C.c_int32), _p(rel, C.c_double), C.c_uint32(n))
        return [(int(ft[i, 0]), int(ft[i, 1]), from_colmajor(rel[i])) for i in range(n)]

    def __del__(self):
        if self.h:
            if getattr(self, "loop", None):
                lib().orc_loop_detach(self.loop); self.loop = None
            lib().orc_slam_destroy(self.h); self.h = None

    def process_scan(self, pts, labels=None, probs=None):
        pts = _f32(pts); labels = _f32(labels); probs = _f32(probs)
        lib().orc_slam_process_scan(self.h, _p(pts), _p(labels), _p(probs), C.c_uint32(pts.shape[0]))

    def pose(self):
        a = np.zeros(16, np.float64)
        lib().orc_slam_get_pose(self.h, _p(a, C.c_double))
        return from_colmajor(a)

    def timestamp(self):
        return lib().orc_slam_timestamp(self.h)

    def stats(self):
        a = np.zeros(16, np.float64)
        lib().orc_slam_get_stats(self.h, _p(a, C.c_double))
        return dict(iterations=a[0], F=a[1], inlier=a[2], outlier=a[3], invalid=a[4], inlier_residual=a[5],
                    track_loss=a[6], surfels=a[7], t_preprocess=a[8], t_icp=a[9], t_mapping=a[10], t_complete=a[11])

    def frame(self, which):
        P = (self.p.data_height, self.p.data_width) if which == 0 else (self.p.model_height, self.p.model_width)
        v, n, s = [np.zeros(P + (4,), np.float32) for _ in range(3)]
        lib().orc_slam_get_frame(self.h, C.c_int(which), _p(v), _p(n), _p(s))
        return v, n, s
