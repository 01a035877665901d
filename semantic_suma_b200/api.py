"""Host-side mirror of the reference's operator surface on top of the C ABI (include/suma_b200.h).

The reference's boundary classes are C++ (core/SurfelMapping.h, Frame2Model.h, SurfelMap.h, Preprocessing.h,
LieGaussNewton.h, Frame.h); include/suma_b200.hpp is the C++ mirror. This module is the same surface for Python
callers (tests, bench): same class and method names, same argument meaning. It only talks to libsuma_b200.so through
ctypes -- plain pointers and sizes -- and fails loudly when the CUDA library is missing: there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build

SB_OK = 0
SB_ERR_INVALID = -1
_ERRORS = {-1: "SB_ERR_INVALID", -2: "SB_ERR_CUDA", -3: "SB_ERR_NOMEM", -4: "SB_ERR_CAPACITY", -5: "SB_ERR_STATE",
           -6: "SB_ERR_NOGPU"}


class SumaError(RuntimeError):
    pass


class LoopParams(C.Structure):  # sb_loop_params
    _fields_ = [("search_distance", C.c_float), ("min_trajectory_distance", C.c_float), ("min_verifications", C.c_int32),
                ("residual_threshold", C.c_float), ("outlier_threshold", C.c_float), ("valid_threshold", C.c_float)]


class LoopInfo(C.Structure):  # sb_loop_info
    _fields_ = [(n, C.c_uint32) for n in ("enabled", "loop_count", "time_without_loop_closure", "candidates_tested",
                                          "loop_edges_added", "unverified", "already_verified", "found_candidate",
                                          "use_candidate", "optimisation_requested")] + \
               [("last_added_candidate", C.c_int32), ("n_edges", C.c_uint32), ("n_poses", C.c_uint32),
                ("valid_ratio", C.c_float), ("outlier_ratio", C.c_float), ("rel_error", C.c_float),
                ("residual_old", C.c_double), ("residual_new", C.c_double), ("current_pose_old", C.c_double * 16)]


class LoopEdge(C.Structure):  # sb_loop_edge
    _fields_ = [("from_", C.c_int32), ("to", C.c_int32), ("rel_pose", C.c_double * 16)]


class TileCacheInfo(C.Structure):  # sb_tile_cache_info
    _fields_ = [(n, C.c_uint32) for n in ("managed", "tiles_in_pool", "tiles_on_host", "pad")] + \
               [(n, C.c_uint64) for n in ("pool_capacity", "pool_used", "pool_referenced", "host_capacity", "host_used",
                                          "reclaims", "reclaim_moved", "evictions", "host_fills", "dropped")]


HOST_UNBOUNDED = 2**64 - 1  # sb_set_tile_cache: no bound on the host tier


class DeskewParams(C.Structure):  # sb_deskew_params
    _fields_ = [("mode", C.c_int32), ("ref_time", C.c_float), ("start_azimuth", C.c_float), ("clockwise", C.c_int32)]


DESKEW_MODES = {"off": 0, "times": 1, "azimuth": 2}


def deskew_params(mode="off", ref_time=0.5, start_azimuth=np.pi, clockwise=True):
    """sb_deskew_params; mode: 0 / "off", 1 / "times" (per-point times), 2 / "azimuth" """
    d = DeskewParams()
    lib().sb_default_deskew(C.byref(d))
    d.mode = DESKEW_MODES.get(mode, mode) if isinstance(mode, str) else int(mode)
    d.ref_time, d.start_azimuth, d.clockwise = ref_time, start_azimuth, 1 if clockwise else 0
    return d


class PointLabel(C.Structure):  # sb_point_label
    _fields_ = [("pixel", C.c_int32), ("flags", C.c_uint32), ("frame_label", C.c_uint32), ("frame_prob", C.c_float),
                ("map_pixel", C.c_int32), ("map_label", C.c_uint32), ("map_prob", C.c_float), ("map_range", C.c_float)]


# sb_point_label as a numpy structured dtype (same names, offsets and 32-byte size) and its flags
POINT_LABEL_DTYPE = np.dtype({"names": [n for n, _ in PointLabel._fields_],
                              "formats": ["<i4", "<u4", "<u4", "<f4", "<i4", "<u4", "<f4", "<f4"],
                              "offsets": [getattr(PointLabel, n).offset for n, _ in PointLabel._fields_],
                              "itemsize": C.sizeof(PointLabel)})
POINT_WON, POINT_VERTEX, POINT_INTEGRATED, POINT_MAP = 1, 2, 4, 8


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

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


# XML key (config/default.xml) -> struct field
XML_KEYS = {
    "max iterations": "max_iterations", "stopping threshold": "stopping_threshold", "icp-max-distance": "icp_max_distance",
    "icp-max-angle": "icp_max_angle", "fallback-max-distance": "fallback_max_distance",
    "fallback-max-angle": "fallback_max_angle", "map-max-distance": "map_max_distance",
    "map-max-angle": "map_max_angle", "submap-dimension": "submap_dimension", "submap-extent": "submap_extent",
    "partial-extraction": "partial_extraction",
}
_WEIGHTING = {"none": 0, "huber": 1, "turkey": 2, "stability": 3}

SURFEL_DTYPE = np.dtype([
    ("x", "f4"), ("y", "f4"), ("z", "f4"), ("radius", "f4"),
    ("nx", "f4"), ("ny", "f4"), ("nz", "f4"), ("confidence", "f4"),
    ("timestamp", "u4"), ("color", "f4"), ("weight", "f4"), ("count", "f4"),
    ("r", "f4"), ("g", "f4"), ("b", "f4"), ("w", "f4"),
])

_lib = None


def library_path():
    return _build.LIB


def lib(build_if_missing=True):
    """Loads libsuma_b200.so (building it with nvcc when stale). Raises if it cannot be had: no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if build_if_missing:
        try:
            path = _build.build()
        except Exception as e:  # noqa: BLE001 - surfaced below if the library is really absent
            if not os.path.exists(_build.LIB):
                raise SumaError("libsuma_b200.so is missing and could not be built: %s" % e)
    if not os.path.exists(path):
        raise SumaError("libsuma_b200.so not found at %s (run python -m semantic_suma_b200.build)" % path)
    L = C.CDLL(path)
    vp, u32, i32, f32, f64 = C.c_void_p, C.c_uint32, C.c_int32, C.c_float, C.c_double
    pf, pd, pv = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_void_p)
    sig = {
        "sb_default_params": [C.POINTER(Params)],
        "sb_create": [C.POINTER(Params), C.c_int, pv],
        "sb_destroy": [vp], "sb_reset": [vp], "sb_set_params": [vp, C.POINTER(Params)], "sb_synchronize": [vp],
        "sb_get_params": [vp, C.POINTER(Params)],
        "sb_frame_create": [vp, C.c_int, C.c_int, pv], "sb_frame_destroy": [vp], "sb_frame_copy": [vp, vp],
        "sb_frame_download": [vp, C.c_int, vp], "sb_frame_upload": [vp, C.c_int, vp],
        "sb_frame_size": [vp, C.POINTER(C.c_int), C.POINTER(C.c_int)],
        "sb_preprocess": [vp, vp, vp, vp, u32, u32, C.c_int, vp],
        "sb_map_render": [vp, pf, pf, f32, vp], "sb_map_render_active": [vp, pf, f32],
        "sb_map_render_inactive": [vp, pf, f32], "sb_map_render_composed": [vp, pf, pf, f32],
        "sb_map_frame": [vp, C.c_int, pv],
        "sb_icp_jacobian": [vp, vp, vp, pd, C.c_int, f32, f32, C.c_int, C.c_int, pd, C.POINTER(C.c_int64)],
        "sb_icp_minimize": [vp, vp, vp, pd, C.c_int, f64, f64, f32, f32, pd, pd, C.POINTER(C.c_int), pd,
                            C.POINTER(C.c_int)],
        "sb_gn_step": [pd, f64, f64, f64, pd, pd],
        "sb_ldlt_solve6": [pd, pd, pd],
        "sb_map_update": [vp, pf, vp], "sb_map_update_poses": [vp, pf, u32], "sb_map_set_pose": [vp, u32, pf],
        "sb_pose_table_info": [vp, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32)],
        "sb_map_size": [vp, C.POINTER(u32)], "sb_map_timestamp": [vp, C.POINTER(u32)],
        "sb_map_download": [vp, vp, u32, C.POINTER(u32)], "sb_map_upload": [vp, vp, u32, u32],
        "sb_map_update_debug": [vp, vp, vp, vp, C.POINTER(u32), C.POINTER(u32)],
        "sb_map_submap_origin": [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(u32)],
        "sb_process_scan": [vp, vp, vp, vp, u32, C.c_int], "sb_prefetch_scan": [vp, vp, vp, vp, u32],
        "sb_set_loop_closure": [vp, C.c_int, vp], "sb_get_loop_info": [vp, vp], "sb_get_loop_edges": [vp, vp, u32, C.POINTER(u32)],
        "sb_set_current_pose": [vp, pd], "sb_default_loop_params": [vp],
        "sb_integrate_loop_closures": [vp, pd, u32, C.POINTER(u32)],
        "sb_get_pose": [vp, pd], "sb_get_last_pose": [vp, pd], "sb_timestamp": [vp, C.POINTER(u32)], "sb_slam_frame": [vp, C.c_int, pv],
        "sb_get_statistics": [vp, pd],
        "sb_comm_export": [vp, vp], "sb_comm_init": [vp, C.c_int, C.c_int, vp, C.c_int, C.c_int],
        "sb_comm_shutdown": [vp],
        "sb_comm_set_callback": [vp, vp, vp, C.c_int, C.c_int],
        "sb_profile_enable": [vp, C.c_int], "sb_profile_collect": [vp, pd, C.POINTER(C.c_uint64), C.c_int],
        "sb_profile_kernels": [],
        "sb_state_size": [vp, C.POINTER(C.c_uint64)], "sb_state_save": [vp, vp, C.c_uint64, C.POINTER(C.c_uint64)],
        "sb_state_load": [vp, vp, C.c_uint64],
        "sb_set_tile_cache": [vp, u32, C.c_uint64], "sb_get_tile_cache_info": [vp, C.POINTER(TileCacheInfo)],
        "sb_set_deskew": [vp, C.POINTER(DeskewParams)], "sb_get_deskew": [vp, C.POINTER(DeskewParams)],
        "sb_process_scan_timed": [vp, vp, vp, vp, vp, u32, C.c_int],
        "sb_preprocess_deskew": [vp, vp, vp, vp, vp, u32, u32, C.POINTER(DeskewParams), pd, C.c_int, vp],
        "sb_set_point_labels": [vp, C.c_int], "sb_get_point_labels": [vp, vp, u32, C.POINTER(u32), C.c_int],
    }
    for name, args in sig.items():
        fn = getattr(L, name)
        fn.argtypes = args
        fn.restype = C.c_int
    L.sb_last_error.argtypes = [vp]; L.sb_last_error.restype = C.c_char_p
    L.sb_stream.argtypes = [vp]; L.sb_stream.restype = vp
    L.sb_launch_count.argtypes = [vp]; L.sb_launch_count.restype = C.c_uint64
    L.sb_device_count.argtypes = []; L.sb_device_count.restype = C.c_int
    L.sb_profile_name.argtypes = [C.c_int]; L.sb_profile_name.restype = C.c_char_p
    L.sb_se3_exp.argtypes = [pd, pd]; L.sb_se3_exp.restype = None
    L.sb_se3_log.argtypes = [pd, pd]; L.sb_se3_log.restype = None
    L.sb_icp_unpack.argtypes = [C.POINTER(C.c_int64), pd]; L.sb_icp_unpack.restype = None
    L.sb_default_deskew.argtypes = [C.POINTER(DeskewParams)]; L.sb_default_deskew.restype = None
    _lib = L
    return L


EXPORTED_SYMBOLS = [
    "sb_default_params", "sb_create", "sb_destroy", "sb_reset", "sb_set_params", "sb_get_params", "sb_last_error",
    "sb_synchronize",
    "sb_device_count", "sb_stream", "sb_launch_count", "sb_frame_create", "sb_frame_destroy", "sb_frame_copy",
    "sb_frame_download", "sb_frame_upload", "sb_frame_size", "sb_preprocess", "sb_map_render", "sb_map_render_active",
    "sb_map_render_inactive", "sb_map_render_composed", "sb_map_frame", "sb_icp_jacobian", "sb_icp_unpack",
    "sb_icp_minimize", "sb_se3_exp", "sb_se3_log", "sb_ldlt_solve6", "sb_gn_step", "sb_map_update",
    "sb_map_update_poses", "sb_map_size", "sb_map_timestamp", "sb_map_download", "sb_map_upload", "sb_map_set_pose",
    "sb_map_update_debug", "sb_map_submap_origin", "sb_pose_table_info", "sb_process_scan", "sb_prefetch_scan", "sb_get_pose", "sb_get_last_pose", "sb_timestamp", "sb_slam_frame",
    "sb_get_statistics", "sb_comm_export", "sb_comm_init", "sb_comm_shutdown", "sb_comm_set_callback",
    "sb_profile_enable", "sb_default_loop_params", "sb_set_loop_closure", "sb_get_loop_info", "sb_get_loop_edges",
    "sb_set_current_pose", "sb_integrate_loop_closures",
    "sb_profile_kernels", "sb_profile_name", "sb_profile_collect", "sb_state_size", "sb_state_save", "sb_state_load",
    "sb_set_tile_cache", "sb_get_tile_cache_info",
    "sb_default_deskew", "sb_set_deskew", "sb_get_deskew", "sb_process_scan_timed", "sb_preprocess_deskew",
    "sb_set_point_labels", "sb_get_point_labels",
]


def default_params(**kw):
    p = Params()
    lib().sb_default_params(C.byref(p))
    for k, v in kw.items():
        k = XML_KEYS.get(k, k)
        if k == "weighting" and isinstance(v, str):
            v = _WEIGHTING[v]
        if not hasattr(p, k):
            raise KeyError(k)
        setattr(p, k, v)
    return p


def colmajor(T, dtype):
    return np.ascontiguousarray(np.asarray(T, dtype=dtype).T).reshape(16)


def from_colmajor(a):
    return np.asarray(a).reshape(4, 4).T.copy()


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _vp(a):
    if a is None:
        return None
    return C.c_void_p(a.ctypes.data)


class Context:
    """One CUDA device + stream (the role the GL context plays in the reference)."""

    def __init__(self, params, device=0):
        self.params = params
        self.h = C.c_void_p()
        rc = lib().sb_create(C.byref(params), device, C.byref(self.h))
        if rc != SB_OK:
            raise SumaError("sb_create failed: %s (libsuma_b200 needs a CUDA device; there is no CPU fallback)" %
                            _ERRORS.get(rc, rc))

    def check(self, rc, what=""):
        if rc != SB_OK:
            msg = lib().sb_last_error(self.h)
            raise SumaError("%s: %s %s" % (what, _ERRORS.get(rc, rc), msg.decode() if msg else ""))

    def close(self):
        if self.h:
            lib().sb_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    def synchronize(self):
        self.check(lib().sb_synchronize(self.h), "synchronize")

    def launch_count(self):
        return int(lib().sb_launch_count(self.h))

    def stream(self):
        return lib().sb_stream(self.h)

    def profile(self, on):
        self.check(lib().sb_profile_enable(self.h, 1 if on else 0), "profile_enable")

    def profile_collect(self):
        """{kernel name: (total_ms, launches)} since the last call (CUDA events on the context's stream)."""
        n = lib().sb_profile_kernels()
        ms = np.zeros(n); cnt = np.zeros(n, np.uint64)
        self.check(lib().sb_profile_collect(self.h, _dp(ms), cnt.ctypes.data_as(C.POINTER(C.c_uint64)), n), "profile")
        return {lib().sb_profile_name(i).decode(): (float(ms[i]), int(cnt[i])) for i in range(n) if cnt[i]}

    def get_params(self):
        """the parameters in effect (sb_get_params)"""
        p = Params()
        self.check(lib().sb_get_params(self.h, C.byref(p)), "get_params")
        return p

    def set_tile_cache(self, pool_surfels, host_surfels=None):
        """Managed submap tile cache (sb_set_tile_cache): pool_surfels in HBM (500 000 .. 16 M), host_surfels in pinned
        host memory (None or inf: no bound). Only while the cache is empty: after creation or reset."""
        if host_surfels is None or host_surfels == float("inf"):
            host_surfels = HOST_UNBOUNDED
        self.check(lib().sb_set_tile_cache(self.h, int(pool_surfels), int(host_surfels)), "set_tile_cache")

    def tile_cache_info(self):
        """counters of the submap tile cache (sb_get_tile_cache_info) as a dict"""
        o = TileCacheInfo()
        self.check(lib().sb_get_tile_cache_info(self.h, C.byref(o)), "get_tile_cache_info")
        return {n: int(getattr(o, n)) for n, _ in TileCacheInfo._fields_ if n != "pad"}

    def pose_table_info(self):
        """the pose table's capacity and the window [begin, end) of its product tables (sb_pose_table_info) as a dict"""
        cap, b, e = C.c_uint32(), C.c_uint32(), C.c_uint32()
        self.check(lib().sb_pose_table_info(self.h, C.byref(cap), C.byref(b), C.byref(e)), "pose_table_info")
        return {"capacity": cap.value, "begin": b.value, "end": e.value}

    def set_params(self, params):
        self.check(lib().sb_set_params(self.h, C.byref(params)), "set_params")
        self.params = params

    def set_deskew(self, mode="off", ref_time=0.5, start_azimuth=np.pi, clockwise=True):
        """per-point deskewing of the scans (sb_set_deskew): mode "off" / "times" / "azimuth" (or 0 / 1 / 2)"""
        d = deskew_params(mode, ref_time, start_azimuth, clockwise)
        self.check(lib().sb_set_deskew(self.h, C.byref(d)), "set_deskew")

    def get_deskew(self):
        """the deskewing setting in effect as a dict (sb_get_deskew)"""
        d = DeskewParams()
        self.check(lib().sb_get_deskew(self.h, C.byref(d)), "get_deskew")
        return {"mode": int(d.mode), "ref_time": float(d.ref_time), "start_azimuth": float(d.start_azimuth),
                "clockwise": bool(d.clockwise)}


class Frame:
    """core/Frame.h:21-79 -- vertex / normal / semantic maps living on the device."""

    def __init__(self, ctx, width=None, height=None, handle=None):
        self.ctx = ctx
        self._own = handle is None
        if handle is None:
            self.h = C.c_void_p()
            ctx.check(lib().sb_frame_create(ctx.h, width, height, C.byref(self.h)), "frame_create")
        else:
            self.h = C.c_void_p(handle)
        w, h = C.c_int(), C.c_int()
        lib().sb_frame_size(self.h, C.byref(w), C.byref(h))
        self.width, self.height = w.value, h.value

    def __del__(self):
        if getattr(self, "_own", False) and self.h and self.ctx.h:
            lib().sb_frame_destroy(self.h)
            self.h = None

    def _get(self, which):
        a = np.empty((self.height, self.width, 4), np.float32)
        self.ctx.check(lib().sb_frame_download(self.h, which, _vp(a)), "frame_download")
        return a

    def _set(self, which, a):
        a = np.ascontiguousarray(a, np.float32)
        assert a.shape == (self.height, self.width, 4)
        self.ctx.check(lib().sb_frame_upload(self.h, which, _vp(a)), "frame_upload")

    vertex_map = property(lambda s: s._get(0), lambda s, a: s._set(0, a))
    normal_map = property(lambda s: s._get(1), lambda s, a: s._set(1, a))
    semantic_map = property(lambda s: s._get(2), lambda s, a: s._set(2, a))

    def maps(self):
        return self._get(0), self._get(1), self._get(2)

    def upload(self, maps):
        for i, a in enumerate(maps):
            self._set(i, a)

    def copy(self, other):  # Frame::copy
        self.ctx.check(lib().sb_frame_copy(self.h, other.h), "frame_copy")


class Preprocessing:
    """core/Preprocessing.h:47-58"""

    def __init__(self, ctx):
        self.ctx = ctx

    def process(self, points, frame, labels=None, probs=None, timestamp=100, times=None, deskew=None, motion=None):
        """deskew: None (the points as they are), or a DeskewParams / dict of deskew_params() arguments, with
        motion = the sweep's 4x4 motion (None = identity) and times = the per-point sweep times of mode 1"""
        pts = np.ascontiguousarray(points, np.float32)
        lab = None if labels is None else np.ascontiguousarray(labels, np.float32)
        prb = None if probs is None else np.ascontiguousarray(probs, np.float32)
        if deskew is None and times is None and motion is None:
            self.ctx.check(lib().sb_preprocess(self.ctx.h, _vp(pts), _vp(lab), _vp(prb), pts.shape[0], timestamp, 0,
                                               frame.h), "preprocess")
            return
        d = deskew if isinstance(deskew, DeskewParams) else deskew_params(**(deskew or {}))
        tms = None if times is None else np.ascontiguousarray(times, np.float32)
        m = None if motion is None else colmajor(motion, np.float64)
        self.ctx.check(lib().sb_preprocess_deskew(self.ctx.h, _vp(pts), _vp(lab), _vp(prb), _vp(tms), pts.shape[0],
                                                  timestamp, C.byref(d), None if m is None else _dp(m), 0, frame.h),
                       "preprocess_deskew")


class Frame2Model:
    """core/Frame2Model.h:28-73 + core/Objective.h:14-82"""

    def __init__(self, ctx, max_distance=None, max_angle=None):
        self.ctx = ctx
        p = ctx.params
        self.max_distance = p.icp_max_distance if max_distance is None else max_distance
        self.max_angle = p.icp_max_angle if max_angle is None else max_angle
        self.pose_ = np.eye(4)
        self.iteration_ = 0
        self.current = self.last = None
        self.out48 = np.zeros(48)
        self.raw32 = np.zeros(32, np.int64)

    def setData(self, current, last):
        self.current, self.last = current, last
        self.iteration_ = 0

    def initialize(self, T0):
        self.pose_ = np.array(T0, np.float64)

    def num_parameters(self):
        return 6

    def jacobianProducts(self, rows=None):
        """returns (F, JtJ[6,6], Jtf[6])"""
        pc = colmajor(self.pose_, np.float64)
        r0, r1 = rows if rows is not None else (0, self.ctx.params.data_height)
        self.ctx.check(lib().sb_icp_jacobian(self.ctx.h, self.current.h, self.last.h, _dp(pc), self.iteration_,
                                             self.max_distance, self.max_angle, r0, r1, _dp(self.out48),
                                             self.raw32.ctypes.data_as(C.POINTER(C.c_int64))), "icp_jacobian")
        o = self.out48
        return o[43], o[:36].reshape(6, 6).T.copy(), o[36:42].copy()

    def increment(self, delta):
        T = np.zeros(16)
        d = np.ascontiguousarray(delta, np.float64)
        lib().sb_se3_exp(_dp(d), _dp(T))
        self.pose_ = from_colmajor(T) @ self.pose_
        self.iteration_ += 1

    def pose(self):
        return self.pose_

    def valid(self):
        return int(self.out48[42])

    def outlier(self):
        return int(self.out48[44])

    def inlier(self):
        return int(self.out48[42]) - int(self.out48[44])

    def invalid(self):
        return int(self.out48[46])

    def inlier_residual(self):
        return float(np.float32(self.out48[45]))


class LieGaussNewton:
    """core/LieGaussNewton.h:25-77. minimize() runs the whole loop on the device (sb_icp_minimize)."""

    def __init__(self, ctx):
        self.ctx = ctx
        p = ctx.params
        self.maxIter, self.epsilon, self.delta = p.max_iterations, p.stopping_threshold, p.delta
        self.Tk_ = np.eye(4)
        self.k_ = 0
        self.history_ = []
        self.out48 = np.zeros(48)

    def minimize(self, F, T0):
        T0c = colmajor(T0, np.float64)
        pose = np.zeros(16); out48 = np.zeros(48); it = C.c_int(0); hl = C.c_int(0)
        bounded = 1 <= self.maxIter <= 256   # a history buffer is only accepted with an explicit iteration limit
        hist = np.zeros((self.maxIter + 1) * 16 if bounded else 16)
        self.ctx.check(lib().sb_icp_minimize(self.ctx.h, F.current.h, F.last.h, _dp(T0c), self.maxIter, self.epsilon,
                                             self.delta, F.max_distance, F.max_angle, _dp(pose), _dp(out48),
                                             C.byref(it), _dp(hist) if bounded else None, C.byref(hl)), "icp_minimize")
        if not bounded:
            hl.value = 0
        self.Tk_ = from_colmajor(pose)
        self.k_ = it.value
        self.out48 = out48
        self.history_ = [from_colmajor(hist[16 * i:16 * i + 16]) for i in range(hl.value)]
        F.pose_ = self.Tk_.copy()
        F.out48 = out48
        return 0

    def minimize_host(self, F, T0):
        """The same loop driven from the host through jacobianProducts (the reference's call pattern)."""
        F.initialize(T0)
        last_error = float(np.finfo(np.float32).max)
        self.history_ = []
        k = 0
        while True:
            self.history_.append(F.pose().copy())
            if self.maxIter > 0 and k >= self.maxIter:
                break
            F.jacobianProducts()
            pose = colmajor(F.pose_, np.float64); dx = np.zeros(6)
            res = lib().sb_gn_step(_dp(F.out48), last_error, self.epsilon, self.delta, _dp(pose), _dp(dx))
            F.pose_ = from_colmajor(pose)
            F.iteration_ += 1
            last_error = F.out48[43]
            if res == 0:
                break
            k += 1
        self.Tk_, self.k_ = F.pose_.copy(), k
        return 0

    def pose(self):
        return self.Tk_

    def iterationCount(self):
        return self.k_

    def history(self):
        return self.history_


class SurfelMap:
    """core/SurfelMap.h:36-78"""

    def __init__(self, ctx):
        self.ctx = ctx

    def update(self, pose, frame):
        pc = colmajor(pose, np.float32)
        self.ctx.check(lib().sb_map_update(self.ctx.h, _fp(pc), frame.h), "map_update")

    def render(self, pose_old, pose_new, frame, confidence_threshold):
        po, pn = colmajor(pose_old, np.float32), colmajor(pose_new, np.float32)
        self.ctx.check(lib().sb_map_render(self.ctx.h, _fp(po), _fp(pn), confidence_threshold, frame.h), "map_render")

    def render_active(self, pose, confidence_threshold):
        pc = colmajor(pose, np.float32)
        self.ctx.check(lib().sb_map_render_active(self.ctx.h, _fp(pc), confidence_threshold), "render_active")

    def render_inactive(self, pose, confidence_threshold):
        pc = colmajor(pose, np.float32)
        self.ctx.check(lib().sb_map_render_inactive(self.ctx.h, _fp(pc), confidence_threshold), "render_inactive")

    def render_composed(self, pose_old, pose_new, confidence_threshold):
        po, pn = colmajor(pose_old, np.float32), colmajor(pose_new, np.float32)
        self.ctx.check(lib().sb_map_render_composed(self.ctx.h, _fp(po), _fp(pn), confidence_threshold), "render_composed")

    def _frame(self, which):
        h = C.c_void_p()
        self.ctx.check(lib().sb_map_frame(self.ctx.h, which, C.byref(h)), "map_frame")
        return Frame(self.ctx, handle=h.value)

    def oldMapFrame(self):
        return self._frame(0)

    def newMapFrame(self):
        return self._frame(1)

    def composedFrame(self):
        return self._frame(2)

    def size(self):
        n = C.c_uint32()
        lib().sb_map_size(self.ctx.h, C.byref(n))
        return n.value

    def timestamp(self):
        n = C.c_uint32()
        lib().sb_map_timestamp(self.ctx.h, C.byref(n))
        return n.value

    def getAllSurfels(self):
        n = self.size()
        a = np.zeros(max(n, 1), SURFEL_DTYPE)
        k = C.c_uint32()
        self.ctx.check(lib().sb_map_download(self.ctx.h, _vp(a), n, C.byref(k)), "map_download")
        return a[:k.value]

    def upload(self, surfels, timestamp):
        a = np.ascontiguousarray(surfels, SURFEL_DTYPE)
        self.ctx.check(lib().sb_map_upload(self.ctx.h, _vp(a), a.shape[0], timestamp), "map_upload")

    def set_pose(self, t, pose):
        pc = colmajor(pose, np.float32)
        self.ctx.check(lib().sb_map_set_pose(self.ctx.h, t, _fp(pc)), "map_set_pose")

    def updatePoses(self, poses):
        a = np.ascontiguousarray(np.stack([colmajor(p, np.float32) for p in poses]), np.float32)
        self.ctx.check(lib().sb_map_update_poses(self.ctx.h, _fp(a), len(poses)), "update_poses")

    def update_debug(self):
        H, W = self.ctx.params.data_height, self.ctx.params.data_width
        idx = np.zeros((H, W), np.uint32); rad = np.zeros((H, W, 4), np.float32); integ = np.zeros((H, W), np.uint8)
        nu, nn = C.c_uint32(), C.c_uint32()
        self.ctx.check(lib().sb_map_update_debug(self.ctx.h, _vp(idx), _vp(rad), _vp(integ), C.byref(nu), C.byref(nn)),
                       "update_debug")
        return idx, rad, integ, nu.value, nn.value

    def submap_origin(self):
        i, j, p = C.c_int32(), C.c_int32(), C.c_uint32()
        lib().sb_map_submap_origin(self.ctx.h, C.byref(i), C.byref(j), C.byref(p))
        return i.value, j.value, p.value

    def setTileCache(self, pool_surfels, host_surfels=None):
        self.ctx.set_tile_cache(pool_surfels, host_surfels)

    def tile_cache_info(self):
        return self.ctx.tile_cache_info()

    def pose_table_info(self):
        return self.ctx.pose_table_info()

    def reset(self):
        self.ctx.check(lib().sb_reset(self.ctx.h), "reset")


class SurfelMapping:
    """core/SurfelMapping.h:33-109. Loop-closure detection / verification (checkLoopClosure) is off unless
    enableLoopClosure() is called ("close-loops" in the reference's parameters); the pose-graph optimisation stays with
    the host application (gtsam is out of scope): see getLoopInfo() / getLoopEdges() / setCurrentPose()."""

    def __init__(self, params, device=0):
        self.ctx = Context(params, device)
        self.map_ = SurfelMap(self.ctx)

    def enableLoopClosure(self, enabled=True, **kw):
        """kw: search_distance, min_trajectory_distance, min_verifications, residual_threshold, outlier_threshold,
        valid_threshold (defaults: config/default.xml:70-76)"""
        lp = LoopParams()
        lib().sb_default_loop_params(C.byref(lp))
        for k, v in kw.items():
            if not hasattr(lp, k):
                raise KeyError(k)
            setattr(lp, k, v)
        self.ctx.check(lib().sb_set_loop_closure(self.ctx.h, 1 if enabled else 0, C.byref(lp)), "set_loop_closure")

    def getLoopInfo(self):
        li = LoopInfo()
        self.ctx.check(lib().sb_get_loop_info(self.ctx.h, C.byref(li)), "get_loop_info")
        d = {n: getattr(li, n) for n, _ in LoopInfo._fields_ if n != "current_pose_old"}
        d["valid_ratio"] = np.float32(d["valid_ratio"]); d["outlier_ratio"] = np.float32(d["outlier_ratio"])
        d["rel_error"] = np.float32(d["rel_error"])
        d["current_pose_old"] = from_colmajor(np.array(li.current_pose_old))
        return d

    def getLoopEdges(self):
        n = C.c_uint32(0)
        self.ctx.check(lib().sb_get_loop_edges(self.ctx.h, None, 0, C.byref(n)), "get_loop_edges")
        arr = (LoopEdge * max(n.value, 1))()
        self.ctx.check(lib().sb_get_loop_edges(self.ctx.h, arr, n.value, C.byref(n)), "get_loop_edges")
        return [(arr[i].from_, arr[i].to, from_colmajor(np.array(arr[i].rel_pose))) for i in range(n.value)]

    def integrateLoopClosures(self, poses=None):
        """SurfelMapping::integrateLoopClosures (SurfelMapping.cpp:212-258) before the next processScan: `poses` = the
        optimised 4x4 poses of scans 0..n-1 (None: the graph's own); returns the number of poses written, 0 if no
        optimisation request was pending"""
        n = C.c_uint32(0)
        if poses is None:
            self.ctx.check(lib().sb_integrate_loop_closures(self.ctx.h, None, 0, C.byref(n)), "integrate_loop_closures")
        else:
            a = np.ascontiguousarray([colmajor(P, np.float64) for P in poses], np.float64)
            self.ctx.check(lib().sb_integrate_loop_closures(self.ctx.h, _dp(a), a.shape[0], C.byref(n)),
                           "integrate_loop_closures")
        return int(n.value)

    def setCurrentPose(self, pose):
        """SurfelMapping::setCurrentPose (core/SurfelMapping.h:66)"""
        self.ctx.check(lib().sb_set_current_pose(self.ctx.h, _dp(colmajor(pose, np.float64))), "set_current_pose")

    def processScan(self, points, labels=None, probs=None, on_device=False, times=None):
        """times: per-point sweep times for deskewing mode 1 (setDeskew); with on_device a device pointer (int)"""
        if on_device:  # raw device pointers (int) + count: (ptr_pts, ptr_labels, ptr_probs, n)
            pp, pl, pq, n = points
            tp = C.c_void_p(times) if times else None
            rc = lib().sb_process_scan_timed(self.ctx.h, C.c_void_p(pp), C.c_void_p(pl) if pl else None,
                                             C.c_void_p(pq) if pq else None, tp, n, 1)
        else:
            pts = np.ascontiguousarray(points, np.float32)
            lab = None if labels is None else np.ascontiguousarray(labels, np.float32)
            prb = None if probs is None else np.ascontiguousarray(probs, np.float32)
            tms = None if times is None else np.ascontiguousarray(times, np.float32)
            rc = lib().sb_process_scan_timed(self.ctx.h, _vp(pts), _vp(lab), _vp(prb), _vp(tms), pts.shape[0], 0)
        self.ctx.check(rc, "process_scan")

    def setDeskew(self, mode="off", ref_time=0.5, start_azimuth=np.pi, clockwise=True):
        """Per-point deskewing of every scan with the motion of the previous increment (sb_set_deskew): mode "off",
        "times" (processScan(..., times=...)) or "azimuth" (sweep time from each point's azimuth)"""
        self.ctx.set_deskew(mode, ref_time, start_azimuth, clockwise)

    def getDeskew(self):
        return self.ctx.get_deskew()

    def process_scan_raw(self, ptr_pts, ptr_labels, ptr_probs, n, on_device):
        rc = lib().sb_process_scan(self.ctx.h, C.c_void_p(ptr_pts), C.c_void_p(ptr_labels) if ptr_labels else None,
                                   C.c_void_p(ptr_probs) if ptr_probs else None, n, 1 if on_device else 0)
        self.ctx.check(rc, "process_scan")

    def prefetch_scan_raw(self, ptr_pts, ptr_labels, ptr_probs, n):
        """stage the NEXT scan's (pinned) host buffers on the copy stream; process_scan_raw(..., on_device=False) with
        the same pointers then skips its own copy (sb_prefetch_scan)"""
        rc = lib().sb_prefetch_scan(self.ctx.h, C.c_void_p(ptr_pts), C.c_void_p(ptr_labels) if ptr_labels else None,
                                    C.c_void_p(ptr_probs) if ptr_probs else None, n)
        self.ctx.check(rc, "prefetch_scan")

    def setPointLabels(self, on=True):
        """Per-point label records of every following scan (sb_set_point_labels; DESIGN.md section 13)"""
        self.ctx.check(lib().sb_set_point_labels(self.ctx.h, 1 if on else 0), "set_point_labels")

    def getPointLabels(self, out=None):
        """The records of the last scan, one per input point in input order: a numpy structured array of
        POINT_LABEL_DTYPE (the fields of sb_point_label). out: an int device pointer to n * 32 bytes to fill instead
        (device-to-device copy); then returns n."""
        n = C.c_uint32(0)
        rc = lib().sb_get_point_labels(self.ctx.h, None, 0, C.byref(n), 0)
        if rc != SB_OK and not (rc == SB_ERR_INVALID and n.value > 0):
            self.ctx.check(rc, "get_point_labels")
        if out is not None:
            self.ctx.check(lib().sb_get_point_labels(self.ctx.h, C.c_void_p(out), n.value, C.byref(n), 1),
                           "get_point_labels")
            return int(n.value)
        a = np.zeros(n.value, POINT_LABEL_DTYPE)
        self.ctx.check(lib().sb_get_point_labels(self.ctx.h, _vp(a) if a.size else None, n.value, C.byref(n), 0),
                       "get_point_labels")
        return a

    def getCurrentPose(self):
        a = np.zeros(16)
        lib().sb_get_pose(self.ctx.h, _dp(a))
        return from_colmajor(a)

    def getLastPose(self):
        a = np.zeros(16)
        lib().sb_get_last_pose(self.ctx.h, _dp(a))
        return from_colmajor(a)

    def timestamp(self):
        t = C.c_uint32()
        lib().sb_timestamp(self.ctx.h, C.byref(t))
        return t.value

    def getMap(self):
        return self.map_

    def _frame(self, which):
        h = C.c_void_p()
        self.ctx.check(lib().sb_slam_frame(self.ctx.h, which, C.byref(h)), "slam_frame")
        return Frame(self.ctx, handle=h.value)

    def getCurrentFrame(self):
        return self._frame(0)

    def getLastFrame(self):
        return self._frame(1)

    def getCurrentModelFrame(self):
        return self._frame(2)

    def getLastModelFrame(self):
        return self._frame(3)

    def setTileCache(self, pool_surfels, host_surfels=None):
        """Managed submap tile cache: see Context.set_tile_cache"""
        self.ctx.set_tile_cache(pool_surfels, host_surfels)

    def tile_cache_info(self):
        return self.ctx.tile_cache_info()

    def pose_table_info(self):
        return self.ctx.pose_table_info()

    def getStatistics(self):
        a = np.zeros(16)
        lib().sb_get_statistics(self.ctx.h, _dp(a))
        return {"num_iterations": a[0], "F": a[1], "inlier": a[2], "outlier": a[3], "invalid": a[4],
                "inlier_residual": a[5], "track_loss": a[6], "surfels": a[7], "preprocessing-time": a[8],
                "icp-time": a[9], "mapping-time": a[10], "complete-time": a[11]}

    def reset(self):
        self.ctx.check(lib().sb_reset(self.ctx.h), "reset")

    def save_state(self):
        """The whole state of the mapping session as bytes (sb_state_save): loading it into a context of the same image
        size and continuing gives the bits of an uninterrupted run. Scans staged by prefetch_scan_raw are dropped."""
        n = C.c_uint64(0)
        self.ctx.check(lib().sb_state_size(self.ctx.h, C.byref(n)), "state_size")
        buf = np.empty(n.value, np.uint8)
        w = C.c_uint64(0)
        self.ctx.check(lib().sb_state_save(self.ctx.h, _vp(buf), n.value, C.byref(w)), "state_save")
        return buf[:w.value].tobytes()

    def load_state(self, blob):
        """Restores a save_state() checkpoint, its parameters included (sb_state_load). Raises SumaError on a blob of
        another format, image size or a corrupted one (after which the context is reset)."""
        a = np.frombuffer(blob, np.uint8)
        self.ctx.check(lib().sb_state_load(self.ctx.h, _vp(a) if a.size else None, a.size), "state_load")
        self.ctx.params = self.ctx.get_params()

    def save_state_file(self, path):
        data = self.save_state()
        with open(path, "wb") as f:
            f.write(data)
        return len(data)

    def load_state_file(self, path):
        with open(path, "rb") as f:
            self.load_state(f.read())
