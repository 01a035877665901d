"""TEST INFRASTRUCTURE: ctypes binding of the CPU oracle's per-point deskewing (oracle/orc_deskew.c; DESIGN.md section 11).

orc_deskew.c moves the points and hands them to the oracle's own preprocessing and processScan in liborc.so, which it
does not change: it is compiled into a library of its own, linked against liborc.so, in a temporary directory keyed by
its sources (the repository tree is not written). Only tests/ may import this module; the product never does.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SOURCES = [os.path.join(_HERE, f) for f in ("orc_deskew.c", "orc_deskew.h", "orc.h", "orc_internal.h", "orc_math.h")]
_SOURCES.append(os.path.join(_HERE, "..", "include", "suma_b200_deskew.h"))
# the flags of oracle/Makefile that the bit parity with the CUDA path rests on
CFLAGS = ["-O2", "-fPIC", "-std=c11", "-D_GNU_SOURCE", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra",
          "-Wno-unused-parameter"]
_lib = None


def build():
    orc = os.path.abspath(O.build())
    h = hashlib.sha256()
    for f in _SOURCES + [orc]:
        with open(f, "rb") as fh:
            h.update(fh.read())
    d = os.path.join(tempfile.gettempdir(), "suma_b200_orc_deskew_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    out = os.path.join(d, "liborc_deskew_%s.so" % h.hexdigest()[:16])
    if not os.path.exists(out):
        tmp = "%s.%d.tmp" % (out, os.getpid())
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc] + CFLAGS + ["-shared", "-o", tmp, os.path.join(_HERE, "orc_deskew.c"), orc,
                                               "-Wl,-rpath," + os.path.dirname(orc), "-lm"])
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        O.lib()  # liborc.so first: the deskewing library shares its loaded instance
        _lib = C.CDLL(build())
        _lib.orc_deskew_points.restype = C.c_int
        _lib.orc_preprocess_deskew.restype = None
        _lib.orc_slam_process_scan_timed.restype = None
    return _lib


def _motion(motion):
    return None if motion is None else O.colmajor(motion, np.float64)


def deskew_points(pts, times=None, mode=2, ref_time=0.5, start_azimuth=np.pi, clockwise=True, motion=None):
    """the points moved to the reference time by `motion` (4x4, the sweep's motion; None = identity): orc_deskew_points"""
    pts = O._f32(pts); times = O._f32(times)
    out = np.empty_like(pts)
    m = _motion(motion)
    lib().orc_deskew_points(O._p(pts), O._p(times), C.c_uint32(pts.shape[0]), C.c_int32(mode), C.c_float(ref_time),
                            C.c_float(start_azimuth), C.c_int32(int(bool(clockwise))), O._p(m, C.c_double), O._p(out))
    return out


def preprocess_deskew(p, pts, labels=None, probs=None, times=None, timestamp=100, mode=2, ref_time=0.5,
                      start_azimuth=np.pi, clockwise=True, motion=None):
    """orc_preprocess of the deskewed points: (vertex, normal, semantic) maps"""
    pts = O._f32(pts); labels = O._f32(labels); probs = O._f32(probs); times = O._f32(times)
    H, W = p.data_height, p.data_width
    v = np.empty((H, W, 4), np.float32); nm = np.empty_like(v); s = np.empty_like(v)
    m = _motion(motion)
    lib().orc_preprocess_deskew(C.byref(p), O._p(pts), O._p(labels), O._p(probs), O._p(times), C.c_uint32(pts.shape[0]),
                                C.c_uint32(timestamp), C.c_int32(mode), C.c_float(ref_time), C.c_float(start_azimuth),
                                C.c_int32(int(bool(clockwise))), O._p(m, C.c_double), O._p(v), O._p(nm), O._p(s))
    return v, nm, s


class Slam(O.Slam):
    """the oracle's SurfelMapping with deskewing: every scan is moved with the slam's own lastIncrement_ when it begins"""

    def __init__(self, p):
        super().__init__(p)
        self.deskew = (0, 0.5, float(np.pi), 1)

    def set_deskew(self, mode, ref_time=0.5, start_azimuth=np.pi, clockwise=True):
        """mode 0 off, 1 per-point times, 2 azimuth"""
        self.deskew = (int(mode), float(ref_time), float(start_azimuth), int(bool(clockwise)))

    def process_scan(self, pts, labels=None, probs=None, times=None):
        pts = O._f32(pts); labels = O._f32(labels); probs = O._f32(probs); times = O._f32(times)
        mode, ref, a0, cw = self.deskew
        lib().orc_slam_process_scan_timed(self.h, O._p(pts), O._p(labels), O._p(probs), O._p(times),
                                          C.c_uint32(pts.shape[0]), C.c_int32(mode), C.c_float(ref), C.c_float(a0),
                                          C.c_int32(cw))
