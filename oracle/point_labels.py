"""TEST INFRASTRUCTURE: ctypes binding of the CPU oracle's per-point label records (oracle/orc_point_labels.c;
DESIGN.md section 13).

orc_point_labels.c computes the records from the oracle's own projection, frames and map update. Like oracle/deskew.py
it is compiled into a library of its own, linked against liborc.so and the deskewing library, in a temporary directory
keyed by its sources (the repository tree is not written). Only tests/ may import this module; the product never does.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import deskew as OD
from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SOURCES = [os.path.join(_HERE, f) for f in ("orc_point_labels.c", "orc_deskew.h", "orc.h", "orc_internal.h",
                                             "orc_math.h")]
_lib = None

# the record, field for field as sb_point_label (include/suma_b200.h)
DTYPE = np.dtype([("pixel", "<i4"), ("flags", "<u4"), ("frame_label", "<u4"), ("frame_prob", "<f4"),
                  ("map_pixel", "<i4"), ("map_label", "<u4"), ("map_prob", "<f4"), ("map_range", "<f4")])
WON, VERTEX, INTEGRATED, MAP = 1, 2, 4, 8


def build():
    orc = os.path.abspath(O.build())
    desk = os.path.abspath(OD.build())
    h = hashlib.sha256()
    for f in _SOURCES + [orc, desk]:
        with open(f, "rb") as fh:
            h.update(fh.read())
    d = os.path.join(tempfile.gettempdir(), "suma_b200_orc_point_labels_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    out = os.path.join(d, "liborc_point_labels_%s.so" % h.hexdigest()[:16])
    if not os.path.exists(out):
        tmp = "%s.%d.tmp" % (out, os.getpid())
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc] + OD.CFLAGS + ["-shared", "-o", tmp, os.path.join(_HERE, "orc_point_labels.c"), desk,
                                                  orc, "-Wl,-rpath," + os.path.dirname(desk),
                                                  "-Wl,-rpath," + os.path.dirname(orc), "-lm"])
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        OD.lib()  # liborc.so and the deskewing library first: this one shares their loaded instances
        _lib = C.CDLL(build())
        _lib.orc_slam_point_labels.restype = C.c_int
        _lib.orc_slam_process_scan_labels.restype = C.c_int
    return _lib


class Slam(OD.Slam):
    """the oracle's SurfelMapping (with deskewing and loop closure as OD.Slam / O.Slam) that keeps the records of its last
    scan in `self.records`"""

    def __init__(self, p):
        super().__init__(p)
        self.records = None

    def process_scan(self, pts, labels=None, probs=None, times=None):
        pts = O._f32(pts); labels = O._f32(labels); probs = O._f32(probs); times = O._f32(times)
        mode, ref, a0, cw = self.deskew
        n = pts.shape[0]
        rec = np.zeros(n, DTYPE)
        rc = lib().orc_slam_process_scan_labels(self.h, O._p(pts), O._p(labels), O._p(probs), O._p(times), C.c_uint32(n),
                                                C.c_int32(mode), C.c_float(ref), C.c_float(a0), C.c_int32(cw),
                                                rec.ctypes.data_as(C.c_void_p))
        if rc != 0:
            raise RuntimeError("orc_slam_point_labels: the view of orc_slam does not match liborc.so")
        self.records = rec
