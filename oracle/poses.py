"""TEST INFRASTRUCTURE: the CPU oracle with a pose table of any size (DESIGN.md section 12).

The oracle restates the reference, whose pose table has 10 000 entries (orc_map.c ORC_MAX_POSES, SurfelMap.h:205). The
library grows its table past that; this module builds a second copy of the oracle from the same, unchanged sources in
which that size is a run-time value (orc_set_pose_cap), so that runs past 10 000 scans can be compared bit for bit. For
input whose surfels all refer to entries below the table's size, a table of any such size gives the same results: the
size only decides where the lookup clamps, and the unwritten entries are identity in both. The copy is compiled with the
oracle's flags into a temporary directory keyed by its sources (the repository tree is not written) and linked
-Bsymbolic, so that it shares nothing with liborc.so loaded in the same process.

Use: `with poses.oracle(cap):` -- inside it, oracle.Map / oracle.Slam created there run on the copy with a table of
`cap` entries. Only tests/ may import this module; the product never does.
"""
import contextlib
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_C = ("orc_core.c", "orc_slam.c")
_ALL = _C + ("orc_map.c", "orc_loop.cpp", "orc.h", "orc_internal.h", "orc_math.h", "Makefile")
# the flags of oracle/Makefile that the bit parity with the CUDA path rests on
CFLAGS = ["-O2", "-fPIC", "-std=c11", "-D_GNU_SOURCE", "-ffp-contract=off", "-fno-fast-math", "-w"]
CXXFLAGS = ["-O2", "-fPIC", "-std=c++14", "-ffp-contract=off", "-fno-fast-math", "-w"]
_FIXED = "#define ORC_MAX_POSES 10000u            /* SurfelMap.h:205 */"
_RUNTIME = ("uint32_t orc_pose_cap = 10000u;\n"
            "void orc_set_pose_cap(uint32_t n) { orc_pose_cap = n; }\n"
            "#define ORC_MAX_POSES orc_pose_cap")
_lib = None


def _omp_cc():
    """the first C compiler that links OpenMP, as oracle/Makefile picks it (results do not depend on the thread count)"""
    for cc in (os.environ.get("CC", "gcc"), "/usr/bin/gcc", "gcc"):
        try:
            r = subprocess.run([cc, "-fopenmp", "-x", "c", "-", "-o", os.devnull], input=b"int main(void){return 0;}",
                               capture_output=True)
        except OSError:
            continue
        if r.returncode == 0:
            return cc, ["-fopenmp"]
    return os.environ.get("CC", "gcc"), []


def build():
    src = open(os.path.join(_HERE, "orc_map.c")).read()
    if src.count(_FIXED) != 1:
        raise RuntimeError("oracle/orc_map.c no longer declares the pose table's size as expected")
    h = hashlib.sha256()
    for f in _ALL + ("../include/suma_b200_loop.hpp",):
        with open(os.path.join(_HERE, f), "rb") as fh:
            h.update(fh.read())
    h.update(open(__file__, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "suma_b200_orc_poses_%d" % os.getuid(), h.hexdigest()[:16])
    out = os.path.join(d, "liborc_poses.so")
    if os.path.exists(out):
        return out
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "orc_map_poses.c"), "w") as f:
        f.write(src.replace(_FIXED, _RUNTIME))
    cc, omp = _omp_cc()
    cxx = os.environ.get("CXX", "g++")
    inc = ["-I", _HERE]
    objs = []
    for s in [os.path.join(_HERE, c) for c in _C] + [os.path.join(d, "orc_map_poses.c")]:
        o = os.path.join(d, os.path.basename(s).replace(".c", ".o"))
        subprocess.check_call([cc] + CFLAGS + omp + inc + ["-c", s, "-o", o])
        objs.append(o)
    o = os.path.join(d, "orc_loop.o")
    subprocess.check_call([cxx] + CXXFLAGS + inc + ["-c", os.path.join(_HERE, "orc_loop.cpp"), "-o", o])
    objs.append(o)
    tmp = "%s.%d.tmp" % (out, os.getpid())
    subprocess.check_call([cc] + omp + ["-shared", "-Wl,-Bsymbolic", "-o", tmp] + objs + ["-lstdc++", "-lm"])
    os.replace(tmp, out)
    return out


def lib():
    """the copy, with the ctypes signatures oracle.lib() gives liborc.so"""
    global _lib
    if _lib is None:
        saved_build, saved_lib = O.build, O._lib
        try:
            O.build, O._lib = build, None
            _lib = O.lib()
        finally:
            O.build, O._lib = saved_build, saved_lib
        _lib.orc_set_pose_cap.argtypes = [C.c_uint32]
        _lib.orc_set_pose_cap.restype = None
    return _lib


@contextlib.contextmanager
def oracle(cap):
    """oracle.Map / oracle.Slam created and used inside run on the copy with a pose table of `cap` entries (set before
    they are created). Drop them inside the block; one that liborc.so destroys later is still freed right (the two
    copies share the struct layouts and the C heap, and destruction does not depend on the table's size)."""
    L = lib()
    L.orc_set_pose_cap(int(cap))
    saved = O._lib
    O._lib = L
    try:
        yield
    finally:
        O._lib = saved
