"""Per-point label records (DESIGN.md section 13) without a GPU:

* the oracle's records (oracle/point_labels.py) against tests/preprocess_reference.py, the exact model of the projection
  and depth test, on the designed scans of tests/preprocess_cases.py and on points the projection refuses (NaN, inf,
  the origin), with the Q1 pairing on and off, movable points before and after timestamp 10, a model image of another
  size and field of view, and scans of 0 and 1 points;
* the sb_point_label layout in Python and in C;
* run_kitti --write-labels with an injected engine: files, names, bytes, the id rule, the refusal without --semantic,
  and a resumed run writing the remaining scans only, byte-identical to an uninterrupted run.
The CUDA path against the oracle: tests/test_gpu_point_labels.py."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from oracle import point_labels as OPL
from semantic_suma_b200 import api, kitti, run_kitti
import preprocess_cases as U
import preprocess_reference as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def model_image(W, H):
    """a model image of another size and field of view than the data image"""
    return dict(model_width=W + 7, model_height=H + 5, model_fov_up=5.0, model_fov_down=-27.0)


def model_pixel(p, v, W, H, up, down):
    """the model pixel of v: (index or -1, False when v lies within PIXEL_MARGIN of a pixel edge there)"""
    q = O.default_params(data_width=W, data_height=H, data_fov_up=up, data_fov_down=down)
    px, py = M.pixel_coords(q, v)
    if px is None:
        return -1, True
    x, y = float(v[0]), float(v[1])
    seam = x < 0.0 and abs(y) <= abs(x) * M.SEAM_RATIO
    ok = abs(py - round(py)) >= M.PIXEL_MARGIN and (seam or abs(px - round(px)) >= M.PIXEL_MARGIN)
    fx, fy = math.floor(px), math.floor(py)
    if not (0 <= fx < W and 0 <= fy < H):
        return -1, ok
    return fy * W + fx, ok


def expected(p, pts, lab, prb, timestamp):
    """the model's records, pixel through frame fields, and the model pixel of every point (with its margin flag)"""
    n = len(pts)
    m = M.preprocess(p, pts, lab, prb, timestamp)
    H, W = p.data_height, p.data_width
    pixel = np.full(n, -1, np.int32)
    flags = np.zeros(n, np.uint32)
    key = {}
    for i in range(n):
        v = M.v3(*pts[i, :3])
        pix, _ = M.pixel_of(p, v)
        if pix is None:
            continue
        d24, _ = M.point_d24(p, v)
        if d24 is None:
            continue
        pixel[i] = pix[1] * W + pix[0]
        key[i] = d24
    best = {}
    for i in sorted(key):  # GL_LESS in buffer order
        if pixel[i] not in best or key[i] < key[best[pixel[i]]]:
            best[pixel[i]] = i
    V, S = m["vertex"].reshape(-1, 4), m["semantic"].reshape(-1, 4)
    frame_label = np.zeros(n, np.uint32)
    frame_prob = np.zeros(n, f32)
    for i in key:
        if best[pixel[i]] == i:
            flags[i] |= OPL.WON
        if V[pixel[i], 3] > 0:
            flags[i] |= OPL.VERTEX
        frame_label[i] = int(np.rint(S[pixel[i], 0] * f32(255.0)))
        frame_prob[i] = S[pixel[i], 3]
    mp = [model_pixel(p, M.v3(*pts[i, :3]), p.model_width, p.model_height, p.model_fov_up, p.model_fov_down)
          if pixel[i] >= 0 else (-1, True) for i in range(n)]
    return pixel, flags, frame_label, frame_prob, mp


def oracle_records(p, pts, lab, prb, timestamp):
    """the records of a scan at `timestamp` on a fresh oracle slam (empty scans before it)"""
    s = OPL.Slam(p)
    empty = np.zeros((0, 4), f32)
    for _ in range(timestamp):
        s.process_scan(empty, np.zeros(0, f32), np.zeros(0, f32))
    s.process_scan(pts, lab, prb)
    return s.records


def check(p, pts, lab, prb, timestamp, what):
    r = oracle_records(p, pts, lab, prb, timestamp)
    pixel, flags, frame_label, frame_prob, mp = expected(p, pts, lab, prb, timestamp)
    assert r.shape[0] == len(pts)
    np.testing.assert_array_equal(r["pixel"], pixel, err_msg=what + " pixel")
    np.testing.assert_array_equal(r["flags"] & (OPL.WON | OPL.VERTEX), flags, err_msg=what + " flags")
    assert not (r["flags"] & OPL.INTEGRATED).any(), what + ": nothing to integrate into on an empty map"
    np.testing.assert_array_equal(r["frame_label"], frame_label, err_msg=what + " frame_label")
    assert r["frame_prob"].tobytes() == frame_prob.tobytes(), what + " frame_prob"
    ok = np.array([m[1] for m in mp], bool)
    np.testing.assert_array_equal(r["map_pixel"][ok], np.array([m[0] for m in mp], np.int32)[ok],
                                  err_msg=what + " map_pixel")
    none = r["pixel"] < 0
    assert (r["map_pixel"][none] == -1).all() and not r["flags"][none].any() and not r["frame_label"][none].any()
    mapped = (r["flags"] & OPL.MAP) != 0
    assert (r["map_range"][mapped] > 0).all() and not r["map_range"][~mapped].any() and not r["map_label"][~mapped].any()
    return r


@pytest.mark.parametrize("shape", U.SHAPES[:2], ids=["%dx%d" % s for s in U.SHAPES[:2]])
@pytest.mark.parametrize("name", U.case_ids())
def test_oracle_records_equal_the_model_on_designed_scans(name, shape):
    c = U.get(name, *shape)
    pts, lab, prb = c.arrays()
    ts = 0 if c.timestamp < 10 else 10
    for kw in (dict(), model_image(c.W, c.H)):
        d = dict(data_width=c.W, data_height=c.H, model_width=c.W, model_height=c.H)
        d.update(c.kw)
        d.update(kw)
        p = O.default_params(**d)
        check(p, pts, lab, prb, ts, "%s %s" % (name, kw))


def test_the_designed_scans_reach_every_point_rule():
    tags = set()
    for name in U.case_ids():
        c = U.get(name, *U.SHAPES[0])
        pts, lab, prb = c.arrays()
        for t in M.preprocess(c.params(O), pts, lab, prb, c.timestamp)["point_tags"]:
            tags |= t
    for t in ("seam:col0", "seam:clipped", "point:clipped", "point:z_below", "point:z_above", "point:won_tie",
              "point:lost_tie", "point:movable_removed", "point:movable_kept"):
        assert t in tags, t


def special_scan(H=40, W=96):
    pts = [U.point(H, W, 10, 20, 8.0), U.point(H, W, 10, 20, 8.0), U.point(H, W, 5, 70, 30.0)]
    pts += [(np.nan, 1.0, 0.0), (np.inf, 0.0, 0.0), (1.0, -np.inf, 0.0), (0.0, 0.0, 0.0), (0.0, 0.0, np.nan)]
    pts += [U.point(H, W, H + 2, 3, 10.0), U.point(H, W, 3, 3, 1.0), U.point(H, W, 3, 4, 500.0)]
    a = np.ones((len(pts), 4), f32)
    a[:, :3] = np.array([tuple(q[:3]) for q in pts], f32)
    lab = np.array([10, 40, 50, 40, 40, 40, 40, 40, 40, 40, 40], f32)[:len(pts)]
    prb = np.linspace(0.5, 0.9, len(pts)).astype(f32)
    return a, lab, prb


@pytest.mark.parametrize("quirk", [0, 1], ids=["q1_off", "q1_on"])
@pytest.mark.parametrize("timestamp", [0, 10], ids=["t0", "t10"])
def test_points_the_projection_refuses_ties_movables_and_q1(quirk, timestamp):
    """NaN / inf / the origin / above the field of view / nearer than min_depth / beyond max_depth give pixel -1; two
    points on one beam at one depth: the lower index WON, the other keeps the pixel; a car (movable) winner before
    timestamp 10 writes no vertex; with Q1 on a pixel's label is the one four points further on"""
    pts, lab, prb = special_scan()
    p = O.default_params(data_width=96, data_height=40, model_width=96, model_height=40, label_offset_quirk=quirk)
    r = check(p, pts, lab, prb, timestamp, "special")
    assert (r["pixel"][3:] == -1).all()
    assert r["pixel"][0] == r["pixel"][1] >= 0 and r["flags"][0] & OPL.WON and not r["flags"][1] & OPL.WON
    if quirk == 0:
        assert bool(r["flags"][0] & OPL.VERTEX) == (timestamp >= 10)  # label 10: a car
        assert r["frame_label"][2] == 50
    else:
        assert r["flags"][0] & OPL.VERTEX and r["frame_label"][0] == 40  # paired with labels[4]


def test_scans_of_zero_and_one_point():
    p = O.default_params(data_width=96, data_height=40, model_width=96, model_height=40, label_offset_quirk=0)
    assert check(p, np.zeros((0, 4), f32), np.zeros(0, f32), np.zeros(0, f32), 0, "n=0").shape == (0,)
    pts, lab, prb = special_scan()
    r = check(p, pts[2:3], lab[2:3], prb[2:3], 0, "n=1")
    assert r["flags"][0] & OPL.WON and r["frame_label"][0] == 50


# ---- the ABI ---------------------------------------------------------------------------------------------------------
OFFSETS = dict(pixel=0, flags=4, frame_label=8, frame_prob=12, map_pixel=16, map_label=20, map_prob=24, map_range=28)


def test_record_layout_in_python():
    assert C.sizeof(api.PointLabel) == 32 and api.POINT_LABEL_DTYPE.itemsize == 32
    for name, off in OFFSETS.items():
        assert getattr(api.PointLabel, name).offset == off
        assert api.POINT_LABEL_DTYPE.fields[name][1] == off
    assert api.POINT_LABEL_DTYPE == OPL.DTYPE
    assert (api.POINT_WON, api.POINT_VERTEX, api.POINT_INTEGRATED, api.POINT_MAP) == (1, 2, 4, 8)


def test_record_layout_in_c(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "suma_b200.h"\nint main(void) {\n'
                   '  printf("size %zu\\n", sizeof(sb_point_label));\n' +
                   "".join('  printf("%s %%zu\\n", offsetof(sb_point_label, %s));\n' % (k, k) for k in OFFSETS) +
                   '  printf("enum %d %d %d %d\\n", SB_POINT_WON, SB_POINT_VERTEX, SB_POINT_INTEGRATED, SB_POINT_MAP);\n'
                   "  return 0;\n}\n")
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), "-o", exe, str(src)])
    out = dict(l.split(" ", 1) for l in subprocess.check_output([exe], text=True).strip().splitlines())
    assert out["size"] == "32" and out["enum"] == "1 2 4 8"
    for name, off in OFFSETS.items():
        assert int(out[name]) == off


def test_the_library_exports_the_calls():
    L = api.lib()
    for name in ("sb_set_point_labels", "sb_get_point_labels"):
        assert name in api.EXPORTED_SYMBOLS
        getattr(L, name)


# ---- run_kitti --write-labels ----------------------------------------------------------------------------------------
class FakeEngine:
    """a pose chain and per-point records that depend on every earlier scan (as the map's labels do)"""

    def __init__(self, params):
        self.pose, self.memory, self.t, self.on, self.rec = np.eye(4), 0.0, 0, False, None

    def setPointLabels(self, on):
        self.on = on

    def processScan(self, pts, labels, probs):
        self.memory = 0.5 * self.memory + 1e-3 * float(np.asarray(pts)[:, 0].mean())
        self.pose = self.pose.copy()
        self.pose[0, 3] += self.memory
        self.t += 1
        if self.on:
            n = len(pts)
            r = np.zeros(n, api.POINT_LABEL_DTYPE)
            k = np.arange(n)
            r["flags"] = np.where((k + self.t) % 3 == 0, 0, api.POINT_MAP | api.POINT_WON)
            r["map_label"] = (np.asarray(labels).astype(np.int64) + self.t + int(1e6 * self.memory) % 7) % 300 + 0x10000
            r["map_label"][k % 5 == 0] = 252  # a moving-car id of SemanticKITTI
            self.rec = r

    def getPointLabels(self):
        if not self.on or self.rec is None:
            raise api.SumaError("get_point_labels: SB_ERR_STATE")
        return self.rec

    def getCurrentPose(self):
        return self.pose

    def timestamp(self):
        return self.t

    def save_state(self):
        return np.array([self.memory, self.t] + list(self.pose.reshape(-1))).tobytes()

    def load_state(self, blob):
        a = np.frombuffer(blob, np.float64)
        self.memory, self.t, self.pose, self.rec = float(a[0]), int(a[1]), a[2:].reshape(4, 4).copy(), None


@pytest.fixture
def seq(tmp_path):
    d = str(tmp_path / "seq")
    run_kitti.make_synthetic_sequence(d, 6, width=300, semantic=True)
    return d


def test_write_labels_files_names_bytes_and_ids(seq, tmp_path):
    out = str(tmp_path / "labels")
    eng = []

    def make(params):
        eng.append(FakeEngine(params))
        return eng[-1]

    assert run_kitti.main([seq, "--width", "300", "--semantic", "--write-labels", out], make_engine=make) == 0
    names = sorted(os.listdir(out))
    assert names == ["%06d.label" % i for i in range(6)]
    # the last file from the engine's last records: map_label in the low 16 bits where MAP is set, 0 elsewhere
    r = eng[0].rec
    raw = np.fromfile(os.path.join(out, names[-1]), np.uint32)
    assert raw.size == r.size == kitti.read_scan(run_kitti.list_scans(seq)[-1])[0].shape[0]
    want = np.where(r["flags"] & api.POINT_MAP, r["map_label"] & 0xFFFF, 0).astype(np.uint32)
    assert raw.tobytes() == want.tobytes()
    assert (raw >> 16 == 0).all() and (raw == 252).any() and (raw == 0).any()
    assert os.path.getsize(os.path.join(out, names[0])) == 4 * kitti.read_scan(run_kitti.list_scans(seq)[0])[0].shape[0]
    np.testing.assert_array_equal(run_kitti.map_label_ids(r), np.where(r["flags"] & 8, r["map_label"], 0))


def test_write_labels_needs_semantic(seq, tmp_path):
    with pytest.raises(SystemExit):
        run_kitti.main([seq, "--write-labels", str(tmp_path / "labels")], make_engine=FakeEngine)
    assert not os.path.exists(str(tmp_path / "labels"))


def test_a_resumed_run_writes_the_remaining_scans_only(seq, tmp_path):
    whole, part, state = str(tmp_path / "whole"), str(tmp_path / "part"), str(tmp_path / "state.bin")
    args = [seq, "--width", "300", "--semantic"]
    assert run_kitti.main(args + ["--write-labels", whole], make_engine=FakeEngine) == 0
    assert run_kitti.main(args + ["--max-scans", "4", "--save-state", state], make_engine=FakeEngine) == 0
    assert run_kitti.main(args + ["--resume", state, "--write-labels", part], make_engine=FakeEngine) == 0
    assert sorted(os.listdir(part)) == ["000004.label", "000005.label"]
    for name in os.listdir(part):
        assert open(os.path.join(part, name), "rb").read() == open(os.path.join(whole, name), "rb").read()
