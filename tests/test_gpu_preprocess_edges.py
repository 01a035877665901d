"""The preprocessing pass K1-K3 (k_project_scatter, k_preprocess_tile) at its decisions, on the designed cases of
tests/preprocess_cases.py. Each case runs on the library, on the oracle and on tests/preprocess_reference.py, an exact
numpy model that shares no code with either: the library's vertex, normal and semantic maps must equal the oracle's bit
for bit, and both must equal the model. Every case also asserts the branches the model says it takes, and a last test
that every branch was reached.

Which k_preprocess_tile instance runs is not visible from here. The rule: an even data width makes the key image's row
pitch, (W + 6) * 8 bytes, a multiple of 16, so a tensor map can be encoded for it, and on a device with a TMA unit the
even-width shapes run k_preprocess_tile<true> (key tile staged by cp.async.bulk.tensor); odd widths, and the CPU
executor, run the plain-load instance <false>. SHAPES holds two of each.

Three paths only a chain of calls reaches:
  * key-image re-arming: the two key images alternate between scans, and each call re-arms its own tile of the other
    image, mirror pads included. The chains below leave every pixel that held a key in scan t empty in scans t + 1 and
    t + 2, with point counts that fall below the earlier indices: a key that was not re-armed would win its pixel with
    an index past the current scan's n;
  * movable classes through SurfelMapping.processScan: removed up to scan index 9, kept from 10;
  * the deskew instance k_project_scatter<true>: the designed cases with azimuth deskewing and identity motion.
"""
import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api
import preprocess_cases as U
import preprocess_reference as M
from helpers import assert_bits_equal
from test_gpu_shapes import _beam_centres

pytestmark = pytest.mark.gpu
IDS = ["%dx%d" % s for s in U.SHAPES]
_ctxs = {}


@pytest.fixture(scope="module", autouse=True)
def _close_contexts():
    yield
    for ctx, _, _ in _ctxs.values():
        ctx.close()
    _ctxs.clear()


def _operator(c):
    """one context per shape and parameter set, kept across the cases of this module and closed at its end: each case
    also runs on key images that earlier cases used. Re-arming itself is checked by the chain tests below, which
    start from a fresh context and do not depend on which cases ran before."""
    key = (c.H, c.W, tuple(sorted(c.kw.items())))
    if key not in _ctxs:
        ctx = api.Context(c.params(api))
        _ctxs[key] = (ctx, api.Frame(ctx, c.W, c.H), api.Preprocessing(ctx))
    return _ctxs[key]


def run_library(c, **kw):
    _, f, pre = _operator(c)
    pts, lab, prb = c.arrays()
    pre.process(pts, f, lab, prb, c.timestamp, **kw)
    return f.maps()


def model_of(c):
    pts, lab, prb = c.arrays()
    m = M.preprocess(c.params(O), pts, lab, prb, c.timestamp)
    U.check_tags(c, m)
    return m


def check(got, model, what):
    for a, nm in zip(got, ("vertex", "normal", "semantic")):
        assert_bits_equal(a, model[nm], "%s: %s map vs model" % (what, nm))


@pytest.mark.parametrize("shape", U.SHAPES, ids=IDS)
@pytest.mark.parametrize("name", U.case_ids())
def test_preprocess_case(name, shape):
    c = U.get(name, *shape)
    model = model_of(c)
    pts, lab, prb = c.arrays()
    o = O.preprocess(c.params(O), pts, lab, prb, c.timestamp)
    g = run_library(c)
    for a, b, nm in zip(g, o, ("vertex", "normal", "semantic")):
        assert_bits_equal(a, b, "%s: %s map vs oracle" % (name, nm))
    check(o, model, name + " (oracle)")
    check(g, model, name + " (CUDA)")


@pytest.mark.parametrize("shape", U.SHAPES, ids=IDS)
@pytest.mark.parametrize("name", U.case_ids())
def test_preprocess_case_through_the_deskew_instance(name, shape):
    """azimuth deskewing with identity motion moves no point: k_project_scatter<true> must give the same bits"""
    c = U.get(name, *shape)
    model = model_of(c)
    check(run_library(c, deskew=dict(mode="azimuth")), model, name + " (CUDA, deskew instance)")


def test_beam_centres_are_those_of_the_shapes_test():
    for H, W in U.SHAPES:
        d = _beam_centres(H, W)
        for r, x in ((0, 0), (H - 1, W - 1), (H // 2, W // 3)):
            assert np.allclose(U.direction(H, W, r + 0.5, x + 0.5), d[r, x], atol=1e-12)


def test_every_branch_was_reached():
    """the models of all designed cases (each checked against CUDA and the oracle above) reach every branch the model
    has (preprocess_reference.TAGS) but those preprocess_cases.UNREACHED lists with their reasons, per shape. At width 4
    the texels at x + 2 and x - 2 coincide and +x is searched first, so offset 2 in -x is never the one that fills
    there."""
    for H, W in U.SHAPES:
        got = set()
        for c in U.all_cases(H, W):
            got |= U.reached(model_of(c))
        want = U.BRANCHES - ({"fill:o2_-x"} if W == 4 else set())
        assert want <= got, "%dx%d: branches never reached: %s" % (H, W, sorted(want - got))


# ---- key-image re-arming -------------------------------------------------------------------------------------------
COUNTS = (257, 256, 255, 1, 0, 257, 1, 256, 0)


def _class_scan(H, W, cls, n, seed):
    """n points on the beam centres of the pixels with (x + y) % 3 == cls, several per pixel (later ones farther, so
    they lose), labels 40..47, near depths with steps so that normals, erosion and flood fill all take place"""
    pix = [(y, x) for y in range(H) for x in range(W) if (x + y) % 3 == cls]
    rng = np.random.default_rng(seed)
    pts, lab, prb = [], [], []
    for i in range(n):
        y, x = pix[i % len(pix)]
        rnd = i // len(pix)
        d = U.direction(H, W, y + 0.5, x + 0.5) * (6.0 + 0.02 * x + 0.03 * y + 0.5 * rnd + rng.uniform(0, 0.01))
        pts.append((*d.astype(np.float32), 1.0))
        lab.append(40.0 + (x // 3 + y // 2) % 8 * (rng.uniform() < 0.8))
        prb.append(rng.uniform(0.1, 0.9))
    return (np.array(pts, np.float32).reshape(-1, 4), np.array(lab, np.float32), np.array(prb, np.float32))


def _chain(H, W):
    return [(t, _class_scan(H, W, t % 3, n, t)) for t, n in enumerate(COUNTS)]


def _pparams(P, H, W):
    return P.default_params(data_width=W, model_width=W, data_height=H, model_height=H, label_offset_quirk=0)


@pytest.mark.parametrize("shape", U.SHAPES, ids=IDS)
def test_key_images_are_rearmed_between_operator_calls(shape):
    H, W = shape
    p = _pparams(O, H, W)
    ctx = api.Context(_pparams(api, H, W))
    f, pre = api.Frame(ctx, W, H), api.Preprocessing(ctx)
    for t, (pts, lab, prb) in _chain(H, W):
        pre.process(pts, f, lab, prb, 100)
        check(f.maps(), M.preprocess(p, pts, lab, prb, 100), "scan %d (n = %d)" % (t, len(pts)))
    ctx.close()


@pytest.mark.parametrize("shape", U.SHAPES, ids=IDS)
def test_key_images_index_keys_and_flags_are_rearmed_in_the_pipeline(shape):
    """the same chain through processScan: the pipeline instance of the tile pass also re-arms the index-map keys and
    the integrated flags and writes the radius map, which must equal the model's radius map of the scan"""
    H, W = shape
    p = _pparams(O, H, W)
    sl = api.SurfelMapping(_pparams(api, H, W))
    for t, (pts, lab, prb) in _chain(H, W):
        sl.processScan(pts, lab, prb)
        m = M.preprocess(p, pts, lab, prb, t)
        check(sl.getCurrentFrame().maps(), m, "processScan %d (n = %d)" % (t, len(pts)))
        assert_bits_equal(sl.getMap().update_debug()[1], m["radius"], "processScan %d radius map" % t)
    sl.ctx.close()


def test_movable_classes_through_the_pipeline():
    """11 processScan calls on a scan with a block of movable labels: the frame at scan index 9 drops those points,
    the frame at index 10 keeps them, each equal to the model"""
    H, W = U.SHAPES[0]
    c = U.tiles(H, W)
    pts, lab, prb = c.arrays()
    for i, q in enumerate(pts):
        pix = M.pixel_of(c.params(O), q[:3])[0]
        if pix and 10 <= pix[0] < 20 and 5 <= pix[1] < 12:
            lab[i] = M.MOVABLE[(pix[0] + pix[1]) % len(M.MOVABLE)]
    p = _pparams(O, H, W)
    sl = api.SurfelMapping(_pparams(api, H, W))
    for t in range(11):
        sl.processScan(pts, lab, prb)
        if t in (9, 10):
            m = M.preprocess(p, pts, lab, prb, t)
            tags = set().union(*m["point_tags"])
            assert ("point:movable_removed" if t == 9 else "point:movable_kept") in tags
            check(sl.getCurrentFrame().maps(), m, "processScan %d" % t)
    sl.ctx.close()
