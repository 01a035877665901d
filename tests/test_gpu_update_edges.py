"""The map update's per-surfel and per-pixel decisions at their thresholds (K6a-K6e: k_index_scatter, k_radius,
k_update_surfels<false>, k_gen_compact), on the designed cases of tests/update_cases.py. Each case runs on the library,
on the oracle and on tests/update_reference.py, an exact numpy model that shares no code with either: CUDA must equal
the oracle bit for bit (index map, radius map, integrated flags, counts, records and their order), and both must equal
the model -- bits for exact outputs, the model's stated tolerances for the outputs of acos / sin / exp / log. Every case
also asserts the branches the model says it takes, and a last test that every branch was reached.

Two paths only the per-scan pipeline takes are driven through SurfelMapping.processScan on scans whose points lie on
beam centres (the vertex map is the points' own bits): the radius map the tiled preprocessing pass writes in place of
k_radius, and the in-place instance k_update_surfels<true>. The pose there is the one Gauss-Newton finds, so the model
is applied to the frame and the pose the pipeline actually produced, and the designed thresholds are those that do not
depend on the pose: the radius map's clamps."""
import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api
import update_cases as U
import update_reference as M
from helpers import assert_bits_equal, surfel_fields_equal
from test_gpu_lazy_map import scan_modes
from test_gpu_shapes import _beam_centres

pytestmark = pytest.mark.gpu


def run_library(c):
    ctx = api.Context(c.params(api))
    m = api.SurfelMap(ctx)
    for t, T in c.poses.items():
        m.set_pose(t, T)
    m.upload(c.records(), U.TS)
    f = api.Frame(ctx, c.W, c.H)
    f.upload(c.frame())
    m.update(c.pose, f)
    out = m.update_debug() + (m.getAllSurfels(),)
    ctx.close()
    return out


def run_oracle(c):
    m = O.Map(c.params(O))
    for t, T in c.poses.items():
        m.set_pose(t, T)
    m.upload(c.records(), U.TS)
    m.update(c.pose, c.frame())
    return m.update_debug() + (m.download(),)


def check_against_model(got, model, what):
    idx, rad, integ, nu, nn, recs = got
    assert np.array_equal(idx, model["index"]), what + ": index map"
    assert_bits_equal(rad, model["radius"], what + ": radius map")
    assert np.array_equal(integ, model["integrated"]), what + ": integrated flags"
    want = (model["n_updated"], model["n_new"])
    assert (nu, nn) == want, "%s: counts %s, model %s" % (what, (nu, nn), want)
    M.compare(model, recs, what + ": surfels")


def model_of(c):
    m = M.update(c.params(O), c.records(), c.frame(), c.pose, U.TS, c.poses)
    U.check_tags(c, m)
    return m


@pytest.mark.parametrize("shape", U.SHAPES, ids=["%dx%d" % s for s in U.SHAPES])
@pytest.mark.parametrize("name", U.case_ids())
def test_update_case(name, shape):
    c = U.get(name, *shape)
    model = model_of(c)
    g, o = run_library(c), run_oracle(c)
    for a, b, nm in zip(g[:3], o[:3], ("index map", "radius map", "integrated flags")):
        assert_bits_equal(a, b, "%s: %s vs oracle" % (name, nm))
    assert g[3:5] == o[3:5], "%s: counts %s vs oracle %s" % (name, g[3:5], o[3:5])
    surfel_fields_equal(g[5], o[5], name + ": surfels vs oracle")
    check_against_model(o, model, name + " (oracle)")
    check_against_model(g, model, name + " (CUDA)")


def test_counts_include_surfels_outside_the_submap_window():
    """sb_map_update_debug counts what the update and the generation pass emit before the submap window, as the
    reference's transform feedback does; the map keeps only the surfels inside it"""
    c = U.get("submap", *U.SHAPES[0])
    model = model_of(c)
    assert model["n_updated"] > model["n_updated_kept"]
    g = run_library(c)
    assert g[3:5] == (model["n_updated"], model["n_new"]) and len(g[5]) == model["n_updated_kept"] + model["n_new_kept"]


def test_derived_uniforms_within_one_ulp():
    """the model's derived uniforms (fp32 of the fp64 formulas of SurfelMap::setParameters) lie within 1 ulp of fp64"""
    for shape in U.SHAPES:
        for c in U.all_cases(*shape):
            p = c.params(O)
            d, e = M.derived(p), M.derived_exact(p)
            for k, v in d.items():
                assert v == e[k] or abs(float(v) - e[k]) <= float(np.spacing(np.float32(abs(e[k])))), (c.name, k, v, e[k])


def test_every_branch_was_reached():
    """the models of all designed cases (each checked against CUDA and the oracle above) reach every branch, per shape"""
    for shape in U.SHAPES:
        got = set()
        for c in U.all_cases(*shape):
            got |= U.reached(model_of(c))
        assert U.BRANCHES <= got, "%s: branches never reached: %s" % (shape, sorted(U.BRANCHES - got))


# ---- the pipeline's own paths ------------------------------------------------------------------------------------------
PIPE = dict(min_radius=0.5, max_radius=1.0, max_depth=60.0, model_max_depth=60.0)  # both radius clamps are active


def _scan(H, W):
    """points on the beam centres of a room with a floor 1.7 m below the sensor and walls 3 to 40 m away (no direction
    left unconstrained for Gauss-Newton): normals from neighbours, radii on both clamps"""
    d = _beam_centres(H, W)
    t = np.linspace(0.0, 2.0 * np.pi, W, endpoint=False)[None, :]
    wall = np.broadcast_to(3.0 + 37.0 * (0.5 + 0.5 * np.cos(t)) + 4.0 * np.sin(3.0 * t), (H, W))
    floor = np.where(d[..., 2] < -1e-3, 1.7 / np.maximum(-d[..., 2], 1e-3), np.inf)
    rho = np.minimum(wall, floor)
    return np.concatenate([(d * rho[..., None]).reshape(-1, 3), np.ones((H * W, 1))], 1).astype(np.float32)


@pytest.mark.parametrize("shape", U.SHAPES, ids=["%dx%d" % s for s in U.SHAPES])
def test_pipeline_radius_copy_and_in_place_update(shape):
    """scan 1 builds the map (dense update); scan 2, the same points, runs the in-place update. After each: the radius
    map written by the tiled preprocessing pass equals the model on getCurrentFrame() and k_radius on the same frame
    uploaded at the operator level; update_debug and the records equal the oracle twin, and after scan 2 the model
    applied to the map before it, the frame and the pose the pipeline used."""
    H, W = shape
    kw = dict(PIPE, data_width=W, model_width=W, data_height=H, model_height=H)
    pp, po = api.default_params(**kw), O.default_params(**kw)
    pts = _scan(H, W)
    gsl, osl = api.SurfelMapping(pp), O.Slam(po)
    gsl.ctx.profile(True)
    before = None
    tags = set()
    for t in range(2):
        gsl.ctx.profile_collect()
        gsl.processScan(pts)
        osl.process_scan(pts)
        mode, _ = scan_modes(gsl)
        assert mode == ("dense" if t == 0 else "lazy"), (t, mode)
        assert_bits_equal(gsl.getCurrentPose(), osl.pose(), "scan %d pose" % t)
        frame = gsl.getCurrentFrame().maps()
        g = gsl.getMap().update_debug()
        o = osl.map.update_debug()
        for a, b, nm in zip(g[:3], o[:3], ("index map", "radius map", "integrated flags")):
            assert_bits_equal(a, b, "scan %d %s vs oracle" % (t, nm))
        assert g[3:5] == o[3:5], (t, g[3:5], o[3:5])
        # the tiled pass's radius copy against the model and against k_radius on the same frame
        d = M.derived(po)
        for y in range(H):
            for x in range(W):
                r, tag = M.radius_pixel(po, d, frame[0][y, x], frame[1][y, x])
                assert_bits_equal(g[1][y, x], r, "scan %d radius (%d, %d) vs model" % (t, y, x))
                tags |= set(tag.split(","))
        ctx = api.Context(pp)
        f = api.Frame(ctx, W, H)
        f.upload(frame)
        api.SurfelMap(ctx).update(np.eye(4, dtype=np.float32), f)
        assert_bits_equal(api.SurfelMap(ctx).update_debug()[1], g[1], "scan %d radius map vs k_radius" % t)
        ctx.close()
        recs = gsl.getMap().getAllSurfels()
        surfel_fields_equal(recs, osl.map.download(), "scan %d surfels vs oracle" % t)
        if before is not None:
            pose = gsl.getCurrentPose().astype(np.float32)
            model = M.update(po, before, frame, pose, t, {0: np.eye(4, dtype=np.float32)})
            check_against_model(g[:5] + (recs,), model, "in-place scan vs model")
        before = recs
    gsl.ctx.profile(False)
    assert {"radius:min", "radius:max", "radius:c_mid"} <= tags, tags
    gsl.ctx.close()
