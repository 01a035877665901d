"""The CUDA path at uneven image shapes, and the exact ICP sums against arithmetic that shares no code with the oracle.

1. Shape matrix, bit for bit against the oracle: preprocessing, sb_icp_jacobian (whole and as row stripes),
   sb_icp_minimize, rendering and map update, three processScan steps. The shapes cover
   - the three regimes of the persistent Gauss-Newton kernel on the device the tests run on (2-deep shared-memory
     pixel cache, 4-deep cache, no cache), each boundary from both sides; the shapes are derived from the device's
     co-resident block count, so they move with the SM count (gn_regime() mirrors sb_icp.cu);
   - the plain-load instantiation of the preprocessing tile (odd widths: the key image's row pitch 8 * (W + 6) bytes
     is then no multiple of 16 and no tensor map can be made), the TMA instantiation on partial tile rows and on an
     image smaller than its 38 x 22 box, images under 256 pixels, and widths 2 and 3, where the three mirror columns on
     each side of the key image overlap the image itself;
   - a model image of odd size different from the data image's.
   A data width of 1 is refused by sb_create (and by the oracle's constructors) with SB_ERR_INVALID: the flood fill
   reaches two columns around the azimuth seam, and the reference's single wrap() leaves the row there.
2. Known-answer sums: frames whose pixels each associate with themselves (points on their pixel's beam centre, the model
   shifted along the normal, nearest sampling, identity pose, no robust weight). The 32 raw Q33.30 sums are recomputed
   here in numpy float32 in the kernel's operation order and summed as Python integers.
3. Q33.30 head-room: a legal-looking size whose exact sum exceeds 2^63 is refused; the largest size accepted at that
   range sums exactly.
4. The update pass's 256 group totals are all cleared also on an image of fewer than 256 pixels (a stale total used to
   shift the compaction of the next update)."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api, synth
from helpers import assert_bits_equal, both_params, sized, surfel_fields_equal

pytestmark = pytest.mark.gpu

ICP_THREADS = 256          # kIcpThreads, sb_icp.cu
BLOCKS_PER_SM = 2          # __launch_bounds__(256, 2) of k_gn_persistent, confirmed by the occupancy query on an H100
INT64_MAX = 2 ** 63 - 1


# ---------------------------------------------------------------------------------------------------------------
# the Gauss-Newton regimes of the device
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def max_blocks(request):
    """co-resident blocks of the persistent Gauss-Newton kernel: 2 per SM of the device (the CPU executor's SM count
    under --cusim)"""
    if getattr(request.config, "_cusim", False):
        sms = min(max(int(os.environ.get("CUSIM_SMS", "4")), 1), 132)
    else:
        import torch
        sms = torch.cuda.get_device_properties(0).multi_processor_count
    return BLOCKS_PER_SM * sms


def gn_regime(pixels, max_blocks):
    """icp_balanced_blocks and the `deep` rule of launch_gn_persistent: "cache2", "cache4" or "nocache"."""
    units = -(-pixels // ICP_THREADS)
    u = -(-units // max_blocks)
    per_pass = -(-units // u) * ICP_THREADS
    if pixels <= 2 * per_pass:
        return "cache2"
    return "cache4" if pixels <= 4 * per_pass else "nocache"


# name -> (data height, data width, model (height, width) or None). B = co-resident blocks: 64 x 8B = 2 * B * 256
# pixels is the last image of the 2-deep regime, 64 x 16B the last of the 4-deep one (at B = 264: 64x2112, 64x4224).
SHAPES = {
    "gn_cache2_last": (64, "8B", None),
    "gn_cache4_first": (65, "8B", None),
    "gn_cache4_last": (64, "16B", None),
    "gn_nocache_first": (65, "16B", None),
    "odd_w361_h33": (33, 361, None),
    "odd_w513_h70": (70, 513, None),
    "odd_w901": (64, 901, None),
    "even_w900_h33": (33, 900, None),
    "even_w450_h70": (70, 450, None),
    "smaller_than_box_34x20": (20, 34, None),
    "under_256px_16x8": (8, 16, None),
    "w2": (16, 2, None),
    "w3": (16, 3, None),
    "model_451x47_data_513x33": (33, 513, (47, 451)),
}


def shape(name, max_blocks):
    H, W, model = SHAPES[name]
    if isinstance(W, str):
        W = int(W[:-1]) * max_blocks
    return H, W, model


def params(name, max_blocks, **kw):
    H, W, model = shape(name, max_blocks)
    Hm, Wm = model or (H, W)
    return both_params(data_width=W, data_height=H, model_width=Wm, model_height=Hm, **kw)


def test_shape_list_covers_every_gauss_newton_regime(max_blocks):
    got = {}
    for name in SHAPES:
        H, W, _ = shape(name, max_blocks)
        got.setdefault(gn_regime(H * W, max_blocks), []).append("%s=%dx%d" % (name, H, W))
    print("co-resident blocks %d: %s" % (max_blocks, got))
    assert set(got) == {"cache2", "cache4", "nocache"}, got
    # each boundary from both sides
    assert [gn_regime(H * W, max_blocks) for H, W, _ in (shape(n, max_blocks) for n in
            ("gn_cache2_last", "gn_cache4_first", "gn_cache4_last", "gn_nocache_first"))] == \
        ["cache2", "cache4", "cache4", "nocache"]


def test_regime_rule_at_132_sms():
    """the boundaries on an H100 SXM (132 SMs, 264 blocks)"""
    assert gn_regime(66 * 2048, 264) == "cache2"
    assert gn_regime(67 * 2048, 264) == "cache4"
    assert gn_regime(64 * 4224, 264) == "cache4"
    assert gn_regime(65 * 4224, 264) == "nocache"
    assert [gn_regime(64 * w, 264) for w in (900, 2048)] == ["cache2", "cache2"]
    assert gn_regime(128 * 4096, 264) == "nocache"


# ---------------------------------------------------------------------------------------------------------------
# 1. shape matrix against the oracle
# ---------------------------------------------------------------------------------------------------------------
_scan_cache = {}


def _scans(H, W, n):
    key = (H, W, n)
    if key not in _scan_cache:
        scene = synth.Scene(width=W, height=H, semantic=True)
        poses = synth.trajectory(n)
        _scan_cache[key] = ([scene.scan(f, poses[f]) for f in range(n)], poses)
    return _scan_cache[key]


def _prep_both(po, ctx, scan, timestamp):
    pts, lab, prb = scan
    ov = O.preprocess(po, pts, lab, prb, timestamp)
    f = api.Frame(ctx, po.data_width, po.data_height)
    api.Preprocessing(ctx).process(pts, f, lab, prb, timestamp)
    return ov, f


def _model_both(po, ctx, ov, pose):
    """a model-sized frame rendered by the oracle from a map of one frame, uploaded as it is for the CUDA path"""
    om = O.Map(po)
    om.update(np.eye(4, dtype=np.float32), ov)
    m = om.render(pose, pose, -1.0)
    g = api.Frame(ctx, po.model_width, po.model_height)
    g.upload(m)
    assert (m[0][..., 3] > 0).any()
    return m, g


@pytest.mark.parametrize("name", list(SHAPES))
def test_preprocess_bit_exact(name, max_blocks):
    po, pp = params(name, max_blocks)
    ctx = api.Context(pp)
    try:
        sc, _ = _scans(po.data_height, po.data_width, 2)
        for s, t in zip(sc, (3, 100)):
            ov, f = _prep_both(po, ctx, s, t)
            for g, o, what in zip(f.maps(), ov, ("vertex", "normal", "semantic")):
                assert_bits_equal(g, o, "%s t=%d %s" % (name, t, what))
            assert (ov[0][..., 3] > 0).any()
    finally:
        ctx.close()


@pytest.mark.parametrize("name", list(SHAPES))
def test_icp_jacobian_whole_and_striped(name, max_blocks):
    po, pp = params(name, max_blocks)
    H = po.data_height
    ctx = api.Context(pp)
    try:
        sc, poses = _scans(H, po.data_width, 2)
        o0, _ = _prep_both(po, ctx, sc[0], 100)
        o1, f1 = _prep_both(po, ctx, sc[1], 100)
        om, gm = _model_both(po, ctx, o0, np.eye(4, dtype=np.float32))
        obj = api.Frame2Model(ctx)
        obj.setData(f1, gm)
        T = np.linalg.inv(poses[0]) @ poses[1]
        T[0, 3] += 0.05
        for it, pose in enumerate([np.eye(4), T]):
            obj.initialize(pose)
            obj.iteration_ = it
            obj.jacobianProducts()
            o48, raw = O.icp_jacobian(po, o1, om, pose, iteration=it)
            assert np.array_equal(obj.raw32, raw), "%s it=%d raw sums %s vs %s" % (name, it, obj.raw32, raw)
            assert_bits_equal(obj.out48, o48, "%s out48" % name)
            assert obj.valid() + obj.invalid() == po.data_width * H
        whole = obj.raw32.copy()
        cut = [0, H // 3, H // 3 + 1, H] if H >= 3 else [0, 1, H]
        tot = np.zeros(32, np.int64)
        for r0, r1 in zip(cut[:-1], cut[1:]):
            obj.jacobianProducts(rows=(r0, r1))
            _, raw = O.icp_jacobian(po, o1, om, T, iteration=1, rows=(r0, r1))
            assert np.array_equal(obj.raw32, raw), "%s rows %d..%d" % (name, r0, r1)
            tot += obj.raw32
        assert np.array_equal(tot, whole), "%s: the row stripes do not add up" % name
    finally:
        ctx.close()


@pytest.mark.parametrize("name", list(SHAPES))
def test_icp_minimize_bit_exact(name, max_blocks):
    po, pp = params(name, max_blocks)
    ctx = api.Context(pp)
    try:
        sc, _ = _scans(po.data_height, po.data_width, 2)
        o0, _ = _prep_both(po, ctx, sc[0], 100)
        o1, f1 = _prep_both(po, ctx, sc[1], 100)
        om, gm = _model_both(po, ctx, o0, np.eye(4, dtype=np.float32))
        obj = api.Frame2Model(ctx)
        obj.setData(f1, gm)
        gn = api.LieGaussNewton(ctx)
        gn.minimize(obj, np.eye(4))
        pose_o, o48, k, hist = O.icp_minimize(po, o1, om, np.eye(4))
        assert gn.iterationCount() == k, name
        assert_bits_equal(gn.pose(), pose_o, "%s pose" % name)
        assert_bits_equal(gn.out48, o48, "%s out48" % name)
        assert len(gn.history()) == len(hist), name
        for a, b in zip(gn.history(), hist):
            assert_bits_equal(a, b, "%s history" % name)
    finally:
        ctx.close()


@pytest.mark.parametrize("name", list(SHAPES))
def test_render_and_map_update_bit_exact(name, max_blocks):
    po, pp = params(name, max_blocks)
    ctx = api.Context(pp)
    try:
        sc, poses = _scans(po.data_height, po.data_width, 3)
        omap, gmap = O.Map(po), api.SurfelMap(ctx)
        out = api.Frame(ctx, po.model_width, po.model_height)
        for t in range(3):
            ov, f = _prep_both(po, ctx, sc[t], t)
            pose = (np.linalg.inv(poses[0]) @ poses[t]).astype(np.float32)
            orr = omap.render(pose, pose, -1.0 + 0.5 * t)
            gmap.render(pose, pose, out, -1.0 + 0.5 * t)
            for g, o, what in zip(out.maps(), orr, ("vertex", "normal", "semantic")):
                assert_bits_equal(g, o, "%s t=%d render %s" % (name, t, what))
            omap.update(pose, ov)
            gmap.update(pose, f)
            oi, orad, oint, onu, onn = omap.update_debug()
            gi, grad, gint, gnu, gnn = gmap.update_debug()
            assert_bits_equal(gi, oi, "%s t=%d index map" % (name, t))
            assert_bits_equal(grad, orad, "%s t=%d radius map" % (name, t))
            assert_bits_equal(gint, oint, "%s t=%d integrated flags" % (name, t))
            assert (gnu, gnn) == (onu, onn), "%s t=%d counts" % (name, t)
            assert gmap.size() == omap.size() > 0, "%s t=%d surfel count" % (name, t)
        surfel_fields_equal(gmap.getAllSurfels(), omap.download(), "%s surfels" % name)
    finally:
        ctx.close()


def _pipeline_equal(po, pp, sc, what, gsl=None, osl=None):
    """tests/test_gpu_parity.py::_pipeline_equal, repeated here so that this file stands alone"""
    osl = osl or O.Slam(po)
    gsl = gsl or api.SurfelMapping(pp)
    try:
        for t, (pts, lab, prb) in enumerate(sc):
            osl.process_scan(pts, lab, prb)
            gsl.processScan(pts, lab, prb)
            assert_bits_equal(gsl.getCurrentPose(), osl.pose(), "%s t=%d pose" % (what, t))
            so, sg = osl.stats(), gsl.getStatistics()
            assert sg["num_iterations"] == so["iterations"], "%s t=%d iterations" % (what, t)
            assert (sg["F"], sg["inlier"], sg["outlier"], sg["invalid"]) == (so["F"], so["inlier"], so["outlier"], so["invalid"]), \
                "%s t=%d statistics pass" % (what, t)
            assert gsl.getMap().size() == osl.map.size(), "%s t=%d surfel count" % (what, t)
        surfel_fields_equal(gsl.getMap().getAllSurfels(), osl.map.download(), what + " surfels")
        for g, o in zip(gsl.getCurrentFrame().maps(), osl.frame(0)):
            assert_bits_equal(g, o, what + " current frame")
        for g, o in zip(gsl.getLastModelFrame().maps(), osl.frame(1)):
            assert_bits_equal(g, o, what + " model frame")
    finally:
        gsl.ctx.close()


@pytest.mark.parametrize("name", list(SHAPES))
def test_process_scan_bit_exact(name, max_blocks):
    po, pp = params(name, max_blocks)
    sc, _ = _scans(po.data_height, po.data_width, 3)
    _pipeline_equal(po, pp, sc, name)


def test_data_width_one_is_refused():
    po, pp = both_params(**sized(1, 16))
    with pytest.raises(api.SumaError, match="INVALID"):
        api.Context(pp)
    assert O.check_params(po) == "data width < 2"
    with pytest.raises(ValueError):
        O.Slam(po)
    # the model image may be one column wide
    po, pp = both_params(data_width=2, data_height=16, model_width=1, model_height=16)
    assert O.check_params(po) is None
    api.Context(pp).close()


# ---------------------------------------------------------------------------------------------------------------
# 2. known-answer sums, independent of the oracle
# ---------------------------------------------------------------------------------------------------------------
def _beam_centres(H, W, fov_up=3.0, fov_down=-25.0):
    """unit directions (float64, [H, W, 3]) through the centre of every pixel (gen_vertexmap.vert:78-89)"""
    fov = fov_up - fov_down
    az = np.pi * (1.0 - 2.0 * (np.arange(W) + 0.5) / W)
    el = np.deg2rad(fov_up - fov * (1.0 - (np.arange(H) + 0.5) / H))
    el, az = np.meshgrid(el, az, indexing="ij")
    return np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], -1)


def kat_frames(H, W, rng=None, rng_range=None, normals="random"):
    """data and model images in which every pixel associates with itself: float32 [H, W, 4] vertex / normal maps"""
    d = _beam_centres(H, W)
    rho = np.full((H, W), rng_range) if rng is None else rng.uniform(4.0, 60.0, (H, W))
    v = (d * rho[..., None]).astype(np.float32)
    if normals == "random":
        n = rng.normal(size=(H, W, 3))
    else:  # the normal that maximises (v x n).x, the Jacobian's rotation about x: JtJ(4,4)
        n = np.stack([np.zeros((H, W)), -v[..., 2], v[..., 1]], -1).astype(np.float64)
        n[np.linalg.norm(n, axis=-1) == 0] = (0, 0, 1)
    n = (n / np.linalg.norm(n, axis=-1, keepdims=True)).astype(np.float32)
    delta = (rng.uniform(-0.3, 0.3, (H, W)) if rng is not None else np.full((H, W), 0.1)).astype(np.float32)
    vm = (v + delta[..., None] * n).astype(np.float32)
    one = np.ones((H, W, 1), np.float32)
    zero = np.zeros((H, W, 4), np.float32)
    data = (np.concatenate([v, one], -1), np.concatenate([n, one], -1), zero)
    model = (np.concatenate([vm, one], -1), np.concatenate([n, one], -1), zero)
    return data, model


def _exact_sum(terms):
    """sum of an int64 array as a Python integer, exactly: high and low 32-bit halves summed separately"""
    t = terms.reshape(-1)
    return int(np.sum(t >> 32)) * 2 ** 32 + int(np.sum(t & 0xffffffff))


def kat_raw32(data, model):
    """the 32 raw sums of Frame2Model_jacobians.geom with weight 1 and every pixel an inlier, as Python integers: the
    kernel's fp32 operations in its order (numpy does not contract a*b+c to an FMA), each term * 2^30 rounded to nearest
    even, summed exactly"""
    f32 = np.float32
    vd = [data[0][..., i].astype(f32) for i in range(3)]
    vm = [model[0][..., i].astype(f32) for i in range(3)]
    nm = [model[1][..., i].astype(f32) for i in range(3)]
    d = [vd[i] - vm[i] for i in range(3)]                                        # sub3(v_d, v_m)
    r = (nm[0] * d[0] + nm[1] * d[1]) + nm[2] * d[2]                             # dot3(n_m, .)
    cp = [vd[1] * nm[2] - vd[2] * nm[1], vd[2] * nm[0] - vd[0] * nm[2], vd[0] * nm[1] - vd[1] * nm[0]]  # cross3(v_d, n_m)
    J = nm + cp
    scale = f32(2.0 ** 30)

    def fix(t):
        assert t.dtype == np.float32
        return np.rint(t * scale).astype(np.int64)

    raw = []
    for c in range(6):
        for rr in range(c, 6):
            raw.append(_exact_sum(fix(J[c] * J[rr])))                             # (w * J_c) * J_r, w = 1
    for rr in range(6):
        raw.append(_exact_sum(fix(r * J[rr])))
    F = _exact_sum(fix(r * r))
    P = vd[0].size
    return raw + [F, F, P, 0, 0]


def _kat_check(po, pp, data, model, what):
    """raw32 of sb_icp_jacobian and out48 of the first step of sb_icp_minimize against kat_raw32"""
    want = kat_raw32(data, model)
    assert all(-2 ** 63 <= x <= INT64_MAX for x in want), "%s: the exact sums leave int64: %s" % (what, want)
    P = po.data_width * po.data_height
    ctx = api.Context(pp)
    try:
        fd = api.Frame(ctx, po.data_width, po.data_height)
        fm = api.Frame(ctx, po.model_width, po.model_height)
        fd.upload(data)
        fm.upload(model)
        obj = api.Frame2Model(ctx)
        obj.setData(fd, fm)
        obj.initialize(np.eye(4))
        obj.jacobianProducts()
        assert (obj.valid(), obj.invalid(), obj.outlier()) == (P, 0, 0), what
        got = [int(x) for x in obj.raw32]
        bad = [i for i in range(32) if got[i] != want[i]]
        assert not bad, "%s: raw sums %s differ: %s vs %s" % (what, bad, [got[i] for i in bad], [want[i] for i in bad])
        # the first Gauss-Newton step evaluates the same sums (out48 = raw * 2^-30, one rounding to double)
        p1 = api.Params.from_buffer_copy(pp)
        p1.max_iterations = 1
        ctx.set_params(p1)
        gn = api.LieGaussNewton(ctx)
        gn.minimize(obj, np.eye(4))
        assert_bits_equal(gn.out48, _unpack48(want), what + " out48 of the first Gauss-Newton step")
        assert gn.iterationCount() <= 1 and len(gn.history()) >= 1
    finally:
        ctx.close()


def _unpack48(raw):
    """sb_icp_unpack in Python: (double)raw * 2^-30 (float(int) rounds to nearest even, as the int64 -> double
    conversion does)"""
    s = 2.0 ** -30
    out = np.zeros(48)
    k = 0
    for c in range(6):
        for r in range(c, 6):
            out[c * 6 + r] = out[r * 6 + c] = float(raw[k]) * s
            k += 1
    out[36:42] = [float(x) * s for x in raw[21:27]]
    out[42], out[43], out[44], out[45], out[46] = float(raw[29]), float(raw[27]) * s, float(raw[30]), float(raw[28]) * s, \
        float(raw[31])
    return out


def _kat_params(H, W, **kw):
    return both_params(**sized(W, H, bilinear_sampling=0, weighting=0, **kw))


@pytest.mark.parametrize("name", [n for n in SHAPES if SHAPES[n][1] != 1])
def test_known_answer_sums(name, max_blocks):
    H, W, _ = shape(name, max_blocks)
    po, pp = _kat_params(H, W)
    rng = np.random.default_rng(H * 100003 + W)
    data, model = kat_frames(H, W, rng)
    _kat_check(po, pp, data, model, "%s (%dx%d, %s)" % (name, H, W, gn_regime(H * W, max_blocks)))


# ---------------------------------------------------------------------------------------------------------------
# 3. Q33.30 head-room
# ---------------------------------------------------------------------------------------------------------------
def test_sums_that_would_leave_int64_are_refused():
    """256x16384 at 75 m (under the 2^24-pixel limit): the exact JtJ(4,4) of surfaces facing away from the x axis is
    above 2^63, so an int64 sum would wrap -- in the oracle as well. Such parameters are refused; the largest image
    accepted at 75 m (128 x 6710) sums exactly."""
    H, W = 256, 16384
    data, model = kat_frames(H, W, rng_range=75.0, normals="max_x")
    want = kat_raw32(data, model)
    assert want[15] > INT64_MAX, "JtJ(4,4) = %d fits: the case shows nothing" % want[15]
    po, pp = _kat_params(H, W)
    try:
        ctx = api.Context(pp)
    except api.SumaError:
        pass
    else:  # accepted: show what the sums became
        try:
            fd, fm = api.Frame(ctx, W, H), api.Frame(ctx, W, H)
            fd.upload(data)
            fm.upload(model)
            obj = api.Frame2Model(ctx)
            obj.setData(fd, fm)
            obj.jacobianProducts()
            got = int(obj.raw32[15])
        finally:
            ctx.close()
        pytest.fail("sb_create accepted %dx%d at 75 m; JtJ(4,4) = %d, exact %d" % (H, W, got, want[15]))
    assert O.check_params(po) is not None
    with pytest.raises(ValueError):
        O.Map(po)
    # the rule's boundary at 75 m, H = 128: 858 880 pixels accepted, 859 008 refused
    po, pp = _kat_params(128, 6711)
    assert O.check_params(po) is not None
    with pytest.raises(api.SumaError):
        api.Context(pp)
    po, pp = _kat_params(128, 6710)
    assert O.check_params(po) is None
    data, model = kat_frames(128, 6710, rng_range=75.0, normals="max_x")
    _kat_check(po, pp, data, model, "128x6710 at 75 m")
    # sb_set_params applies the same rule (a depth range of 200 m at 128x4096 is refused; the context keeps working)
    po, pp = both_params(**sized(4096, 128))
    assert O.check_params(po) is None
    ctx = api.Context(pp)
    try:
        p2 = api.default_params(**sized(4096, 128), max_depth=200.0)
        with pytest.raises(api.SumaError, match="int64"):
            ctx.set_params(p2)
        p2.max_depth = 75.0
        ctx.set_params(p2)
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# 4. group totals of the update pass on an image under 256 pixels
# ---------------------------------------------------------------------------------------------------------------
def _random_surfels(rng, n, t_now):
    s = np.zeros(n, O.SURFEL_DTYPE)
    d = rng.uniform(1.0, 80.0, n)
    yaw = rng.uniform(-np.pi, np.pi, n)
    pitch = np.deg2rad(rng.uniform(-30.0, 6.0, n))
    s["x"], s["y"], s["z"] = d * np.cos(pitch) * np.cos(yaw), d * np.cos(pitch) * np.sin(yaw), d * np.sin(pitch)
    nrm = rng.normal(size=(n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    s["nx"], s["ny"], s["nz"] = nrm[:, 0], nrm[:, 1], nrm[:, 2]
    s["radius"] = rng.uniform(0.01, 1.2, n) * (d / 20.0 + 0.2)
    s["confidence"] = rng.uniform(-1.0, 3.0, n)
    creation = rng.integers(0, t_now + 1, n)
    s["count"] = creation
    s["timestamp"] = np.minimum(creation + rng.integers(0, 40, n), t_now)
    s["weight"] = rng.uniform(0.5, 19.5, n)
    return s


N_SURFELS = 3_600_000  # 220 groups of 64 x 256 surfels: more than the 128 pixels of a 16x8 image


def test_map_updates_on_an_image_under_256_pixels():
    """three updates of a 3.6 M-surfel map with one 16x8 frame: every update's compaction must start from zeroed group
    totals. It used to see the previous update's totals of groups 128..255 and grew the map to capacity."""
    po, pp = both_params(**sized(16, 8))
    ctx = api.Context(pp)
    try:
        S = _random_surfels(np.random.default_rng(11), N_SURFELS, 50)
        om, gm = O.Map(po), api.SurfelMap(ctx)
        om.upload(S, 50)
        gm.upload(S, 50)
        sc, _ = _scans(8, 16, 1)
        ov, f = _prep_both(po, ctx, sc[0], 100)
        sizes = []
        for t in range(3):
            om.update(np.eye(4, dtype=np.float32), ov)
            gm.update(np.eye(4, dtype=np.float32), f)
            sizes.append(om.size())
            assert gm.size() == om.size(), "update %d: %d surfels, oracle %d" % (t, gm.size(), om.size())
        assert sizes[-1] > 16384 * 128, sizes  # groups past the image's pixel count still hold surfels
        surfel_fields_equal(gm.getAllSurfels(), om.download(), "surfels after three updates")
    finally:
        ctx.close()


def test_process_scan_on_an_image_under_256_pixels():
    """the same through processScan, whose tiled preprocessing pass clears the group totals"""
    po, pp = both_params(**sized(16, 8))
    S = _random_surfels(np.random.default_rng(12), N_SURFELS, 50)
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    osl.map.upload(S, 50)
    gsl.getMap().upload(S, 50)
    sc, _ = _scans(8, 16, 1)
    _pipeline_equal(po, pp, [sc[0]] * 3, "16x8 with 3.6 M surfels", gsl=gsl, osl=osl)
