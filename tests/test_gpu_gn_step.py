"""The Gauss-Newton step and the ICP weights against exact arithmetic: degenerate systems, pivot ties, stop tests and the
thresholds of the per-pixel decisions.

1. Designed systems. Frames are uploaded directly, every pixel associates with itself (kat_frames of
   test_gpu_shapes.py: points on their pixel's beam centre, the model shifted along its normal, identity pose, nearest
   sampling), and the model normals give J^T J a known structure exactly: axis-aligned normals make the affected Jacobian
   entries exact zeros in fp32 (cross3(v, e_z) = (v.y, -v.x, 0)). Cases: an empty model (every pivot zero), a plane
   (three zero pivots), a corridor (one), a symmetric box (translation diagonals that are exact pixel counts: exact ties
   in the pivot search, or a forced pivot order), two equal translation columns (a tie that decides which component the
   zero pivot sets to 0, so that the strict `>` of the pivot search changes the step, not just its rounding), a
   near-singular plane (tiny pivots, a large step, se3_exp past its range reduction) and random normals. The error tie
   is taken from a later pose of the same run where the run from identity never isolates it. For each: the raw sums of sb_icp_jacobian against kat_raw32; an LDL^T in
   fractions.Fraction with diagonal pivoting (first maximum wins, a zero pivot leaves its component 0) against the host
   sb_ldlt_solve6 / sb_gn_step; one step of sb_icp_minimize (the device's gn_step_warp) against the host step bit for
   bit. The chain: exact model => host step within a conditioning-scaled bound => device step bit for bit.
2. Stop tests. sb_icp_minimize with max_iterations 1, 2 and 7 and each stop test (linf < delta, |max J^T r| < eps, the
   error tie) at equality and one ulp either side, replayed on the host (sb_icp_jacobian = k_icp_jacobian, then
   sb_icp_unpack and sb_gn_step = sbg::gn_step): iteration count, history, out48 and pose bit-identical, at one shape
   per regime of the persistent kernel (2-deep cache, 4-deep cache, no cache) of the device the tests run on.
3. Weights and inlier tests at their thresholds, against a numpy model of the kernel's per-pixel fp32 arithmetic in its
   operation order: residuals at the robust-weight factor and one ulp either side (both signs, Huber, weighting 4,
   Tukey at iterations 0 and 1), distances at distance_thresh +- 1 ulp, normal dots at the angle threshold +- 1 ulp,
   invalid data / model pixels, projections outside the model image, and semantic weights.
   Bilinear sampling is covered by oracle parity only (test_gpu_shapes.py, test_gpu_parity.py): its weights depend on
   the pinned atan2f_ / asinf_ of the projection, which a numpy model would have to copy rather than check.
4. Degenerate scenes through sb_process_scan, bit for bit against the oracle: a ground plane, a corridor, an empty scan
   and a scan entirely beyond max_depth in the middle of a sequence, and a 0.5 m vertical jump over a plane that sends
   the track-loss recovery onto a degenerate system."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as O
from semantic_suma_b200 import api
from semantic_suma_b200.api import lib
from helpers import assert_bits_equal, both_params, sized
from test_gpu_shapes import (_beam_centres, _exact_sum, _model_both, _pipeline_equal, _scans, _unpack48, gn_regime,
                             kat_raw32, max_blocks, shape)  # noqa: F401  (max_blocks is a fixture)

pytestmark = pytest.mark.gpu

f32 = np.float32
FLT_MAX = float(np.finfo(np.float32).max)  # LieGaussNewton.cpp:48, the last error before the first step
EPS64 = 2.0 ** -53
KINDS = ["empty", "plane", "corridor", "box", "box_uneven", "tied_columns", "near_singular", "generic"]
ZERO_PIVOTS = {"empty": 6, "plane": 3, "corridor": 1, "box": 0, "box_uneven": 0, "tied_columns": 1, "near_singular": 0,
               "generic": 0}
H1, W1 = 16, 96  # the shape of the single-step cases: 1536 pixels, a multiple of 6


# ---------------------------------------------------------------------------------------------------------------
# designed frames
# ---------------------------------------------------------------------------------------------------------------
def _axis_normals(rng, P, counts, axes):
    """P unit normals: counts[i] of them +-e_axes[i] (random signs), at random pixels"""
    n = np.zeros((P, 3))
    idx = rng.permutation(P)
    at = 0
    for c, a in zip(counts, axes):
        n[idx[at:at + c], a] = rng.choice((-1.0, 1.0), c)
        at += c
    assert at == P
    return n


def designed_frames(kind, H, W, seed=0):
    """data and model images (float32 [H, W, 4] vertex / normal / semantic maps) in which every pixel associates with
    itself, with model normals chosen for `kind`"""
    rng = np.random.default_rng(seed * 7919 + KINDS.index(kind))
    P = H * W
    d = _beam_centres(H, W)
    # the box needs rotation diagonals below the translation ones (points within 0.3 m), so that the translation pivots
    # are chosen first while they are still exact pixel counts
    rho = rng.uniform(0.05, 0.3, (H, W)) if kind.startswith(("box", "tied")) else rng.uniform(4.0, 60.0, (H, W))
    v = (d * rho[..., None]).astype(f32)
    if kind == "plane":
        n = _axis_normals(rng, P, [P], [2])
        n[:, 2] = 1.0
    elif kind == "corridor":
        n = _axis_normals(rng, P, [P // 3, P - P // 3], [1, 2])
        n[:, 2] = np.abs(n[:, 2])
    elif kind == "box":  # equal counts (x and y at least, when P is no multiple of 3)
        n = _axis_normals(rng, P, [P // 3, P // 3, P - 2 * (P // 3)], [0, 1, 2])
    elif kind == "box_uneven":  # z > y > x: the pivot order becomes 2, 1, 0
        n = _axis_normals(rng, P, [P // 6, P // 3, P - P // 6 - P // 3], [0, 1, 2])
    elif kind == "tied_columns":
        # n = +-(1, 1, 0) (not unit: the kernel takes the normal as it is) on a power-of-two number of pixels, +-e_z on the
        # rest: the tx and ty columns are equal, their diagonal is a power of two times 2^30, so eliminating one leaves
        # the other exactly 0. The tie between them decides which of the two components the zero pivot sets to 0.
        m = 1 << int(math.log2(P // 3))
        n = _axis_normals(rng, P, [m, P - m], [0, 2])
        n[:, 1] = n[:, 0]
        n = n.reshape(H, W, 3).astype(f32)
    elif kind == "near_singular":  # the plane with 8 pixels tilted by 2e-4 rad
        n = np.zeros((P, 3))
        n[:, 2] = 1.0
        a, b = 2e-4, rng.uniform(-np.pi, np.pi, 8)
        n[rng.choice(P, 8, replace=False)] = np.stack([np.sin(a) * np.cos(b), np.sin(a) * np.sin(b),
                                                       np.full(8, np.cos(a))], -1)
    else:  # generic, empty
        n = rng.normal(size=(P, 3))
    if kind != "tied_columns":
        n = (n / np.linalg.norm(n, axis=-1, keepdims=True)).reshape(H, W, 3).astype(f32)
    delta = rng.uniform(-0.3, 0.3, (H, W)).astype(f32)
    vm = (v + delta[..., None] * n).astype(f32)
    one = np.ones((H, W, 1), f32)
    zero = np.zeros((H, W, 4), f32)
    data = (np.concatenate([v, one], -1), np.concatenate([n, one], -1), zero)
    mw = one * (0.0 if kind == "empty" else 1.0)
    model = (np.concatenate([vm, mw], -1), np.concatenate([n, mw], -1), zero)
    return data, model


def designed_raw32(kind, data, model):
    if kind == "empty":
        return [0] * 31 + [data[0].shape[0] * data[0].shape[1]]
    return kat_raw32(data, model)


# ---------------------------------------------------------------------------------------------------------------
# the 6x6 solve: exact model and a float mirror
# ---------------------------------------------------------------------------------------------------------------
def ldlt6(A48, num):
    """sbg::ldlt_solve6 on out48[0:36], b = -out48[36:42], in the number type `num` (Fraction: exact; float: the fp64
    operation order of the library). Diagonal pivoting, the first maximum wins, a zero pivot is skipped and leaves its
    solution component 0. Returns (x, perm, the steps k whose pivot was zero)."""
    A = [num(a) for a in A48[:36]]
    b = [-num(a) for a in A48[36:42]]
    perm = list(range(6))
    zero = []
    for k in range(6):
        piv, best = k, abs(A[k * 6 + k])
        for i in range(k + 1, 6):
            if abs(A[i * 6 + i]) > best:
                best, piv = abs(A[i * 6 + i]), i
        if piv != k:
            for i in range(6):
                A[k * 6 + i], A[piv * 6 + i] = A[piv * 6 + i], A[k * 6 + i]
            for i in range(6):
                A[i * 6 + k], A[i * 6 + piv] = A[i * 6 + piv], A[i * 6 + k]
            perm[k], perm[piv] = perm[piv], perm[k]
        dk = A[k * 6 + k]
        if dk == 0:
            zero.append(k)
            continue
        for i in range(k + 1, 6):
            A[k * 6 + i] = A[k * 6 + i] / dk
        for j in range(k + 1, 6):
            for i in range(j, 6):
                A[j * 6 + i] = A[j * 6 + i] - (A[k * 6 + i] * dk) * A[k * 6 + j]
                A[i * 6 + j] = A[j * 6 + i]
    y = [b[perm[i]] for i in range(6)]
    for i in range(6):
        for k in range(i):
            y[i] = y[i] - A[k * 6 + i] * y[k]
    for i in range(6):
        y[i] = num(0) if A[i * 6 + i] == 0 else y[i] / A[i * 6 + i]
    for i in range(5, -1, -1):
        for k in range(i + 1, 6):
            y[i] = y[i] - A[i * 6 + k] * y[k]
    x = [num(0)] * 6
    for i in range(6):
        x[perm[i]] = y[i]
    return x, perm, zero


def host_solve(A48):
    A = np.ascontiguousarray(A48[:36], np.float64)
    b = np.ascontiguousarray(-np.asarray(A48[36:42]), np.float64)
    x = np.zeros(6)
    lib().sb_ldlt_solve6(api._dp(A), api._dp(b), api._dp(x))
    return x


def host_step(out48, last_error, eps, delta, pose):
    """sb_gn_step: (result, new pose 4x4, dx)"""
    o = np.ascontiguousarray(out48, np.float64)
    p = api.colmajor(pose, np.float64)
    dx = np.zeros(6)
    res = lib().sb_gn_step(api._dp(o), last_error, eps, delta, api._dp(p), api._dp(dx))
    return res, api.from_colmajor(p), dx


def check_solve(A48, what):
    """exact model => host solve. Returns the exact model's (x, perm, zero pivots)."""
    xe, pe, ze = ldlt6(A48, Fraction)
    xm, pm, zm = ldlt6(A48, float)
    xh = host_solve(A48)
    # the float mirror is the host's code: the same bits, hence the host took the mirror's permutation
    assert_bits_equal(xh, np.array(xm), what + ": sb_ldlt_solve6 vs its fp64 mirror")
    assert (pm, zm) == (pe, ze), "%s: permutation / zero pivots %s %s, exact %s %s" % (what, pm, zm, pe, ze)
    for i in range(6):
        if xe[i] == 0:
            assert xh[i] == 0.0, "%s: x[%d] = %r where the exact solution is 0" % (what, i, xh[i])
    # the nonzero-pivot part: a backward-stable solve, ||x - x_exact|| <= c * eps * kappa * ||x_exact|| (c = 64 for six
    # unknowns; kappa of the system restricted to the unknowns whose pivots are nonzero)
    live = [i for i in range(6) if i not in [pe[k] for k in ze]]
    if live:
        A = np.array(A48[:36]).reshape(6, 6)[np.ix_(live, live)]
        kappa = np.linalg.cond(A)
        xn = max(abs(xe[i]) for i in live)
        err = max(abs(Fraction(float(xh[i])) - xe[i]) for i in live)
        if xn > 0:
            assert float(err / xn) <= 64 * EPS64 * kappa, \
                "%s: relative error %.3g over the bound %.3g (kappa %.3g)" % (what, float(err / xn), 64 * EPS64 * kappa,
                                                                            kappa)
    return xe, pe, ze


def _params(H, W, **kw):
    kw.setdefault("bilinear_sampling", 0)
    kw.setdefault("weighting", 0)
    return both_params(**sized(W, H, **kw))


def _frames(ctx, po, data, model):
    fd = api.Frame(ctx, po.data_width, po.data_height)
    fm = api.Frame(ctx, po.model_width, po.model_height)
    fd.upload(data)
    fm.upload(model)
    obj = api.Frame2Model(ctx)
    obj.setData(fd, fm)
    return obj


def first_step_equal(ctx, po, pp, obj, data, model, raw, what):
    """one iteration of sb_icp_minimize from identity: device pose = host sb_gn_step on the unpacked sums = oracle"""
    A48 = _unpack48(raw)
    _, pose_h, dx_h = host_step(A48, FLT_MAX, pp.stopping_threshold, pp.delta, np.eye(4))
    p1 = api.Params.from_buffer_copy(pp)
    p1.max_iterations = 1
    ctx.set_params(p1)
    gn = api.LieGaussNewton(ctx)
    gn.minimize(obj, np.eye(4))
    assert_bits_equal(gn.out48, A48, what + ": out48 of the first step")
    assert_bits_equal(gn.pose(), pose_h, what + ": device step vs sb_gn_step")
    po.max_iterations = 1
    pose_o, o48, k, _ = O.icp_minimize(po, data, model, np.eye(4))
    assert_bits_equal(pose_o, pose_h, what + ": oracle step vs sb_gn_step")
    assert_bits_equal(o48, A48, what + ": oracle out48")
    assert gn.iterationCount() == k
    return dx_h


# ---------------------------------------------------------------------------------------------------------------
# 1. designed systems
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_designed_system(kind):
    data, model = designed_frames(kind, H1, W1)
    want = designed_raw32(kind, data, model)
    po, pp = _params(H1, W1)
    ctx = api.Context(pp)
    try:
        obj = _frames(ctx, po, data, model)
        obj.initialize(np.eye(4))
        obj.jacobianProducts()
        got = [int(x) for x in obj.raw32]
        bad = [i for i in range(32) if got[i] != want[i]]
        assert not bad, "%s: raw sums %s differ: %s vs %s" % (kind, bad, [got[i] for i in bad], [want[i] for i in bad])
        A48 = _unpack48(want)
        xe, perm, zero = check_solve(A48, kind)
        assert len(zero) == ZERO_PIVOTS[kind], "%s: zero pivots at steps %s" % (kind, zero)
        if kind == "plane":  # tx, ty, rz
            assert sorted(perm[k] for k in zero) == [0, 1, 5]
        if kind == "corridor":
            assert [perm[k] for k in zero] == [0]
        if kind == "box":  # three equal counts: ties at steps 0 and 1, resolved in favour of the first
            assert A48[0] == A48[7] == A48[14] == (H1 * W1 // 3), A48[:15:7]
            assert perm[:3] == [0, 1, 2]
        if kind == "box_uneven":
            assert A48[0] < A48[7] < A48[14]
            assert perm[:3] == [2, 1, 0]
        if kind == "tied_columns":  # tz first, then the tie: ty (position 1) before tx (position 2); tx gets the zero
            assert A48[0] == A48[7] == A48[1] < A48[14], A48[:15]
            assert perm[:2] == [2, 1] and [perm[k] for k in zero] == [0]
            assert xe[0] == 0 and xe[1] != 0
        dx = first_step_equal(ctx, po, pp, obj, data, model, want, kind)
        assert_bits_equal(dx, host_solve(A48), kind + ": sb_gn_step's increment vs sb_ldlt_solve6")
        if kind == "near_singular":  # se3_exp at a large angle: sincos_ reduces by a multiple of pi/4
            theta = math.sqrt(dx[3] ** 2 + dx[4] ** 2 + dx[5] ** 2)
            assert theta > math.pi / 4 and max(abs(x) for x in xe) > 1.0, (theta, dx)
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# 2. stop tests and iteration counts, replayed on the host
# ---------------------------------------------------------------------------------------------------------------
def replay(obj, T0, max_iter, eps, delta):
    """LieGaussNewton::minimize driven from the host: k_icp_jacobian, sb_icp_unpack, sb_gn_step. Returns the pose,
    the last out48, k, the history, the trace [(linf, |max J^T r|, error)] and the step at which a stop test fired."""
    pose, last, k, hist, trace, stop = np.array(T0, np.float64), FLT_MAX, 0, [], [], None
    out48 = np.zeros(48)
    while True:
        hist.append(pose.copy())
        if k >= max_iter:
            break
        obj.initialize(pose)
        obj.iteration_ = k
        obj.jacobianProducts()
        out48 = np.zeros(48)
        lib().sb_icp_unpack(obj.raw32.ctypes.data_as(api.C.POINTER(api.C.c_int64)), api._dp(out48))
        assert_bits_equal(out48, obj.out48, "sb_icp_unpack")
        res, pose, dx = host_step(out48, last, eps, delta, pose)
        trace.append((float(np.max(np.abs(dx))), abs(float(np.max(out48[36:42]))), float(out48[43])))
        last = float(out48[43])
        if res == 0:
            stop = len(trace) - 1
            break
        k += 1
    return pose, out48, k, hist, trace, stop


def _stop_frames(case, H, W):
    """(po, pp, data, model) of a stop-test case: a designed system with Tukey weights, or a real scene pair"""
    if case == "scene":
        po, pp = both_params(**sized(W, H))
        sc, _ = _scans(H, W, 2)
        o0 = O.preprocess(po, *sc[0], timestamp=100)
        o1 = O.preprocess(po, *sc[1], timestamp=100)
        om = O.Map(po)
        om.update(np.eye(4, dtype=f32), o0)
        return po, pp, o1, om.render(np.eye(4, dtype=f32), np.eye(4, dtype=f32), -1.0)
    po, pp = _params(H, W, weighting=2)
    data, model = designed_frames(case, H, W, seed=1)
    return po, pp, data, model


def _isolated_tie(trace):
    """(k, |error_k - error_k-1|) of the first step k >= 1 at which the error tie alone decides at eps = that
    difference plus one ulp: the error fell, no earlier step fell by as little, and |max Jtr| stays above it"""
    for k in range(1, len(trace)):
        dec = abs(trace[k][2] - trace[k - 1][2])
        up = float(np.nextafter(dec, np.inf))
        if trace[k][2] < trace[k - 1][2] and all(m > up for _, m, _ in trace[:k + 1]) and \
                not any(trace[j][2] < trace[j - 1][2] and abs(trace[j][2] - trace[j - 1][2]) <= up for j in range(1, k)):
            return k, dec
    return None


REGIME_SHAPE = {"cache2": "gn_cache2_last", "cache4": "gn_cache4_first", "nocache": "gn_nocache_first"}


@pytest.mark.parametrize("regime", list(REGIME_SHAPE))
@pytest.mark.parametrize("case", KINDS + ["scene"])
def test_stop_tests_at_their_boundaries(case, regime, max_blocks):
    H, W, _ = shape(REGIME_SHAPE[regime], max_blocks)
    assert gn_regime(H * W, max_blocks) == regime
    po, pp, data, model = _stop_frames(case, H, W)
    ctx = api.Context(pp)
    try:
        obj = _frames(ctx, po, data, model)
        gn = api.LieGaussNewton(ctx)
        T0 = np.eye(4)
        _, _, _, _, trace, stop = replay(obj, T0, 7, 0.0, 0.0)
        assert stop is None, "%s: a stop test fired with both thresholds 0" % case
        linf0, maxc0, _ = trace[0]
        settings = []  # (what, eps, delta, the step the boundary is at, its side, the first pose)
        for side, d in (("-1ulp", -np.inf), ("=", None), ("+1ulp", np.inf)):
            nx = (lambda v: v) if d is None else (lambda v, d=d: float(np.nextafter(v, d)))
            settings.append(("linf < delta at delta %s" % side, 0.0, nx(linf0), 0, side, T0))
            settings.append(("|max Jtr| < eps at eps %s" % side, nx(maxc0), 0.0, 0, side, T0))
        # the error tie at the first step k >= 1 whose error fell by less than every |max Jtr| up to it; where the run
        # from identity has no such step, from a later pose of that run (closer to convergence the error steps shrink
        # faster than the gradient)
        hist0 = replay(obj, T0, 12, 0.0, 0.0)[3]
        tie = None
        for start in hist0:
            tie = _isolated_tie(replay(obj, start, 7, 0.0, 0.0)[4])
            if tie is not None:
                break
        if case in ("generic", "scene"):
            assert tie is not None, "%s: no run isolates the error tie" % case
        if tie is not None:
            k, dec = tie
            for side, d in (("-1ulp", -np.inf), ("=", None), ("+1ulp", np.inf)):
                e = dec if d is None else float(np.nextafter(dec, d))
                settings.append(("error tie at eps %s" % side, e, 0.0, k, side, start))
        for what, eps, delta, at, side, start in settings:
            for max_iter in (1, 2, 7):
                tag = "%s %s: %s, max_iter %d" % (case, regime, what, max_iter)
                pose_h, o48_h, k_h, hist_h, tr, stop_h = replay(obj, start, max_iter, eps, delta)
                if max_iter > at:  # the boundary is reached: taken one ulp past it only
                    assert (stop_h == at) == (side == "+1ulp"), "%s: stop at step %s" % (tag, stop_h)
                gn.maxIter, gn.epsilon, gn.delta = max_iter, eps, delta
                gn.minimize(obj, start)
                assert gn.iterationCount() == k_h, "%s: %d iterations, host %d" % (tag, gn.iterationCount(), k_h)
                assert len(gn.history()) == len(hist_h), tag
                for a, b in zip(gn.history(), hist_h):
                    assert_bits_equal(a, b, tag + " history")
                assert_bits_equal(gn.out48, o48_h, tag + " out48")
                assert_bits_equal(gn.pose(), pose_h, tag + " pose")
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# 3. weights and inlier tests at their thresholds
# ---------------------------------------------------------------------------------------------------------------
FACTOR = f32(0.75)   # the robust-weight factor, in [0.5, 1) with its neighbours: one ulp is 2^-24 on both sides
DIST = f32(0.875)    # icp_max_distance
ANGLE = f32(30.0)    # icp_max_angle in degrees
H3, W3 = 16, 64
MOVABLE = (10.0, 11.0, 13.0, 15.0, 18.0, 20.0, 30.0, 31.0, 32.0)  # is_movable, sb_math.cuh


def angle_threshold(max_angle_deg):
    """the fp32 threshold icp_args (sb_api.cu) derives: (float)cos(max_angle * pi / 180) in fp64"""
    return f32(math.cos(float(max_angle_deg) * math.pi / 180.0))


def _ulps(x):
    x = f32(x)
    return [np.nextafter(x, f32(-np.inf)), x, np.nextafter(x, f32(np.inf))]


def threshold_frames():
    """(data, model, outside, kinds): n_m = e_z everywhere, model = data shifted along z only, so that the residual and
    the distance of every threshold pixel are the exact float chosen for it. outside marks the pixels whose projection
    leaves the model image."""
    rng = np.random.default_rng(3)
    H, W, P = H3, W3, H3 * W3
    d = _beam_centres(H, W).reshape(P, 3)
    v = (d * 0.25).astype(f32)  # |z| < 0.11: v.z - r stays below 1 in magnitude for every r used here
    v[:, 2] = (np.round(v[:, 2].astype(np.float64) * 2 ** 24) / 2 ** 24).astype(f32)  # on the 2^-24 grid
    nd = np.zeros((P, 3), f32)
    nd[:, 2] = 1.0
    r = rng.uniform(-0.3, 0.3, P).astype(f32)
    exact = np.zeros(P, bool)
    vw, mw = np.ones(P, f32), np.ones(P, f32)
    outside = np.zeros(P, bool)
    sd, sm = np.zeros((P, 4), f32), np.zeros((P, 4), f32)
    kinds = []
    spots = iter(rng.permutation(P))

    def put(kind, res=None):
        i = next(spots)
        kinds.append((i, kind))
        if res is not None:
            r[i] = res
            exact[i] = True
        return i
    for s in (1.0, -1.0):
        for x in _ulps(FACTOR):
            put("residual %+.9g" % (s * x), f32(s * x))
        for x in _ulps(DIST):
            put("distance %+.9g" % (s * x), f32(s * x))
    for c in _ulps(angle_threshold(ANGLE)):
        i = put("normal dot %.9g" % c, f32(0.125))
        nd[i] = (f32(math.sqrt(1.0 - float(c) ** 2)), 0.0, c)
    vw[put("invalid data")] = 0.0
    mw[put("invalid model")] = 0.0
    for z in (4.0, -4.0):  # steeply up / down: outside the vertical field of view
        i = put("outside %+g" % z)
        v[i] = (0.01, 0.0, z)
        outside[i] = True
    for ml in (10.0, 40.0):
        for same in (True, False):
            for prob in (0.0, 1.0, 0.5):
                for res in (0.125, -1.0):
                    i = put("semantic model %g %s prob %g r %g" % (ml, "same" if same else "other", prob, res), f32(res))
                    dl = ml if same else ml + 1.0
                    sm[i, 0] = f32(ml) / f32(255.0)
                    sd[i, 0], sd[i, 3] = f32(dl) / f32(255.0), prob
    vm = v.copy()
    vm[:, 2] = (v[:, 2] - r).astype(f32)
    bad = exact & ((v[:, 2] - vm[:, 2]) != r)
    assert not bad.any(), "a residual is not exact"
    one = np.ones(P, f32)
    nm = np.zeros((P, 3), f32)
    nm[:, 2] = 1.0
    img = lambda a, w: np.concatenate([a, w[:, None]], -1).reshape(H, W, 4).astype(f32)  # noqa: E731
    data = (img(v, vw), img(nd, one), sd.reshape(H, W, 4))
    model = (img(vm, mw), img(nm, mw), sm.reshape(H, W, 4))
    return data, model, outside, kinds


def _round_away(x):
    return np.sign(x) * np.floor(np.abs(x) + f32(0.5))


def weighted_raw32(data, model, outside, weighting, factor, iteration, dist_thr, angle_thr):
    """icp_pixel_v (sb_icp.cu) for frames whose pixels associate with themselves (or leave the image where `outside`),
    identity pose, nearest sampling: the fp32 operations in the kernel's order, each term * 2^30 rounded to nearest
    even, summed exactly. Returns the 32 raw sums as Python integers."""
    P = data[0].shape[0] * data[0].shape[1]
    Vd, Nd, Sd = [a.reshape(P, 4).astype(f32) for a in data]
    Vm, Nm, Sm = [a.reshape(P, 4).astype(f32) for a in model]
    invalid = ~((Vd[:, 3] + Nd[:, 3]) > f32(1.5)) | outside
    invalid |= ~((Vm[:, 3] + Nm[:, 3]) > f32(1.5))
    ok = ~invalid
    vd, nd, vm, nm = [[a[ok, i] for i in range(3)] for a in (Vd, Nd, Vm, Nm)]
    dot = lambda a, b: (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]  # noqa: E731
    dist = np.sqrt(dot([vm[i] - vd[i] for i in range(3)], [vm[i] - vd[i] for i in range(3)]))
    inlier = ~(dist > dist_thr) & ~(dot(nm, nd) < angle_thr)
    res = dot(nm, [vd[i] - vm[i] for i in range(3)])
    cp = [vd[1] * nm[2] - vd[2] * nm[1], vd[2] * nm[0] - vd[0] * nm[2], vd[0] * nm[1] - vd[1] * nm[0]]
    J = nm + cp
    w = np.ones_like(res)
    big = np.abs(res) > factor
    if weighting in (1, 4):
        w[big] = factor / np.abs(res[big])
    elif weighting == 2 and iteration > 0:
        alpha = res / factor
        t = f32(1.0) - alpha * alpha
        w = np.where(big, f32(0.0), t * t).astype(f32)
    dl, dp, ml = Sd[ok, 0] * f32(255.0), Sd[ok, 3], Sm[ok, 0] * f32(255.0)
    mov = np.isin(ml, np.array(MOVABLE, f32))
    diff = _round_away(dl) != _round_away(ml)
    w = np.where(mov & diff, w * (f32(1.0) - dp), np.where(mov, w * dp, w)).astype(f32)
    assert w.dtype == f32 and res.dtype == f32

    def fix(t):
        assert t.dtype == f32
        return np.rint(t * f32(2.0 ** 30)).astype(np.int64)
    wr = w * res
    raw = []
    for c in range(6):
        wc = w * J[c]
        for rr in range(c, 6):
            raw.append(_exact_sum(fix(wc * J[rr])[inlier]))
    for rr in range(6):
        raw.append(_exact_sum(fix(wr * J[rr])[inlier]))
    raw.append(_exact_sum(fix(wr * res)))
    raw.append(_exact_sum(fix(wr * res)[inlier]))
    return raw + [int(ok.sum()), int((~inlier).sum()), int(invalid.sum())], dict(w=w, inlier=inlier, ok=ok)


@pytest.mark.parametrize("weighting,iteration", [(0, 0), (1, 0), (4, 0), (2, 0), (2, 1), (2, 3), (1, 2)])
def test_weights_and_inlier_tests_at_thresholds(weighting, iteration):
    data, model, outside, kinds = threshold_frames()
    po, pp = _params(H3, W3, weighting=weighting, factor=float(FACTOR), icp_max_distance=float(DIST),
                     icp_max_angle=float(ANGLE))
    want, per = weighted_raw32(data, model, outside, weighting, FACTOR, iteration, DIST, angle_threshold(ANGLE))
    # what the designed pixels must show (the model's decisions, restated from the kernel's rules)
    okidx = np.flatnonzero(per["ok"])
    pos = {i: np.searchsorted(okidx, i) for i in okidx}
    for i, kind in kinds:
        if kind.startswith(("invalid", "outside")):
            assert i not in pos, kind
            continue
        w, inl = per["w"][pos[i]], per["inlier"][pos[i]]
        if kind.startswith("distance"):
            assert inl == (abs(float(kind.split()[1])) <= DIST), kind
        if kind.startswith("normal dot"):
            assert inl == (f32(kind.split()[2]) >= angle_threshold(ANGLE)), kind
        if kind.startswith("residual"):
            x = f32(kind.split()[1])
            if weighting in (1, 4):
                assert w == (f32(1.0) if abs(x) <= FACTOR else FACTOR / abs(x)) and w > 0, (kind, w)
            if weighting == 2 and iteration > 0:
                assert (w == 0) == (abs(x) >= FACTOR), (kind, w)
            if weighting == 0 or (weighting == 2 and iteration == 0):
                assert w == 1, (kind, w)
    assert want[29] + want[31] == H3 * W3 and want[31] == 4 and want[30] > 0
    ctx = api.Context(pp)
    try:
        obj = _frames(ctx, po, data, model)
        obj.initialize(np.eye(4))
        obj.iteration_ = iteration
        obj.jacobianProducts()
        got = [int(x) for x in obj.raw32]
        bad = [i for i in range(32) if got[i] != want[i]]
        assert not bad, "raw sums %s differ: %s vs %s" % (bad, [got[i] for i in bad], [want[i] for i in bad])
        assert (obj.valid(), obj.outlier(), obj.invalid()) == tuple(want[29:32])
        _, raw_o = O.icp_jacobian(po, data, model, np.eye(4), iteration=iteration)
        assert [int(x) for x in raw_o] == want, "oracle"
        if iteration == 0:
            first_step_equal(ctx, po, pp, obj, data, model, want, "weighting %d" % weighting)
    finally:
        ctx.close()


def test_angle_threshold_is_hit_at_equality():
    """the threshold pixel's normal dot is the library's threshold itself: the fp64 cos of 30 degrees rounded once"""
    t = angle_threshold(ANGLE)
    assert t == f32(np.cos(np.float64(30.0) * np.pi / 180.0))
    data, model, _, kinds = threshold_frames()
    dots = [data[1].reshape(-1, 4)[i, 2] for i, k in kinds if k.startswith("normal dot")]
    assert dots == _ulps(t)


# ---------------------------------------------------------------------------------------------------------------
# 4. degenerate scenes through sb_process_scan
# ---------------------------------------------------------------------------------------------------------------
H4, W4 = 32, 360
GROUND = -1.75


def raycast(planes, origin, max_range=70.0):
    """points (float32 [N, 4], sensor frame, no rotation) where the beams through the pixel centres first hit one of the
    planes (normal axis, offset, sign of the side the sensor is on); every point of a plane z = c gets z exactly"""
    d = _beam_centres(H4, W4).reshape(-1, 3)
    best = np.full(d.shape[0], np.inf)
    which = np.full(d.shape[0], -1)
    for j, (axis, c) in enumerate(planes):
        with np.errstate(divide="ignore", invalid="ignore"):
            s = (c - origin[axis]) / d[:, axis]
        hit = (s > 0) & (s < best)
        best[hit] = s[hit]
        which[hit] = j
    keep = best < max_range
    pts = np.ones((int(keep.sum()), 4), f32)
    pts[:, :3] = (d[keep] * best[keep, None]).astype(f32)
    for j, (axis, c) in enumerate(planes):  # on its plane exactly: exact axis-aligned normals in the preprocessing
        pts[which[keep] == j, axis] = f32(c - origin[axis])
    return pts


def _scene(name):
    ground = [(2, GROUND)]
    corridor = [(2, GROUND), (1, 3.0), (1, -3.0)]
    step = lambda t, z=0.0: np.array([0.8 * t, 0.0, z])  # noqa: E731
    if name == "plane":
        return [raycast(ground, step(t)) for t in range(4)]
    if name == "corridor":
        return [raycast(corridor, step(t)) for t in range(4)]
    if name == "empty_scan":
        sc = [raycast(corridor, step(t)) for t in range(4)]
        sc[2] = np.zeros((0, 4), f32)
        return sc
    if name == "beyond_max_depth":
        sc = [raycast(corridor, step(t)) for t in range(4)]
        far = raycast([(0, 200.0), (0, -200.0)], np.zeros(3), max_range=1e9)
        assert np.linalg.norm(far[:, :3], axis=1).min() > 75.0
        sc[2] = far
        return sc
    if name == "jump":  # the sensor drops 0.5 m at scan 3
        return [raycast(ground, step(t, -0.5 if t >= 3 else 0.0)) for t in range(5)]
    raise KeyError(name)


def _run_scene(po, pp, scans, what):
    """_pipeline_equal, then the statistics of both (the context stays open until they are read)"""
    osl, gsl = O.Slam(po), api.SurfelMapping(pp)
    close, gsl.ctx.close = gsl.ctx.close, lambda: None
    try:
        _pipeline_equal(po, pp, scans, what, gsl=gsl, osl=osl)
        return gsl.getStatistics(), osl.stats()
    finally:
        close()


@pytest.mark.parametrize("name", ["plane", "corridor", "empty_scan", "beyond_max_depth", "jump"])
def test_degenerate_scene(name):
    po, pp = both_params(**sized(W4, H4))
    scans = _scene(name)
    sg, so = _run_scene(po, pp, [(s, None, None) for s in scans], name)
    assert sg["track_loss"] == so["track_loss"], name
    if name == "jump":
        assert sg["track_loss"] >= 1, "the jump did not take the track-loss recovery"
    if name == "plane":
        # the first alignment's sums: data normals and rendered model normals are exactly e_z, so the tx, ty and rz
        # columns are exactly zero and the solve meets zero pivots
        o = [O.preprocess(po, s, timestamp=100) for s in scans[:2]]
        ctx = api.Context(pp)
        try:
            om, gm = _model_both(po, ctx, o[0], np.eye(4, dtype=f32))
            fd = api.Frame(ctx, W4, H4)
            fd.upload(o[1])
            obj = api.Frame2Model(ctx)
            obj.setData(fd, gm)
            obj.jacobianProducts()
            _, raw_o = O.icp_jacobian(po, o[1], om, np.eye(4))
            assert np.array_equal(obj.raw32, raw_o)
            _, perm, zero = check_solve(_unpack48(obj.raw32), "plane scene")
            assert sorted(perm[k] for k in zero) == [0, 1, 5], (perm, zero)
        finally:
            ctx.close()
