"""Per-point deskewing (DESIGN.md section 11) on the CPU: the oracle's orc_deskew_points against an independent fp64
numpy restatement of the model, the rolling-shutter scans of synth.py, the deskewing tests on the CPU executor for the
CUDA sources, and the experiment that shows deskewing helps (three oracle runs of one turning sequence)."""
import numpy as np
import pytest

from oracle import deskew as OD
from oracle import oracle as O
from semantic_suma_b200 import synth
from test_cusim import _child

# |orc_deskew_points - fp64 model| <= BOUND * (|p| + |t_M|) per coordinate: a dozen fp32 roundings of terms of size
# |p| and |t_M|, the fp32 rounding of w and t_M, and the pinned fp32 atan2 of the azimuth mode (measured worst: 1.7e-7)
BOUND = 1.0e-6


def model(pts, times, mode, ref, a0, clockwise, M):
    """the deskewing model in fp64: w = log R_M and t_M rounded to fp32 (as the library hands them to the kernel)"""
    p = pts[:, :3].astype(np.float64)
    w = synth.so3_log(M[:3, :3]).astype(np.float32).astype(np.float64)
    t = M[:3, 3].astype(np.float32).astype(np.float64)
    if mode == 1:
        s = times.astype(np.float64)
        s = np.where(np.isfinite(s), np.clip(s, 0.0, 1.0), ref)
    else:
        yaw = np.arctan2(p[:, 1], p[:, 0])
        u = (a0 - yaw) if clockwise else (yaw - a0)
        s = np.mod(u / (2 * np.pi), 1.0)
    tau = s - np.float64(np.float32(ref))
    R = synth.so3_exp(tau[:, None] * w)
    return np.einsum("nij,nj->ni", R, p) + tau[:, None] * t, s


def random_motion(rng, deg=30.0, m=3.0):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    T = np.eye(4)
    T[:3, :3] = synth.so3_exp(np.deg2rad(rng.uniform(-deg, deg)) * axis)
    T[:3, 3] = rng.uniform(-m, m, 3)
    return T


@pytest.mark.parametrize("mode", [1, 2], ids=["times", "azimuth"])
@pytest.mark.parametrize("clockwise", [True, False], ids=["clockwise", "counter-clockwise"])
def test_oracle_deskew_equals_the_fp64_model(mode, clockwise):
    rng = np.random.default_rng(11 * mode + clockwise)
    n = 20000
    pts = np.ones((n, 4), np.float32)
    pts[:, :3] = rng.uniform(-60, 60, (n, 3))
    pts[:, 3] = rng.uniform(0, 2, n)  # w is carried through
    times = rng.uniform(-0.2, 1.2, n).astype(np.float32)  # some clamped
    times[::50] = np.nan
    times[1::70] = np.inf
    worst = 0.0
    for _ in range(12):
        M = random_motion(rng)
        ref, a0 = float(np.float32(rng.uniform(0, 1))), float(np.float32(rng.uniform(-4, 4)))
        got = OD.deskew_points(pts, times, mode=mode, ref_time=ref, start_azimuth=a0, clockwise=clockwise, motion=M)
        want, s = model(pts, times, mode, ref, a0, clockwise, M)
        assert got[:, 3].tobytes() == pts[:, 3].tobytes()
        ok = np.ones(n, bool) if mode == 1 else np.minimum(s, 1.0 - s) > 1e-5  # the azimuth seam wraps s
        scale = np.linalg.norm(pts[:, :3].astype(np.float64), axis=1) + np.linalg.norm(M[:3, 3])
        err = np.abs(got[:, :3].astype(np.float64) - want).max(axis=1)[ok] / scale[ok]
        worst = max(worst, float(err.max()))
        # the points did move by about what the motion says
        assert np.abs(got[:, :3] - pts[:, :3]).max() > 0.5
    print("worst |error| / (|p| + |t_M|): %.3g" % worst)
    assert worst <= BOUND, worst


def test_zero_motion_and_reference_time_keep_the_bits():
    rng = np.random.default_rng(5)
    pts = rng.uniform(-30, 30, (1000, 4)).astype(np.float32)
    pts[:10, 1] = -0.0
    M = random_motion(rng)
    for kw in (dict(mode=1, times=np.full(1000, 0.3, np.float32), ref_time=0.3, motion=M),
               dict(mode=2, motion=np.eye(4)), dict(mode=2, motion=None), dict(mode=0, motion=M)):
        assert OD.deskew_points(pts, **kw).tobytes() == pts.tobytes()


def test_rolling_shutter_scan_deskews_to_the_plain_scan():
    """synth's rolling-shutter scan moved back with the true increment is the plain scan up to fp32 round-off; the
    plain output of the same seed is unchanged by the option"""
    sc = synth.Scene(width=900, height=64)
    poses = synth.trajectory(3, step=1.5, yaw_deg=2.0)
    inc = synth.translate(1.5, 0, 0) @ synth.rot_z(np.deg2rad(2.0))
    plain, _, _ = sc.scan(2, poses[2])
    rolled, _, _, s = sc.scan(2, poses[2], rolling=inc)
    assert s.min() > 0 and s.max() < 1 and len(s) == len(rolled)
    back = OD.deskew_points(rolled, s, mode=1, ref_time=0.5, motion=inc)
    moved = np.linalg.norm(rolled[:, :3] - back[:, :3], axis=1)
    assert moved.max() > 0.5  # the sweep's ends are ~0.75 m from the reference time
    assert abs(len(rolled) - len(plain)) < 0.05 * len(plain)


def test_deskewing_on_the_cpu_executor():
    """the -m gpu deskewing tests on tests/cusim: operator parity at an uneven shape, zero motion, launch counts, scan 0,
    whole 64x900 runs in both modes, paging, checkpoints and refusals, bit for bit against the oracle"""
    k = ("37x333 or zero_motion or launches or first_scan or (900 and geometric) or paging or checkpoint or refusals")
    assert _child(["tests/test_gpu_deskew.py"], k) >= 12


# ---- does it help? ---------------------------------------------------------------------------------------------------
# One turning sequence at 15 m/s and 20 deg/s sampled at 10 Hz (1.5 m and 2 deg per sweep), 40 scans at 64x900, run
# through the oracle three times: (a) unskewed scans, deskewing off; (b) rolling-shutter scans, off; (c) rolling-shutter
# scans, azimuth deskewing. Measured (DESIGN.md section 11): translational error a 0.51 %, b 1.02 %, c 0.68 %; end-point error a 0.37 m,
# b 0.74 m, c 0.41 m. The margins below sit between those values.
STEP, YAW, N = 1.5, 2.0, 40


def drift(est, gt):
    """(mean relative translational error in % over 10 / 20 / 30 / 40 m segments, as the KITTI devkit forms it, end-point
    error in m)"""
    rel = [np.linalg.inv(gt[0]) @ g for g in gt]
    d = np.concatenate([[0], np.cumsum([np.linalg.norm(rel[i + 1][:3, 3] - rel[i][:3, 3]) for i in range(len(gt) - 1)])])
    errs = []
    for L in (10.0, 20.0, 30.0, 40.0):
        for i in range(len(gt)):
            j = int(np.searchsorted(d, d[i] + L))
            if j >= len(gt):
                break
            E = np.linalg.inv(np.linalg.inv(rel[i]) @ rel[j]) @ (np.linalg.inv(est[i]) @ est[j])
            errs.append(np.linalg.norm(E[:3, 3]) / L)
    return 100.0 * float(np.mean(errs)), float(np.linalg.norm(est[-1][:3, 3] - rel[-1][:3, 3]))


def oracle_run(rolling, mode):
    inc = synth.translate(STEP, 0, 0) @ synth.rot_z(np.deg2rad(YAW))
    gt = synth.trajectory(N, step=STEP, yaw_deg=YAW)
    sc = synth.Scene(width=900, height=64)
    s = OD.Slam(O.default_params(data_width=900, model_width=900))
    s.set_deskew(mode)
    est = []
    for f in range(N):
        out = sc.scan(f, gt[f], rolling=inc if rolling else None)
        s.process_scan(out[0])
        est.append(s.pose())
    return drift(est, gt)


def test_deskewing_helps_on_a_turning_sequence():
    a, b, c = oracle_run(False, 0), oracle_run(True, 0), oracle_run(True, 2)
    print("translational error %% / end-point error m: a %s b %s c %s" % (a, b, c))
    for k in (0, 1):
        assert c[k] < 0.75 * b[k], (a, b, c)       # clearly better than without deskewing
        assert c[k] < a[k] + 0.5 * (b[k] - a[k]), (a, b, c)  # and closer to the unskewed run than to the skewed one
