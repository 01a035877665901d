"""Seeded synthetic LiDAR scans (SURVEY.md section 8d): a ground plane plus the 23 boxes of the reference's
SimulationReader world (io/SimulationReader.cpp:68-98), ray-cast from a sensor 2 m above ground that moves
1.0 m forward + 0.5 deg yaw per frame. Pure numpy; this is input generation, not part of the timed path.
"""
import numpy as np

# (x, y, z, yaw_deg, size) -- io/SimulationReader.cpp:72-98
_BOXES = [
    (10, 10, 0.5, 0.0, 1.0), (112, -15, 1.25, 45.0, 2.5), (34, 20, 0.75, 0.0, 1.5), (50, -10, 0.75, 79.0, 1.5),
    (65, 5, 0.75, 45.0, 1.5), (70, -15, 0.85, 25.0, 1.5), (100, 30, 0.65, 0.0, 1.5), (120, -10, 0.65, 25.0, 1.5),
    (170, -10, 0.65, 15.0, 1.5), (190, -30, 0.65, 35.0, 1.5), (230, 15, 0.65, 5.0, 3.5), (270, -7, 0.65, -3.5, 2.5),
    (280, 20, 0.65, 2.0, 4.5), (320, 20, 0.65, 2.0, 4.5), (370, 10, 0.65, 15.0, 1.5), (390, -30, 0.65, 35.0, 1.5),
    (430, -15, 0.65, 5.0, 3.5), (470, 7, 0.65, -3.5, 2.5), (480, 20, 0.65, 2.0, 4.5), (40, -20, 0.65, 15.0, 3.0),
    (50, -75, 5.0, 25.0, 10.0), (-20, -54, 0.65, 15.0, 4.5),
    (20, -6, 0.75, 10.0, 1.5),  # 23rd object: a car-sized box close to the lane (semantic configs label it "car")
]


def _street(n=64, seed=7):
    """A 'street canyon' of building-sized boxes on both sides of the lane so that projective ICP is well
    conditioned along the driving direction (the SimulationReader world alone is almost a bare plane)."""
    r = np.random.default_rng(seed)
    out = []
    for k in range(n):
        side = 1.0 if k % 2 == 0 else -1.0
        x = -60.0 + 9.0 * (k // 2) + r.uniform(-2, 2)
        size = r.uniform(5.0, 9.0)
        y = side * (r.uniform(11.0, 22.0) + 0.5 * size)
        out.append((x, y, 0.5 * size - 0.2, r.uniform(-30, 30), size))
    return out


_BOXES = _BOXES + _street()
_CAR_BOXES = (0, 2, 3, 4, 19, 22)   # labelled car (10) in the semantic configuration
_MOVING = (3, 22)                   # two of them move 0.5 m / frame along +x


def rot_z(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float64)


def so3_log(R):
    """axis-angle of a rotation matrix (fp64)"""
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    sv = np.linalg.norm(v)
    return np.zeros(3) if sv == 0.0 else np.arctan2(0.5 * sv, 0.5 * (np.trace(R) - 1.0)) / sv * v


def so3_exp(w):
    """rotation matrices of axis-angle vectors w[..., 3] (Rodrigues, fp64)"""
    w = np.asarray(w, np.float64)
    th = np.linalg.norm(w, axis=-1)[..., None, None]
    K = np.zeros(w.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -w[..., 2], w[..., 1], -w[..., 0]
    K[..., 1, 0], K[..., 2, 0], K[..., 2, 1] = w[..., 2], -w[..., 1], w[..., 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.where(th > 0, np.sin(th) / th, 1.0)
        b = np.where(th > 0, (1.0 - np.cos(th)) / (th * th), 0.5)
    return np.eye(3) + a * K + b * (K @ K)


def translate(x, y, z):
    T = np.eye(4)
    T[:3, 3] = (x, y, z)
    return T


def trajectory(n_frames, step=1.0, yaw_deg=0.5):
    """Ground-truth sensor poses (world <- sensor), frame 0 at (0,0,2)."""
    T = translate(0, 0, 2.0)
    out = [T.copy()]
    inc = translate(step, 0, 0) @ rot_z(np.deg2rad(yaw_deg))
    for _ in range(n_frames - 1):
        T = T @ inc
        out.append(T.copy())
    return out


class Scene:
    def __init__(self, width=2048, height=64, fov_up=3.0, fov_down=-25.0, min_range=2.0, max_range=75.0,
                 sigma=0.02, angle_jitter_px=0.25, seed=1337, semantic=False):
        self.W, self.H = width, height
        self.fov_up, self.fov_down = fov_up, fov_down
        self.min_range, self.max_range = min_range, max_range
        self.sigma, self.jit, self.seed, self.semantic = sigma, angle_jitter_px, seed, semantic
        fov = abs(fov_up) + abs(fov_down)
        # beam centres aim at pixel centres of the reference's projection (gen_vertexmap.vert:78-89)
        k = np.arange(width) + 0.5
        r = np.arange(height) + 0.5
        self.az = np.pi * (1.0 - 2.0 * k / width)                     # yaw of column k
        self.el = np.deg2rad(abs(fov_up) - fov * (1.0 - r / height))  # elevation of row r (row 0 = lowest)
        self.daz = 2.0 * np.pi / width
        self.delv = np.deg2rad(fov) / height

    def scan(self, frame, pose=None, rolling=None, ref_time=0.5, clean_labels=False):
        """Returns (pts[N,4] float32 (x,y,z,1) in the sensor frame, labels[N] float32, probs[N] float32).
        Point order: azimuth-major, beams inner (as io/SimulationReader.cpp:103-116 builds its beam table).

        rolling (a 4x4 per-frame increment, the sensor's true motion over one sweep): a rolling-shutter scan. Column k
        is measured at sweep time s_k = (k + 0.5) / W (column 0 first, as a clockwise spin starting at yaw +pi) from
        pose . D(s_k), D(s) = (Exp((s - ref_time) w), (s - ref_time) t) with (w, t) = (log R, t) of the increment; the
        points come back in that instantaneous sensor frame and a fourth array holds their s_k. The same seed gives the
        same noise and, with rolling=None, exactly the output of a plain scan.

        clean_labels (semantic scenes): one more array at the end, the labels before the 2 % random flips; every other
        output is unchanged."""
        rng = np.random.default_rng(self.seed + frame)
        if pose is None:
            pose = trajectory(frame + 1)[-1]
        W, H = self.W, self.H
        az = np.repeat(self.az, H) + rng.normal(0, self.jit, W * H) * self.daz
        el = np.tile(self.el, W) + rng.normal(0, self.jit, W * H) * self.delv
        ds = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1)
        R, o = pose[:3, :3], pose[:3, 3]
        margin = 0.0
        if rolling is None:
            d = ds @ R.T
        else:
            times = np.repeat((np.arange(W) + 0.5) / W, H)
            tau = times - ref_time
            w, t = so3_log(np.asarray(rolling)[:3, :3]), np.asarray(rolling)[:3, 3]
            Rk = R @ so3_exp(tau[:, None] * w)           # world <- instantaneous sensor, per point
            d = np.einsum("nij,nj->ni", Rk, ds)
            o_center = o
            o = o + (tau[:, None] * t) @ R.T
            margin = float(np.linalg.norm(t))
        o_c = o if rolling is None else o_center
        t_best = np.full(W * H, np.inf)
        hit = np.full(W * H, -1, np.int32)  # -1 none, 0 ground, 1+b box b
        with np.errstate(divide="ignore", invalid="ignore"):
            tg = -o[..., 2] / d[:, 2]
        m = (d[:, 2] < 0) & (tg > 0)
        t_best[m] = tg[m]
        hit[m] = 0
        for b, (bx, by, bz, yaw, size) in enumerate(_BOXES):
            if b in _MOVING:
                bx = bx + 0.5 * frame
            if (bx - o_c[0]) ** 2 + (by - o_c[1]) ** 2 > (self.max_range + size + margin) ** 2:
                continue
            Rb = rot_z(np.deg2rad(yaw))[:3, :3]
            ob = (o - np.array([bx, by, bz])) @ Rb
            db = d @ Rb
            h = 0.5 * size
            with np.errstate(divide="ignore", invalid="ignore"):
                t1 = (-h - ob) / db
                t2 = (h - ob) / db
            tmin = np.nanmax(np.minimum(t1, t2), axis=1)
            tmax = np.nanmin(np.maximum(t1, t2), axis=1)
            ok = (tmax >= tmin) & (tmin > 0) & (tmin < t_best)
            t_best[ok] = tmin[ok]
            hit[ok] = 1 + b
        rngs = t_best + rng.normal(0, self.sigma, W * H)
        keep = (hit >= 0) & (rngs >= self.min_range) & (rngs < self.max_range) & np.isfinite(rngs)
        pts = np.ones((int(keep.sum()), 4), np.float32)
        pts[:, :3] = (ds[keep] * rngs[keep, None]).astype(np.float32)
        extra = () if rolling is None else (times[keep].astype(np.float32),)
        if not self.semantic:
            return (pts, None, None) + extra
        hk = hit[keep]
        labels = np.where(hk == 0, 40.0, 50.0).astype(np.float32)
        for b in _CAR_BOXES:
            labels[hk == 1 + b] = 10.0
        clean = labels.copy()
        flips = rng.random(labels.shape[0]) < 0.02
        labels[flips] = rng.choice(np.array([10.0, 40.0, 50.0, 70.0, 30.0], np.float32), int(flips.sum()))
        probs = rng.uniform(0.6, 1.0, labels.shape[0]).astype(np.float32)
        return (pts, labels, probs) + extra + ((clean,) if clean_labels else ())


def make_sequence(n_frames, **kw):
    sc = Scene(**kw)
    poses = trajectory(n_frames)
    return [sc.scan(f, poses[f]) for f in range(n_frames)], poses
