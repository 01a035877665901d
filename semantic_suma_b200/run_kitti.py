"""Run the hot path over a KITTI-odometry-style sequence directory and write / evaluate the trajectory
(SURVEY.md 8f-4: the callers and data formats on either side of `SurfelMapping::processScan`).

    <seq>/velodyne/000000.bin ...      scans (N x 4 float32)                     io/KITTIReader.cpp:40-62, 136-170
    <seq>/labels/000000.label ...      optional per-point class ids (stand-in for the RangeNet++ call, :172-203)
    <seq>/calib.txt                    optional; "Tr" moves the exported poses to the camera frame
    <seq>/poses.txt                    optional ground truth (camera frame if calib.txt has Tr) -> odometry errors

    python -m semantic_suma_b200.run_kitti <seq> [--out poses_out.txt] [--semantic] [--max-scans N] [--width 2048]
    python -m semantic_suma_b200.run_kitti --make-synthetic <dir> --scans 50     # writes such a directory

Long runs can be checkpointed and resumed (sb_state_save / sb_state_load): --save-state PATH writes the library's state
to PATH and the trajectory so far to PATH.poses.npy, after every --save-every N scans and at the end of the run;
--resume PATH continues at the scan after the saved one. The pose file of a resumed run is byte-identical to the one of
an uninterrupted run.

Full sequences extract more submap tiles than the default HBM tile cache holds: --tile-cache-host N turns on the managed
cache (sb_set_tile_cache) with up to N surfels in pinned host memory (inf: no bound, as the reference's cache; 0: the
default cache). The run then prints the cache's counters.

--write-labels DIR (with --semantic) writes DIR/NNNNNN.label per scan in the SemanticKITTI format: one uint32 per input
point, the label the fused map gives the point in the low 16 bits (0, unlabeled, where the map has no surfel at the
point's pixel) and instance 0 (sb_get_point_labels; DESIGN.md section 13). A resumed run writes the files from the scan
after the checkpoint on, byte-identical to those of an uninterrupted run.

The engine is the CUDA library (an H100 is required); tests inject another engine through `make_engine` to check the
file plumbing without a GPU.
"""
import argparse
import glob
import json
import os
import sys
import time

import numpy as np

from . import kitti


def list_scans(seq_dir):
    return sorted(glob.glob(os.path.join(seq_dir, "velodyne", "*.bin")))


def _cuda_engine(params):
    from . import api
    return api.SurfelMapping(params)


def trajectory_path(state_path):
    return state_path + ".poses.npy"


def write_checkpoint(engine, state_path, poses):
    """the engine's state to `state_path`, the poses so far beside it; each file is replaced only once it is complete,
    the trajectory last, so that an interrupted save leaves the previous checkpoint readable"""
    blob = engine.save_state()
    tmp = state_path + ".tmp"
    with open(tmp, "wb") as f:
        f.write(blob)
    os.replace(tmp, state_path)
    tmp = trajectory_path(state_path) + ".tmp.npy"
    np.save(tmp, np.asarray(poses, np.float64).reshape(-1, 4, 4))
    os.replace(tmp, trajectory_path(state_path))


def read_checkpoint(engine, state_path):
    """loads `state_path` into the engine; -> the poses saved with it (one per scan already processed)"""
    with open(state_path, "rb") as f:
        engine.load_state(f.read())
    poses = [p.copy() for p in np.load(trajectory_path(state_path))]
    if engine.timestamp() != len(poses):
        raise ValueError("%s holds %d scans but its trajectory %d poses" % (state_path, engine.timestamp(), len(poses)))
    return poses


def parse_host_surfels(text):
    """--tile-cache-host: a surfel count, or inf for no bound"""
    if text.strip().lower() in ("inf", "infinity"):
        return float("inf")
    n = int(text)
    if n < 0:
        raise ValueError("--tile-cache-host must be >= 0 or inf")
    return n


TILE_POOL_SURFELS = 16 * 1024 * 1024  # the HBM share of a managed tile cache: the whole pool
POINT_MAP = 8  # sb_point_label flag: the model frame has a surfel at the point's pixel


def map_label_ids(records):
    """the SemanticKITTI id of every point of a scan: the map's label where it has one, 0 (unlabeled) elsewhere"""
    return np.where(records["flags"] & POINT_MAP, records["map_label"], 0).astype(np.uint32)


def run_sequence(seq_dir, params, make_engine=None, semantic=False, max_scans=None, on_scan=None, save_state=None,
                 save_every=None, resume=None, tile_cache_host=0, deskew="off", write_labels=None):
    """-> dict(poses=[4x4 float64 in the velodyne frame, from scan 0], seconds, scans processed by this call, and
    tile_cache: the cache's counters when tile_cache_host is set).
    `make_engine(params)` must return an object with processScan(points4, labels, probs) and getCurrentPose() -- the
    SurfelMapping surface -- and, for save_state / resume, save_state(), load_state(bytes) and timestamp(); for
    tile_cache_host, setTileCache(pool, host) and tile_cache_info().
    resume: a checkpoint written by save_state; the run continues at the scan after it (with the cache it was saved with).
    tile_cache_host: surfels the managed tile cache may keep in host memory (inf: no bound; 0: the default cache).
    deskew: "off" or "azimuth" (per-point deskewing by each point's azimuth, setDeskew); a resumed run keeps the setting
    of its checkpoint.
    write_labels: a directory for one SemanticKITTI .label file per scan from the map's labels (map_label_ids); the
    engine then needs setPointLabels(on) and getPointLabels() (records with the fields of sb_point_label)."""
    files = list_scans(seq_dir)
    if max_scans is not None:
        files = files[:max_scans]
    if not files:
        raise FileNotFoundError("no scans under %s/velodyne" % seq_dir)
    engine = (make_engine or _cuda_engine)(params)
    if tile_cache_host:
        engine.setTileCache(TILE_POOL_SURFELS, tile_cache_host)
    if deskew != "off":
        engine.setDeskew(deskew)
    if write_labels:
        os.makedirs(write_labels, exist_ok=True)
        engine.setPointLabels(True)
    poses = read_checkpoint(engine, resume) if resume else []
    first = len(poses)
    if first > len(files):
        raise ValueError("%s is past the end of the sequence (%d scans)" % (resume, len(files)))
    t0 = time.time()
    for i, f in enumerate(files):
        if i < first:
            continue
        pts, _ = kitti.read_scan(f)
        labels = probs = None
        if semantic:
            lf = os.path.join(seq_dir, "labels", os.path.splitext(os.path.basename(f))[0] + ".label")
            labels, probs = kitti.read_labels(lf, n_points=pts.shape[0])
        engine.processScan(pts, labels, probs)
        if write_labels:
            name = os.path.splitext(os.path.basename(f))[0] + ".label"
            kitti.write_labels(os.path.join(write_labels, name), map_label_ids(engine.getPointLabels()))
        poses.append(np.asarray(engine.getCurrentPose(), np.float64).copy())
        if on_scan:
            on_scan(i, poses[-1])
        if save_state and save_every and (i + 1) % save_every == 0 and i + 1 < len(files):
            write_checkpoint(engine, save_state, poses)
    if save_state:
        write_checkpoint(engine, save_state, poses)
    out = {"poses": poses, "seconds": time.time() - t0, "scans": len(files) - first}
    if tile_cache_host:
        out["tile_cache"] = engine.tile_cache_info()
    return out


def evaluate_against_ground_truth(seq_dir, poses_velo):
    """odometry errors of `poses_velo` against <seq>/poses.txt, in the frame that file uses (camera if calib has Tr)"""
    gt_file = os.path.join(seq_dir, "poses.txt")
    if not os.path.exists(gt_file):
        return None
    gt = kitti.load_poses(gt_file)[:len(poses_velo)]
    calib_file = os.path.join(seq_dir, "calib.txt")
    Tr = kitti.read_calibration(calib_file).get("Tr") if os.path.exists(calib_file) else None
    est = [np.asarray(p, np.float32) for p in poses_velo]
    if Tr is not None:
        est = kitti.poses_to_camera_frame(est, Tr)
    # both trajectories start at identity in the devkit's convention
    g0, e0 = np.linalg.inv(gt[0]), np.linalg.inv(est[0])
    gt = [(g0 @ g).astype(np.float32) for g in gt]
    est = [(e0 @ e).astype(np.float32) for e in est]
    out = kitti.evaluate(gt, est[:len(gt)])
    out["end_point_error_m"] = float(np.linalg.norm(gt[-1][:3, 3] - est[len(gt) - 1][:3, 3]))
    return out


def make_synthetic_sequence(seq_dir, n_scans, width=2048, height=64, semantic=False, seed=1337):
    """writes a synthetic sequence (semantic_suma_b200/synth.py scene) in the KITTI layout, with calib.txt (the usual
    velodyne -> camera axis change) and ground-truth poses in the camera frame"""
    from . import synth
    os.makedirs(os.path.join(seq_dir, "velodyne"), exist_ok=True)
    if semantic:
        os.makedirs(os.path.join(seq_dir, "labels"), exist_ok=True)
    Tr = np.array([[0, -1, 0, 0], [0, 0, -1, 0], [1, 0, 0, 0], [0, 0, 0, 1]], np.float32)
    with open(os.path.join(seq_dir, "calib.txt"), "w") as f:
        f.write("Tr: " + " ".join(repr(float(x)) for x in Tr[:3].reshape(-1)) + "\n")
    sc = synth.Scene(width=width, height=height, seed=seed, semantic=semantic)
    poses = synth.trajectory(n_scans)
    for i in range(n_scans):
        pts, labels, _ = sc.scan(i, poses[i])
        kitti.write_scan(os.path.join(seq_dir, "velodyne", "%06d.bin" % i), pts[:, :3], np.full(pts.shape[0], 0.5))
        if semantic:
            kitti.write_labels(os.path.join(seq_dir, "labels", "%06d.label" % i), labels.astype(np.uint32))
    rel = [np.linalg.inv(poses[0]) @ p for p in poses]          # start at identity
    kitti.save_poses(os.path.join(seq_dir, "poses.txt"), rel, Tr=Tr)
    return seq_dir


def main(argv=None, make_engine=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("seq", nargs="?")
    ap.add_argument("--out", default=None, help="pose file to write (KITTI format; camera frame if calib.txt has Tr)")
    ap.add_argument("--semantic", action="store_true")
    ap.add_argument("--max-scans", type=int, default=None)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--make-synthetic", default=None, metavar="DIR")
    ap.add_argument("--scans", type=int, default=50)
    ap.add_argument("--save-state", default=None, metavar="PATH",
                    help="checkpoint file (and PATH.poses.npy): written at the end and every --save-every scans")
    ap.add_argument("--save-every", type=int, default=None, metavar="N")
    ap.add_argument("--resume", default=None, metavar="PATH", help="continue from a --save-state checkpoint")
    ap.add_argument("--tile-cache-host", type=parse_host_surfels, default=0, metavar="N",
                    help="managed submap tile cache with up to N surfels in host memory (inf: no bound; 0: default cache)")
    ap.add_argument("--deskew", choices=("off", "azimuth"), default="off",
                    help="per-point deskewing by azimuth (off for KITTI odometry, whose scans are treated as already "
                         "motion-compensated)")
    ap.add_argument("--write-labels", default=None, metavar="DIR",
                    help="write DIR/NNNNNN.label per scan: the fused map's label of every point (needs --semantic)")
    args = ap.parse_args(argv)
    if args.save_every is not None and (args.save_every <= 0 or not args.save_state):
        ap.error("--save-every needs --save-state and N > 0")
    if args.write_labels and not args.semantic:
        ap.error("--write-labels needs --semantic")
    if args.make_synthetic:
        make_synthetic_sequence(args.make_synthetic, args.scans, width=args.width, semantic=args.semantic)
        print("wrote", args.make_synthetic)
        if not args.seq:
            return 0
    if not args.seq:
        ap.error("need a sequence directory")
    from . import api
    params = api.default_params(data_width=args.width, model_width=args.width)
    res = run_sequence(args.seq, params, make_engine=make_engine, semantic=args.semantic, max_scans=args.max_scans,
                       save_state=args.save_state, save_every=args.save_every, resume=args.resume,
                       tile_cache_host=args.tile_cache_host, deskew=args.deskew, write_labels=args.write_labels)
    calib_file = os.path.join(args.seq, "calib.txt")
    Tr = kitti.read_calibration(calib_file).get("Tr") if os.path.exists(calib_file) else None
    if args.out:
        kitti.save_poses(args.out, res["poses"], Tr=Tr)
    report = {"scans": res["scans"], "seconds": round(res["seconds"], 3),
              "scans_per_sec_incl_file_io": round(res["scans"] / res["seconds"], 2) if res["seconds"] > 0 else None,
              "odometry": evaluate_against_ground_truth(args.seq, res["poses"])}
    if "tile_cache" in res:
        report["tile_cache"] = res["tile_cache"]
    print(json.dumps(report))
    return 0


if __name__ == "__main__":
    sys.exit(main())
