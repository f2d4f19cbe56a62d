"""Time resection on the GPU over a scene of bench.py's C4 size: cube_scene(500, 200000, max_obs_per_point=10), its
true tracks, half the shots reconstructed at their true poses with every point at its true position, all other shots
as candidates with 20 % of their observations moved to random positions.  Bearings come from a distortion-free
pinhole camera over the normalised image coordinates.

    python tools/measure_resection.py [--reps 5] [--oracle-shots 4]

Prints one JSON line: the card's name and power limit (read in the same run), the workload (candidates, rows), and
  * `kernel_ms`: the device time of the resection kernels (CUDA events), median of --reps;
  * `host_ms`: resect_candidates' host clock by part (bearings, packing, device_call, map_writes), medians;
  * `oracle_ms_per_shot`: oracle/absolute_pose_oracle.py (numpy, one CPU core) on --oracle-shots candidates, for
    scale only; pyrobust itself is not measured.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


class PinholeCamera:
    id = "cam"

    def pixel_bearing_many(self, p):
        p = np.asarray(p, dtype=np.float64).reshape(-1, 2)
        b = np.column_stack([p, np.ones(len(p))])
        return b / np.sqrt((b * b).sum(axis=1))[:, None]


class Dataset:
    config = {"use_altitude_tag": True}

    def load_exif(self, image):
        return {"camera": "cam"}

    def load_rig_assignments(self):
        return {}


def build(cameras, points, seed=42, outliers=0.2):
    from opensfm_b200 import map_types as M
    from opensfm_b200 import synthetic as syn
    from opensfm_b200 import tracking
    from opensfm_b200 import types as T

    sc = syn.cube_scene(cameras, points, with_descriptors=False, max_obs_per_point=10)
    rng = np.random.RandomState(seed)
    order = np.lexsort((sc.obs_shot, sc.obs_point))
    pts, shots = sc.obs_point[order], sc.obs_shot[order]
    keep = np.isin(pts, np.nonzero(np.bincount(pts, minlength=points) >= 2)[0])
    pts, shots = pts[keep], shots[keep].astype(np.int32)
    images = ["im%04d" % s for s in range(cameras)]
    reconstructed = cameras // 2
    pc = np.einsum("nij,nj->ni", sc.R_wc[shots], sc.points[pts] - sc.origins[shots])
    xy = pc[:, :2] / pc[:, 2:3]
    moved = (rng.rand(len(xy)) < outliers) & (shots >= reconstructed)
    xy[moved] = rng.uniform(-0.5, 0.5, (int(moved.sum()), 2))
    by_shot = np.argsort(shots, kind="stable")
    start = np.searchsorted(shots[by_shot], np.arange(cameras + 1))
    feature = np.zeros(len(pts), dtype=np.int32)
    feats = {}
    for s in range(cameras):
        rows = by_shot[start[s]:start[s + 1]]
        feature[rows] = np.arange(len(rows))
        feats[images[s]] = np.column_stack([xy[rows], np.full(len(rows), 0.004)])
    colors = {im: np.zeros((len(f), 3), dtype=np.int32) for im, f in feats.items()}
    track = np.searchsorted(np.unique(pts), pts).astype(np.int32)
    track_start = np.searchsorted(track, np.arange(track.max() + 2)).astype(np.int64)
    tm = tracking.TracksManager(None, images, track, shots, feature, track_start, feats, colors, {}, {}, None, True,
                                1.0, 0.0)
    rec = M.Reconstruction()
    rec.add_camera(PinholeCamera())
    for s in range(reconstructed):
        pose = T.Pose()
        pose.set_rotation_matrix(sc.R_wc[s])
        pose.set_origin(sc.origins[s])
        rec.create_shot(images[s], "cam", pose)
    seen = np.unique(track[shots < reconstructed])
    point_of_track = np.unique(pts)
    ids = tm._track_ids()
    for t in seen.tolist():
        rec.create_point(ids[t], sc.points[point_of_track[t]])
    return tm, rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-shots", type=int, default=4)
    ap.add_argument("--cameras", type=int, default=500)
    ap.add_argument("--points", type=int, default=200000)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("measure_resection.py needs a CUDA device")
    from measure_tracks import card

    from opensfm_b200 import reconstruction as rec
    from oracle import absolute_pose_oracle as apo

    info = card()
    tm, r = build(args.cameras, args.points)
    data = Dataset()
    candidates = rec.reconstructed_points_for_images(tm, r, set(tm.images))
    # min_inliers above every count: nothing is added, so every repetition resects the same candidates
    never = 10 ** 9
    times = []
    for _ in range(args.reps + 1):
        _, _, _, reports = rec.resect_candidates(data, tm, r, candidates, 0.004, never)
        times.append(rec.last_resect_times())
    times = times[1:]
    med = {k: float(np.median([t[k] for t in times])) for k in times[0]}
    rows = int(sum(rep["num_common_points"] for rep in reports))

    order, start = tm._shot_order()
    xy = tm._points()[0]
    cam = PinholeCamera()
    ms = []
    index = {im: i for i, im in enumerate(tm.images)}
    for im, _ in candidates[:: max(1, len(candidates) // max(1, args.oracle_shots))][:args.oracle_shots]:
        rows_i = order[start[index[im]]:start[index[im] + 1]]
        rows_i = rows_i[np.array([tm._track_ids()[t] in r.points for t in tm.obs_track[rows_i]], dtype=bool)]
        X = np.array([r.points[tm._track_ids()[t]].coordinates for t in tm.obs_track[rows_i]])
        t0 = time.perf_counter()
        apo.ransac_absolute_pose(cam.pixel_bearing_many(xy[rows_i]), X, 0.004)
        ms.append(1e3 * (time.perf_counter() - t0))
    print(json.dumps({
        "card": info, "candidates": len(candidates), "rows": rows,
        "kernel_ms": med["device_ms"],
        "host_ms": {k: 1e3 * med[k] for k in ("bearings", "packing", "device_call", "map_writes")},
        "succeeded_at_min_inliers_10": int(sum(rep.get("num_inliers", 0) >= 10 for rep in reports)),
        "oracle_ms_per_shot": float(np.median(ms)) if ms else None,
        "reps": args.reps}))


if __name__ == "__main__":
    main()
