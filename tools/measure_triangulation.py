"""Time track triangulation on the GPU over the tracks of tools/measure_tracks.py: cube_scene(500, 200000,
max_obs_per_point=10), every pair of shots sharing at least --min-shared points matched on exactly those points, every
shot in the reconstruction at its true pose.

    python tools/measure_triangulation.py [--reps 3] [--oracle-tracks 2000]

Prints one JSON line: the card's name and power limit (read in the same run), the sizes, the statuses, and
  * `kernel_ms`: CUDA events around tri_tracks on the tracks handle's stream (after the uploads), median of --reps
    calls of the bulk form;
  * `bulk_ms`: host clock around TracksManager.triangulate (upload of the per-image arrays and the bearings, kernel,
    download of X and status; the call ends in a stream synchronise);
  * `retriangulate_ms`: host clock around triangulation.retriangulate, and its parts: `bearings` (pixel_bearing_many
    once per image), `device_call` (the bulk form) and `write` (create_point / add_observation into the map);
  * `oracle_ms_per_1000_tracks`: oracle/triangulation_oracle.py (numpy, one track at a time, on the CPU) over the
    first --oracle-tracks selected tracks, for scale.
The reference's own time (pygeometry's midpoint and TinySolver behind a Python loop) is not measured: pygeometry cannot
be built without Eigen and Ceres.
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


class DistortedPerspective:
    """pixel_bearing_many of cube_scene's camera (perspective, k1 / k2 radial distortion): the radius undistorted by
    Newton's method."""

    def __init__(self, k1: float, k2: float, focal: float):
        self.k1, self.k2, self.focal, self.id = k1, k2, focal, "cube"

    def pixel_bearing_many(self, p):
        d = np.asarray(p, dtype=np.float64).reshape(-1, 2) / self.focal
        rd = np.linalg.norm(d, axis=1)
        r = rd.copy()
        for _ in range(20):
            r2 = r * r
            f = r * (1 + self.k1 * r2 + self.k2 * r2 * r2) - rd
            r -= f / (1 + 3 * self.k1 * r2 + 5 * self.k2 * r2 * r2)
        scale = np.where(rd > 0, r / np.where(rd > 0, rd, 1.0), 1.0)
        b = np.column_stack([d * scale[:, None], np.ones(len(d))])
        return b / np.linalg.norm(b, axis=1)[:, None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--min-shared", type=int, default=30)
    ap.add_argument("--cameras", type=int, default=500)
    ap.add_argument("--points", type=int, default=200000)
    ap.add_argument("--oracle-tracks", type=int, default=2000)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("measure_triangulation.py needs a CUDA device")
    from measure_tracks import card, scene_matches

    from opensfm_b200 import map_types, synthetic as syn, tracking, triangulation
    from opensfm_b200 import types as T
    from oracle import triangulation_oracle as to

    scene = syn.cube_scene(args.cameras, args.points, max_obs_per_point=10, with_descriptors=False)
    features, matches = scene_matches(scene, args.min_shared)
    tm = tracking.create_tracks_manager(features, {s: np.zeros((len(f), 3), dtype=np.uint8) for s, f in features.items()},
                                        {}, {}, matches, 2)
    k1, k2, focal = scene.cam_params[0]
    camera = DistortedPerspective(k1, k2, focal)
    rec = map_types.Reconstruction()
    rec.add_camera(camera)
    for s in tm.images:
        pose = T.Pose()
        pose.set_rotation_matrix(scene.R_wc[s])
        pose.set_origin(scene.origins[s])
        rec.create_shot(s, camera.id, pose)
    config = {"triangulation_threshold": 0.006, "triangulation_min_ray_angle": 1.0, "triangulation_min_depth": 0.001,
              "triangulation_type": "FULL", "triangulation_refinement_iterations": 10}
    opts = triangulation._options(config)
    rays = triangulation.shot_rays(tm, rec)
    selected = np.ones(tm.num_tracks(), dtype=np.uint8)
    args_bulk = (rays["image_rt"], rays["image_origin"], rays["image_in"], rays["bearings"], selected) + opts

    def stats(ts):
        return {"median": float(np.median(ts)), "min": float(min(ts)), "max": float(max(ts))}

    tm.triangulate(*args_bulk)   # warm-up: module load, workspaces
    kernel, bulk = [], []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        X, status = tm.triangulate(*args_bulk)
        bulk.append((time.perf_counter() - t0) * 1e3)
        kernel.append(tm.triangulate_device_ms)
    retri, parts = [], {"bearings": [], "device_call": [], "write": []}
    for _ in range(args.reps):
        report = triangulation.retriangulate(tm, rec, config)
        retri.append(report["wall_time"] * 1e3)
        for k in parts:
            parts[k].append(report["wall_times"][k] * 1e3)
    n = min(args.oracle_tracks, tm.num_tracks())
    ts = tm.track_start[:n + 1]
    t0 = time.perf_counter()
    ost, oX, _ = to.triangulate_tracks(ts, tm.obs_image, rays["image_rt"], rays["image_origin"], rays["image_in"],
                                       rays["bearings"], selected[:n], *opts)
    oracle_ms = (time.perf_counter() - t0) * 1e3
    ok = (ost == to.OK) & (status[:n] == to.OK)
    rec_out = {
        "card": card(), "reps": args.reps,
        "sizes": {"images": len(tm.images), "tracks": tm.num_tracks(), "observations": int(len(tm.obs_track))},
        "statuses": np.bincount(status, minlength=5).tolist(),
        "points_after": report["num_points_after"],
        "kernel_ms": stats(kernel), "bulk_ms": stats(bulk), "retriangulate_ms": stats(retri),
        "retriangulate_parts_ms": {k: stats(v) for k, v in parts.items()},
        "oracle_tracks": n, "oracle_ms_per_1000_tracks": oracle_ms * 1000.0 / max(n, 1),
        "oracle_status_agrees": bool(np.array_equal(ost, status[:n])),
        "oracle_max_point_difference": float(np.abs(oX[ok] - X[:n][ok]).max()) if ok.any() else None,
    }
    print(json.dumps(rec_out))


if __name__ == "__main__":
    main()
