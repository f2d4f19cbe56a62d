"""Time the ranking of image pairs for the reconstruction bootstrap on the GPU over tracks shaped like bench.py's C4
scene: cube_scene(500, 200000, max_obs_per_point=10) matched on its ground-truth correspondences (as
tools/measure_tracks.py), linked into tracks, every pair with at least 50 common tracks ranked.  Bearings come from a
distortion-free pinhole camera over the normalised image coordinates.

    python tools/measure_image_pairs.py [--reps 3] [--oracle-pairs 20]

Prints one JSON line: the card's name and power limit, the workload (pairs with 50 common tracks, rows), and
  * `from_tracks`: compute_image_pairs_from_tracks (bearings once per image, rows from the device's common-track
    lists): host clock end to end, and the device time of the RANSAC kernels (CUDA events), medians of --reps;
  * `lists`: tracking.all_common_tracks_with_features then compute_image_pairs on its per-pair lists, the same two
    clocks, plus the time of the lists alone;
  * `oracle_ms_per_pair`: oracle/rotation_ransac_oracle.py (numpy, one CPU core) on --oracle-pairs pairs spread over
    the workload, and that rate extrapolated to all pairs;
  * `agree`: both paths return the same ranking.
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
    def pixel_bearing_many(self, p):
        p = np.asarray(p, dtype=np.float64).reshape(-1, 2)
        b = np.column_stack([p, np.ones(len(p))])
        return b / np.sqrt((b * b).sum(axis=1))[:, None]


class Dataset:
    config = {"five_point_algo_threshold": 0.004, "processes": 1}
    camera = PinholeCamera()

    def load_camera_models(self):
        return {"cam": self.camera}

    def load_exif(self, image):
        return {"camera": "cam"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-pairs", type=int, default=20)
    ap.add_argument("--cameras", type=int, default=500)
    ap.add_argument("--points", type=int, default=200000)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("measure_image_pairs.py needs a CUDA device")
    from measure_tracks import card, scene_matches
    from opensfm_b200 import reconstruction as rec, rotation_ransac as rr, synthetic as syn, tracking

    scene = syn.cube_scene(args.cameras, args.points, max_obs_per_point=10, with_descriptors=False)
    features, matches = scene_matches(scene, 30)
    tm = tracking.create_tracks_manager(features, {}, {}, {}, matches, 2)
    data = Dataset()
    cameras = {im: data.camera for im in tm.images}

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        return (time.perf_counter() - t0) * 1e3, r

    fast = lambda: rec.compute_image_pairs_from_tracks(tm, cameras, data.config)
    fast()   # warm-up: module load, workspaces, the device's sample stream
    t_fast, d_fast, t_lists, t_rank, d_rank = [], [], [], [], []
    for _ in range(args.reps):
        ms, ranked_fast = clock(fast)
        t_fast.append(ms)
        d_fast.append(rr.last_device_ms())
        ms, track_dict = clock(lambda: tracking.all_common_tracks_with_features(tm))
        t_lists.append(ms)
        ms, ranked = clock(lambda: rec.compute_image_pairs(track_dict, data))
        t_rank.append(ms)
        d_rank.append(rr.last_device_ms())

    from oracle import rotation_ransac_oracle as ro

    keys = list(track_dict)
    pick = np.linspace(0, len(keys) - 1, min(args.oracle_pairs, len(keys))).astype(int)
    t0 = time.perf_counter()
    for q in pick:
        _, p1, p2 = track_dict[keys[q]]
        ro.ransac_rotation(data.camera.pixel_bearing_many(p1), data.camera.pixel_bearing_many(p2),
                           4 * data.config["five_point_algo_threshold"])
    per_pair = (time.perf_counter() - t0) * 1e3 / len(pick)

    med = lambda xs: float(np.median(xs))
    rec_out = {
        "card": card(), "reps": args.reps,
        "workload": {"images": scene.num_shots, "pairs": len(keys), "rows": int(sum(len(v[0]) for v in track_dict.values())),
                     "ranked_pairs": len(ranked)},
        "from_tracks": {"end_to_end_ms": med(t_fast), "device_ms": med(d_fast)},
        "lists": {"all_common_tracks_with_features_ms": med(t_lists), "compute_image_pairs_ms": med(t_rank),
                  "end_to_end_ms": med(t_lists) + med(t_rank), "device_ms": med(d_rank)},
        "oracle_ms_per_pair": per_pair, "oracle_ms_all_pairs_estimate": per_pair * len(keys),
        "agree": ranked == ranked_fast,
    }
    print(json.dumps(rec_out))


if __name__ == "__main__":
    main()
