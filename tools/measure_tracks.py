"""Time track creation on the GPU over matches shaped like bench.py's C4 scene: cube_scene(500, 200000,
max_obs_per_point=10), every pair of shots that shares at least --min-shared points matched on exactly those points
(ground-truth matches; what a matcher followed by a perfect verification would hand over).

    python tools/measure_tracks.py [--reps 5] [--min-shared 30] [--no-oracle]

Prints one JSON line: the card's name and power limit, the graph (images, pairs, nodes = features, edges = match
rows), the result (tracks, observations, connected image pairs, R = common observations over all pairs), and
  * `build_device_ms` / `common_device_ms`: CUDA events on the handle's stream around the kernels, sorts and scans of
    osfm_tracks_build (after the uploads) and of osfm_tracks_common (osfm_tracks_last_device_ms), median of --reps;
  * `create_tracks_manager_ms`: host clock around tracking.create_tracks_manager (marshalling, upload, device work,
    download; the call ends in a stream synchronise), median of --reps after one warm-up call;
  * `all_common_tracks_with_features_ms`: the same around tracking.all_common_tracks_with_features(min_common=50) on
    a fresh TracksManager (device work, download, one dictionary entry per image pair);
  * `oracle_ms`: oracle/tracks_oracle.py (scipy connected components and Python loops, on the CPU) computing both
    results once, for scale.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:   # the measurement still needs a GPU: the timed calls below fail without one
        return {"name": "unknown (%s)" % e}


def scene_matches(scene, min_shared):
    """(features {shot: n x 3}, matches {(i, j): K x 2}) of the scene's own observations: feature k of shot s is the
    k-th observation of s; shots i < j are matched on the points both see."""
    S = scene.num_shots
    order = np.lexsort((scene.obs_shot, scene.obs_point))      # by (point, shot)
    shot, point = scene.obs_shot[order].astype(np.int64), scene.obs_point[order]
    start = np.searchsorted(scene.obs_shot, np.arange(S + 1))   # the scene's observations are shot-major
    assert np.all(np.diff(scene.obs_shot) >= 0)
    feat = order - start[shot]
    key, rows = [], []
    d = 1
    while d < len(point):
        same = point[d:] == point[:-d]
        if not same.any():
            break
        key.append(shot[:-d][same] * S + shot[d:][same])
        rows.append(np.column_stack([feat[:-d][same], feat[d:][same]]))
        d += 1
    key, rows = np.concatenate(key), np.concatenate(rows).astype(np.int32)
    by_pair = np.argsort(key, kind="stable")
    key, rows = key[by_pair], rows[by_pair]
    pairs, first, count = np.unique(key, return_index=True, return_counts=True)
    matches = {(int(k // S), int(k % S)): rows[b:b + n] for k, b, n in zip(pairs, first, count) if n >= min_shared}
    features = {s: np.column_stack([scene.obs_xy[start[s]:start[s + 1]], scene.obs_sigma[start[s]:start[s + 1]]])
                for s in range(S)}
    return features, matches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--min-shared", type=int, default=30)
    ap.add_argument("--cameras", type=int, default=500)
    ap.add_argument("--points", type=int, default=200000)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("measure_tracks.py needs a CUDA device")
    from opensfm_b200 import synthetic as syn, tracking

    scene = syn.cube_scene(args.cameras, args.points, max_obs_per_point=10, with_descriptors=False)
    features, matches = scene_matches(scene, args.min_shared)

    def create():
        return tracking.create_tracks_manager(features, {}, {}, {}, matches, 2)

    def clock(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        return (time.perf_counter() - t0) * 1e3, r

    def stats(ts):
        return {"median": float(np.median(ts)), "min": float(min(ts)), "max": float(max(ts))}

    tracking.all_common_tracks_with_features(create())   # warm-up: module load, workspaces
    t_create, t_common, d_build, d_common = [], [], [], []
    for _ in range(args.reps):
        ms, tm = clock(create)
        t_create.append(ms)
        d_build.append(tm.build_device_ms)
        ms, common = clock(lambda: tracking.all_common_tracks_with_features(tm))
        t_common.append(ms)
        d_common.append(tm.common_device_ms)
    pa, _, _, ca, _ = tm._common_arrays()
    rec = {
        "card": card(), "reps": args.reps,
        "graph": {"images": scene.num_shots, "pairs": len(matches), "nodes": int(sum(len(f) for f in features.values())),
                  "edges": int(sum(len(m) for m in matches.values()))},
        "result": {"tracks": tm.num_tracks(), "observations": int(len(tm.obs_track)), "connected_pairs": int(len(pa)),
                   "R": int(len(ca)), "pairs_with_50_common": len(common)},
        "build_device_ms": stats(d_build), "common_device_ms": stats(d_common),
        "create_tracks_manager_ms": stats(t_create), "all_common_tracks_with_features_ms": stats(t_common),
    }
    if not args.no_oracle:
        from oracle import tracks_oracle

        t0 = time.perf_counter()
        part, pairs = tracks_oracle.tracks(features, matches, 2)
        rec["oracle_ms"] = (time.perf_counter() - t0) * 1e3
        rec["oracle_agrees"] = bool(len(part) == tm.num_tracks() and sum(len(v) for v in pairs.values()) == len(ca))
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
