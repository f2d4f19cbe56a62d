"""Time the geometric verification of calibrated image pairs on the GPU (relative_pose.robust_match_pairs, the
batched robust_match_calibrated) after the matcher, on a C2-sized pair list: the cube scene with 50 cameras and 5000
points (k1 = -0.1, k2 = 0.01), all 1225 pairs, symmetric descriptor matches at ratio 0.8; and on the relative-pose
test batch (0 to 65 % injected outliers, its pairs of at least 8 rows).

    python tools/measure_robust_match.py [--reps 3] [--oracle-pairs 4]

Prints one JSON line: the card's name and power limit, and per workload
  * `pairs`, `rows`: the pairs verified on the device and their match rows;
  * `ransac_kernel_ms`, `filter_kernel_ms`: CUDA events around the RANSAC kernels and around rp_match_filter
    (relative_pose.last_stage_ms), medians of --reps after a warm-up call;
  * `call_ms`: host clock around the verification call (packing, upload, kernels, download; it ends in a stream
    synchronise), median of --reps;
  * for the scene, `match_ms`: host clock around PairMatcher.match_pairs of the pair list, and `table_ms`: the host
    time of building the bearing table and the row tables (pixel_bearing_many once per image, the rows of every
    pair), median of --reps; `driver_ms`: matching.match_images_with_pairs with `verify`, end to end, once;
  * `oracle_ms_per_pair`: oracle/robust_match_oracle.py (its RANSAC and the relax rounds) on --oracle-pairs pairs
    of the outlier batch, on one CPU core, for scale only.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:   # the measurement still needs a GPU: the timed calls below fail without one
        return {"name": "unknown (%s)" % e}


def timed(fn, reps):
    """fn() once to warm up, then --reps times: (last result, median host ms, median RANSAC ms, median filter ms)."""
    from opensfm_b200 import relative_pose as rp

    res = fn()
    call, ransac, filt = [], [], []
    for _ in range(reps):
        t = time.perf_counter()
        res = fn()
        call.append(1e3 * (time.perf_counter() - t))
        a, b = rp.last_stage_ms()
        ransac.append(a)
        filt.append(b)
    return res, statistics.median(call), statistics.median(ransac), statistics.median(filt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-pairs", type=int, default=4)
    args = ap.parse_args()

    import relative_pose_cases as C
    import robust_match_cases as RC
    from opensfm_b200 import matching
    from opensfm_b200 import relative_pose as rp
    from opensfm_b200 import synthetic as syn
    from oracle import robust_match_oracle as rmo

    config = RC.CONFIG
    thr = config["robust_matching_calib_threshold"]
    out = {"card": card()}

    # the C2-sized scene: matcher, then the device verification of every pair past the min-match gate
    sc = syn.cube_scene(50, 5000, seed=42)
    desc, points, _, cam = RC.cube_images(sc)
    images = sorted(desc)
    pairs = [(a, b) for i, a in enumerate(images) for b in images[i + 1:]]
    pm = matching.PairMatcher()
    pm.add_many([(im, desc[im]) for im in images])
    pm.match_pairs(pairs, config)
    match_ms = []
    for _ in range(args.reps):
        t = time.perf_counter()
        raw = pm.match_pairs(pairs, config)
        match_ms.append(1e3 * (time.perf_counter() - t))
    live = [p for p in pairs if len(raw[p]) >= config["robust_matching_min_match"]]

    def tables():
        base, tabs, n = {}, [], 0
        for im in images:
            base[im] = n
            tabs.append(cam.pixel_bearing_many(points[im][:, :2]))
            n += len(tabs[-1])
        start = np.concatenate([[0], np.cumsum([len(raw[p]) for p in live])]).astype(np.int64)
        ra = np.concatenate([base[p[0]] + raw[p][:, 0] for p in live]).astype(np.int64)
        rb = np.concatenate([base[p[1]] + raw[p][:, 1] for p in live]).astype(np.int64)
        return np.concatenate(tabs), start, ra, rb

    table_ms = []
    for _ in range(args.reps):
        t = time.perf_counter()
        tab = tables()
        table_ms.append(1e3 * (time.perf_counter() - t))
    res, call, ransac, filt = timed(lambda: rp.robust_match_pairs(*tab, thr), args.reps)
    t = time.perf_counter()
    got = matching.match_images_with_pairs(desc, pairs, config, verify={"cameras": {im: cam for im in images},
                                                                        "points": points})
    driver_ms = 1e3 * (time.perf_counter() - t)
    out["scene"] = {"cameras": 50, "points": 5000, "pairs": len(live), "rows": int(tab[1][-1]),
                    "match_ms": round(statistics.median(match_ms), 1), "table_ms": round(statistics.median(table_ms), 1),
                    "ransac_kernel_ms": round(ransac, 2), "filter_kernel_ms": round(filt, 2), "call_ms": round(call, 1),
                    "driver_ms": round(driver_ms, 1), "kept_matches": int(sum(len(v) for v in got.values())),
                    "empty_pairs": int(sum(res.empty_round(p) is not None for p in range(len(live))))}

    # injected outliers: the relative-pose test batch
    b1s, b2s = C.batch_pairs()
    keep = [p for p in range(len(b1s)) if len(b1s[p]) >= 8]
    b1s, b2s = [b1s[p] for p in keep], [b2s[p] for p in keep]
    res, call, ransac, filt = timed(lambda: rp.robust_match_lists(b1s, b2s, thr), args.reps)
    out["outliers"] = {"ratios": list(C.OUTLIERS), "pairs": len(b1s), "rows": int(sum(len(b) for b in b1s)),
                       "ransac_kernel_ms": round(ransac, 2), "filter_kernel_ms": round(filt, 2),
                       "call_ms": round(call, 1)}

    pick = np.linspace(0, len(b1s) - 1, args.oracle_pairs).astype(int)
    t = time.perf_counter()
    for p in pick:
        rmo.robust_match_calibrated(b1s[p], b2s[p], thr)
    out["oracle_ms_per_pair"] = round(1e3 * (time.perf_counter() - t) / len(pick), 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
