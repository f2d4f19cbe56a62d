"""Device time of the dense stage on textured_scene shots at 640x480 with the reference's default configuration
(patch 7, 100 planes for brute force, 3 PatchMatch iterations, 6 matching views): estimate, clean and prune in ms by
CUDA events, shots/s and NCC taps/s, per method, for a full batch and for a batch smaller than the SM count.  The
oracle's time ("port", one CPU thread, raster order) is given for one shot at 320x240 for scale.

    python tools/measure_dense.py [--shots 16] [--small 4]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from opensfm_b200 import dense as D  # noqa: E402
from opensfm_b200 import synthetic as syn  # noqa: E402


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "not measured"
    return name, out, torch.cuda.get_device_properties(0).multi_processor_count


def taps(method, n_views, w, h, patch=7, planes=100, iters=3):
    px = (w - patch + 1) * (h - patch + 1) * patch * patch
    if method == "BRUTE_FORCE":
        return px * planes * (n_views - 1)
    cand = 1 + iters * 2 * (2 + 6 + (1 if method == "PATCH_MATCH_SAMPLE" else 0))
    return px * cand * (1 if method == "PATCH_MATCH_SAMPLE" else n_views - 1)


def run(shots, w, h, method, seed=0):
    n = shots + 6
    sc = syn.textured_scene(n, w, h, arc_degrees=min(10.0 * n, 90.0))
    views = [D.View(K=sc.K[k], R=sc.R[k], t=sc.t[k], width=w, height=h, gray=sc.gray[k],
                    mask=np.ones((h, w), np.uint8), color=sc.rgb[k], labels=np.zeros((h, w), np.uint8))
             for k in range(n)]
    refs = []
    for k in range(shots):
        others = sorted(range(n), key=lambda v: abs(v - k))[1:7]
        refs.append(D.Reference([k] + others, 3.0, 60.0, method, 7, 100, 3, key=k))
    D.depthmaps(views, refs[:1], 0.1, 0.01, 2, seed)          # warm-up: module load, allocations
    t0 = time.perf_counter()
    _, _, pruned, ms = D.depthmaps(views, refs, 0.1, 0.01, 2, seed)
    wall = time.perf_counter() - t0
    return ms, wall, sum(len(p[0]) for p in pruned)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shots", type=int, default=16)
    ap.add_argument("--small", type=int, default=4)
    ap.add_argument("--port", action="store_true", help="also time the oracle on one 320x240 shot per method")
    a = ap.parse_args()
    name, power, sms = card()
    print(json.dumps({"card": name, "power_limit": power, "sms": sms}))
    for method in ("PATCH_MATCH_SAMPLE", "PATCH_MATCH", "BRUTE_FORCE"):
        for shots in (a.shots, a.small):
            ms, wall, pts = run(shots, 640, 480, method)
            tp = taps(method, 7, 640, 480) * shots
            print(json.dumps({"method": method, "shots": shots, "estimate_ms": round(ms[0], 2),
                              "clean_ms": round(ms[1], 3), "prune_ms": round(ms[2], 3), "wall_s": round(wall, 3),
                              "shots_per_s": round(shots / (sum(ms) / 1e3), 2),
                              "taps_per_s": "%.3g" % (tp / (ms[0] / 1e3)), "points": pts}))
        if a.port:
            from oracle import dense_oracle as do

            sc = syn.textured_scene(7, 320, 240)
            t0 = time.perf_counter()
            do.estimate(sc.K, sc.R, sc.t, list(sc.gray), np.ones((240, 320), np.uint8), method, 7, 100, 3, 25.0, 3.0,
                        60.0)
            print(json.dumps({"method": method, "port_s_per_shot_320x240": round(time.perf_counter() - t0, 2)}))


if __name__ == "__main__":
    main()
