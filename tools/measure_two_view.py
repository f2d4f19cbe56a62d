"""Time the five-point relative-pose RANSAC on the GPU against its numpy restatement, on the pairs of the
relative-pose test batch (tests/relative_pose_cases.batch_pairs: 196 cube-scene pairs of 5 to 3000 rows with 0 to
65 % outliers) and on single pairs.

    python tools/measure_two_view.py [--reps 5] [--oracle-pairs 8]

Prints one JSON line: the card's name and power limit and
  * `batch_kernel_ms`: CUDA events around the kernels of one osfm_relpose_run over the whole batch
    (relative_pose.last_device_ms), median of --reps after a warm-up call;
  * `batch_call_ms`: host clock around relative_pose.ransac_lists over the batch (packing, upload, kernels,
    download; the call ends in a stream synchronise), median of --reps;
  * `single_pair`: per row count, the median host-clock latency of relative_pose.relative_pose_ransac on one pair
    of that size with 30 % outliers, and its kernel time;
  * `oracle_ms_per_pair`: oracle/relative_pose_oracle.py on --oracle-pairs pairs of the batch spread over its sizes,
    on one CPU core, for scale only (pyrobust is not built with this project);
  * `two_view`: the full two-view call (relative_pose.two_view_lists) over the batch, with check_reversal off and
    on: the kernel time of RANSAC and of the two-view stage (CUDA events, relative_pose.last_stage_ms), the host
    time of the cv2.findHomography loop (relative_pose.plane_motion over every pair) and the call's host time,
    medians of --reps; and the single-pair latency of reconstruction.two_view_reconstruction_general per row count.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:   # the measurement still needs a GPU: the timed calls below fail without one
        return {"name": "unknown (%s)" % e}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-pairs", type=int, default=8)
    args = ap.parse_args()

    import relative_pose_cases as C
    from opensfm_b200 import relative_pose as rp
    from oracle import relative_pose_oracle as ro

    out = {"card": card()}
    b1s, b2s = C.batch_pairs()
    out["batch"] = {"pairs": len(b1s), "rows": int(sum(len(b) for b in b1s))}
    rp.ransac_lists(b1s, b2s, C.THRESHOLD)
    kernel, call = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        rp.ransac_lists(b1s, b2s, C.THRESHOLD)
        call.append((time.perf_counter() - t0) * 1e3)
        kernel.append(rp.last_device_ms())
    out["batch_kernel_ms"] = float(np.median(kernel))
    out["batch_call_ms"] = float(np.median(call))

    single = {}
    for n in (50, 200, 1000, 3000):
        a, b = C.cube_pairs(8, 3000, 21, count=1, sizes=(n,), outlier_ratios=(0.3,))
        rp.relative_pose_ransac(a[0], b[0], C.THRESHOLD, 1000, 0.999)
        lat, ker = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            rp.relative_pose_ransac(a[0], b[0], C.THRESHOLD, 1000, 0.999)
            lat.append((time.perf_counter() - t0) * 1e3)
            ker.append(rp.last_device_ms())
        single[str(n)] = {"latency_ms": float(np.median(lat)), "kernel_ms": float(np.median(ker))}
    out["single_pair"] = single

    tv = {}
    for check in (False, True):
        rp.two_view_lists(b1s, b2s, C.THRESHOLD, 1000, check, 0.95)
        ker_r, ker_t, call, host = [], [], [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            rp.two_view_lists(b1s, b2s, C.THRESHOLD, 1000, check, 0.95)
            call.append((time.perf_counter() - t0) * 1e3)
            r_ms, t_ms = rp.last_stage_ms()
            ker_r.append(r_ms)
            ker_t.append(t_ms)
            t0 = time.perf_counter()
            for a, b in zip(b1s, b2s):
                rp.plane_motion(a, b, C.THRESHOLD)
            host.append((time.perf_counter() - t0) * 1e3)
        tv["check_reversal" if check else "default"] = {
            "ransac_kernel_ms": float(np.median(ker_r)), "two_view_kernel_ms": float(np.median(ker_t)),
            "find_homography_loop_ms": float(np.median(host)), "call_ms": float(np.median(call))}
    from image_pair_cases import PinholeCamera
    from opensfm_b200 import reconstruction as rec

    cam = PinholeCamera()
    single_tv = {}
    for n in (50, 200, 1000, 3000):
        a, b = C.cube_pairs(8, 3000, 21, count=1, sizes=(n,), outlier_ratios=(0.3,))
        p1, p2 = a[0][:, :2] / a[0][:, 2:], b[0][:, :2] / b[0][:, 2:]
        rec.two_view_reconstruction_general(p1, p2, cam, cam, C.THRESHOLD, 1000)
        lat, kr, kt = [], [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            rec.two_view_reconstruction_general(p1, p2, cam, cam, C.THRESHOLD, 1000)
            lat.append((time.perf_counter() - t0) * 1e3)
            r_ms, t_ms = rp.last_stage_ms()
            kr.append(r_ms)
            kt.append(t_ms)
        single_tv[str(n)] = {"latency_ms": float(np.median(lat)), "ransac_kernel_ms": float(np.median(kr)),
                             "two_view_kernel_ms": float(np.median(kt))}
    tv["single_pair"] = single_tv
    out["two_view"] = tv

    picks = np.linspace(0, len(b1s) - 1, args.oracle_pairs).astype(int).tolist()
    t0 = time.perf_counter()
    for k in picks:
        ro.ransac_relative_pose(b1s[k], b2s[k], C.THRESHOLD)
    out["oracle_ms_per_pair"] = (time.perf_counter() - t0) * 1e3 / len(picks)
    out["oracle_pairs"] = picks
    out["reps"] = args.reps
    print(json.dumps(out))


if __name__ == "__main__":
    main()
