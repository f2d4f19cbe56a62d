"""Times the bundle adjuster's covariance pass on the C4 scene (500 cameras, 200k points, 10 observations per point)
with GPS priors on every rig instance: n_c = 4500, m = 3000.

Reports the card name and power limit (read in the same process as the measurement), run() with and without
covariances, the pass time and the Cholesky time from the CUDA events around them inside run(), and the Cholesky
rate n_c^3 / 3 over its kernel time next to the H100 SXM data-sheet FP64 tensor-core figure (67 TFLOP/s at 700 W).
Fails without a GPU.  Usage: python tools/measure_covariance.py [--repeats N]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from opensfm_b200 import bundle  # noqa: E402
from opensfm_b200 import synthetic as syn  # noqa: E402

FP64_TC_PEAK = 67e12   # H100 SXM data sheet, dense FP64 tensor core, 700 W


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().split("\n")[0]
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--points", type=int, default=200000)
    a = ap.parse_args()
    sc = syn.cube_scene(500, a.points, 1.0, seed=42, with_descriptors=False, max_obs_per_point=10)
    pb = syn.scene_to_problem(sc)
    rng = np.random.RandomState(11)
    pb.inst_has_prior[:] = 1
    pb.inst_prior_pos = pb.inst[:, 3:] + rng.normal(0, 0.02, (len(pb.inst), 3))
    pb.inst_prior_std = np.full((len(pb.inst), 3), 0.05)
    bundle.solve(pb, compute_covariances=True)   # warm-up: module load, allocations, shared-memory opt-ins
    bundle.solve(pb)
    rows = []
    for _ in range(a.repeats):
        for cov in (False, True):
            t0 = time.perf_counter()
            res = bundle.solve(pb, compute_covariances=cov)
            wall = time.perf_counter() - t0
            row = {"covariances": cov, "run_wall_s": wall, "run_device_ms": res["summary"]["time_device_ms"],
                   "iterations": res["summary"]["iterations"]}
            if cov:
                pass_ms, chol_ms = res["covariance_ms"]
                nc = res["summary"]["reduced_dim"]
                row.update(pass_ms=pass_ms, cholesky_ms=chol_ms, n_c=nc,
                           status=res["covariance_status"],
                           cholesky_tflops=nc ** 3 / 3 / (chol_ms * 1e-3) / 1e12,
                           cholesky_share_of_fp64_tc_datasheet=nc ** 3 / 3 / (chol_ms * 1e-3) / FP64_TC_PEAK)
            rows.append(row)
    print(json.dumps({"card": card(), "runs": rows}, indent=1))


if __name__ == "__main__":
    main()
