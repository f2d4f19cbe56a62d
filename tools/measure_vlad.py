"""Time VLAD pair selection on the GPU over bench.py's matching workload (C4: 500 images, about 4000 HAHOG-like
descriptors each, resident as uint8-stored L2 like bench.py keeps them).

    python tools/measure_vlad.py [--reps 10] [--k 10]

Prints one JSON line: the card's name and power limit, the work computed from shapes (operations and the least
bytes each phase must move), and for
  * histograms: `PairMatcher.compute_vlad` over all images (word assignment, residual sums, normalisation);
  * select: `match_candidates_with_vlad` of every image against every image (distances + neighbour selection on
    the device, the selected pairs back on the host), k = --k, with and without camera groups;
two times, each after one warm-up call:
  * `*_device_ms`: device time per call, the summed durations of the VLAD kernels that torch.profiler (CUDA
    activities, CUPTI timestamps) records over --reps calls, divided by --reps, per kernel and in total.  The work
    runs on the matcher's own CUDA stream, which the library does not expose, so CUDA events recorded from Python
    on a torch stream would not bracket it; the profiler sees every stream.
  * `*_ms`: end-to-end time per call, the median of --reps host-clock timings of calls that end in a stream
    synchronise.  This is what a caller waits for: kernels plus ctypes marshalling, the small table uploads and the
    copy of the results back.
The two passes are separate, so the profiler's overhead does not enter the end-to-end times.
"""
import argparse
import json
import os
import re
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--k", type=int, default=10)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("measure_vlad.py needs a CUDA device")
    import bench
    from opensfm_b200 import matching, pairs_selection as ps

    words = np.load(os.path.join(ROOT, "tests", "golden", "vlad_words_64.npz"))["words"]
    _, feats, _, _ = bench.build_workload("c4")
    names = list(range(len(feats)))
    pm = matching.PairMatcher()
    pm.add_many([(i, f.astype(np.uint8)) for i, f in enumerate(feats)], uint8_is_l2=True)
    exifs = {i: {"camera": "cam%d" % (i % 3)} for i in names}

    def hist():
        pm.compute_vlad(names, words)

    def select(enforce):
        return ps.match_candidates_with_vlad(pm, names, names, exifs, args.k, enforce)

    def timed(fn):
        fn()
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts)), float(min(ts)), float(max(ts))

    n, nc, dim = len(feats), words.shape[0], words.shape[1]
    nfeat = int(sum(len(f) for f in feats))
    L = nc * dim
    work = {
        "images": n, "features": nfeat, "centers": nc, "dim": dim,
        # float32 subtract + multiply + add per (feature, centre, element)
        "assign_flop": 3 * nfeat * nc * dim,
        "assign_bytes": 4 * nfeat * dim,
        "accumulate_flop": 2 * nfeat * dim + 4 * n * L,
        "accumulate_bytes": 4 * nfeat * dim + 8 * n * L,
        # fp64 subtract + fused multiply-add (2) per (reference, candidate, element)
        "distance_flop": 3 * n * n * L,
        "distance_bytes": 4 * 2 * n * L,
    }

    def device(fn):
        from torch.profiler import ProfilerActivity, profile

        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                fn()
            torch.cuda.synchronize()
        per = {}
        for ev in prof.events():
            m = re.search(r"(vlad_\w+|neighbor_select)_kernel", ev.name)
            if ev.device_type == torch.autograd.DeviceType.CUDA and m:
                per[m.group(0)] = per.get(m.group(0), 0.0) + ev.device_time / 1e3 / args.reps
        return {"total": sum(per.values()), "kernels": per}

    rec = {"card": card(), "work": work, "reps": args.reps}
    phases = (("histograms", hist), ("select", lambda: select(False)),
              ("select_enforce_other_cameras", lambda: select(True)))
    for name, fn in phases:
        med, lo, hi = timed(fn)
        rec[name + "_ms"] = {"median": med, "min": lo, "max": hi}
    rec["select_ms"]["pairs"] = len(select(False))
    rec["select_enforce_other_cameras_ms"]["pairs"] = len(select(True))
    for name, fn in phases:
        rec[name + "_device_ms"] = device(fn)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
