"""Time BoW pair selection on the GPU over bench.py's matching workload (C4: 500 images, about 4000 HAHOG-like
descriptors each, resident as uint8-stored L2 like bench.py keeps them) with a 10000-word vocabulary at k = 50 words
per feature (the reference's bow_words_to_match).

    python tools/measure_bow.py [--reps 5] [--k 10]

The vocabulary is synthesised from the committed 1024-word fixture (tests/golden/bow_words_1024.npz) by seeded
perturbation, as tests/test_bow_gpu.py does; the reference's own 10000-word file is not part of the repository.
Prints one JSON line: the card's name and power limit, the work computed from shapes, and for
  * words: `PairMatcher.compute_words` over all images (k = 50 nearest words, back on the host);
  * histograms: `PairMatcher.bow_histograms` over all images;
  * select: `match_candidates_with_bow` of every image against every image, k = --k, with and without camera groups;
two times, each after one warm-up call:
  * `*_device_ms`: device time per call, the summed durations of the BoW kernels that torch.profiler (CUDA
    activities) records over --reps calls, divided by --reps, per kernel and in total (the matcher's stream is not
    exposed, so CUDA events from Python would not bracket its work; the profiler sees every stream).
  * `*_ms`: end-to-end time per call, the median of --reps host-clock timings of calls that end in a stream
    synchronise.
`words_fp32_rate`: the word assignment's float32 operations (subtract, multiply, add per feature, word and element)
over bow_words_kernel's device time, and its share of the 67 TFLOP/s FP32 data-sheet peak of an H100 SXM at 700 W.
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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--k", type=int, default=10)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("measure_bow.py needs a CUDA device")
    import bench
    from opensfm_b200 import bow, matching, pairs_selection as ps

    z = np.load(os.path.join(ROOT, "tests", "golden", "bow_words_1024.npz"))
    rng = np.random.RandomState(10000)
    extra = z["words"][rng.randint(0, 1024, 10000 - 1024)] + rng.normal(0, 4, (10000 - 1024, 128))
    words = np.concatenate([z["words"], np.clip(extra, 0, 255)]).astype(np.float32)
    freq = np.concatenate([z["frequencies"], rng.randint(1, 3000, 10000 - 1024)]).astype(np.int64)
    bows = bow.BagOfWords(words, freq)
    _, feats, _, _ = bench.build_workload("c4")
    names = list(range(len(feats)))
    pm = matching.PairMatcher()
    pm.add_many([(i, f.astype(np.uint8)) for i, f in enumerate(feats)], uint8_is_l2=True)
    exifs = {i: {"camera": "cam%d" % (i % 3)} for i in names}

    def wordsfn():
        pm.compute_words(names, bows, 50)

    def hist():
        pm.bow_histograms(names, bows)

    def select(enforce):
        return ps.match_candidates_with_bow(pm, names, names, exifs, args.k, enforce)

    def timed(fn):
        fn()
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts)), float(min(ts)), float(max(ts))

    n, nw, dim = len(feats), words.shape[0], words.shape[1]
    nfeat = int(sum(len(f) for f in feats))
    work = {
        "images": n, "features": nfeat, "words": nw, "dim": dim, "k": 50,
        # float32 subtract + multiply + add per (feature, word, element)
        "words_flop": 3 * nfeat * nw * dim,
        "words_bytes": 4 * nfeat * dim + 4 * nfeat * 50,
        "histogram_bytes": 4 * nfeat + 8 * 2 * n * nw,
        # fp64 subtract + add per (reference, candidate, word)
        "distance_flop": 2 * n * n * nw,
        "distance_bytes": 8 * n * nw,
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
            m = re.search(r"(bow_\w+|neighbor_select)_kernel", ev.name)
            if ev.device_type == torch.autograd.DeviceType.CUDA and m:
                per[m.group(0)] = per.get(m.group(0), 0.0) + ev.device_time / 1e3 / args.reps
        return {"total": sum(per.values()), "kernels": per}

    rec = {"card": card(), "work": work, "reps": args.reps}
    phases = (("words", wordsfn), ("histograms", hist), ("select", lambda: select(False)),
              ("select_enforce_other_cameras", lambda: select(True)))
    for name, fn in phases:
        med, lo, hi = timed(fn)
        rec[name + "_ms"] = {"median": med, "min": lo, "max": hi}
    rec["select_ms"]["pairs"] = len(select(False))
    rec["select_enforce_other_cameras_ms"]["pairs"] = len(select(True))
    for name, fn in phases:
        rec[name + "_device_ms"] = device(fn)
    wk = rec["words_device_ms"]["kernels"].get("bow_words_kernel", 0.0)
    if wk > 0:
        rate = work["words_flop"] / (wk * 1e-3)
        rec["words_fp32_rate"] = {"flop_per_s": rate, "share_of_67_tflops": rate / 67e12}
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
