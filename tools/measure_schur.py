"""Times the reduced-camera-system (Schur) phase of bundle adjustment on the C4 scene of bench.py (500 cameras, 200k
points, 10 observations per point) for one or more source trees, alternating between them.

Every tree must be built (opensfm_b200/lib/libopensfm_b200.so).  The scene is built once, here, and handed to one
worker process per tree; the workers then take turns, one full bundle() each, for --runs rounds.  Per run it reports
the Schur time per launch (CUDA events around ba_point_blocks + the Schur kernel inside run()), time_device_ms, the
headline value (observations x LM iterations / time_device_ms, as bench.py computes it), the iteration count; per tree, the
device memory the library holds after its first run.  With --trace each tree also does one run under OSFM_BA_TRACE=1 and its in-kernel
clock lines are printed.  With --profile each tree also does one run of its own under torch.profiler (CUDA activities), after
the timed runs and in a fresh process, and the device time of every kernel of that one bundle() is printed, summed by
kernel name, with its launch count.  The card's name and power limit are read in the same process.  Fails without a GPU.

    python tools/measure_schur.py --trees OLD_TREE . --runs 5 [--trace] [--profile] [--out FILE]"""
import argparse
import json
import os
import pickle
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().split("\n")[0]


def worker(tree, problem_path):
    """Loads the library of `tree`, then answers one JSON line per 'run' or 'profile' read from stdin."""
    sys.path.insert(0, os.path.abspath(tree))
    import torch
    from opensfm_b200 import bundle

    with open(problem_path, "rb") as f:
        pb = pickle.load(f)
    torch.cuda.init()
    free0, _ = torch.cuda.mem_get_info()
    bundle.solve(pb)   # warm-up: module load, allocations, shared-memory opt-ins
    # device memory the library holds after one run (a device-wide reading: other work on the card shows up in it)
    free1, _ = torch.cuda.mem_get_info()
    print(json.dumps({"ready": True, "library_mb": (free0 - free1) / 2 ** 20}), flush=True)
    for line in sys.stdin:
        if line.strip() == "profile":
            print(json.dumps(profile_one(bundle, pb)), flush=True)
            continue
        if line.strip() != "run":
            break
        s = bundle.solve(pb)["summary"]
        print(json.dumps({
            "schur_ms_per_launch": s["time_schur_ms"] / max(s["schur_launches"], 1), "schur_launches": s["schur_launches"],
            "time_schur_ms": s["time_schur_ms"], "time_linearize_ms": s["time_linearize_ms"],
            "linearize_launches": s["linearize_launches"], "time_pcg_ms": s["time_pcg_ms"],
            "time_backsub_ms": s["time_backsub_ms"], "time_device_ms": s["time_device_ms"],
            "iterations": s["iterations"], "kernel_launches": s["kernel_launches"],
            "pcg_iterations": s["pcg_iterations"], "linear_solves": s["linear_solves"],
            "value": pb.num_observations * s["iterations"] / (s["time_device_ms"] * 1e-3),
            "final_cost": s["final_cost"], "termination": s["termination"]}), flush=True)


def profile_one(bundle, pb):
    """One bundle() under torch.profiler: {kernel name: [device ms, launches]}, the summary's phase timers."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s = bundle.solve(pb)["summary"]
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.events():   # device-side events: one per kernel launch, memset and copy
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name.split("(")[0].replace("void ", "").replace("osfm::", "")
        k = kernels.setdefault(name, [0.0, 0])
        k[0] += ev.device_time_total / 1e3
        k[1] += 1
    return {"kernels": kernels, "time_device_ms": s["time_device_ms"], "time_linearize_ms": s["time_linearize_ms"],
            "time_schur_ms": s["time_schur_ms"], "iterations": s["iterations"],
            "linearize_launches": s["linearize_launches"], "schur_launches": s["schur_launches"]}


def spawn(tree, problem_path, env=None, stderr=None):
    p = subprocess.Popen([sys.executable, os.path.abspath(__file__), "--worker", tree, "--problem", problem_path],
                         stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=stderr, text=True, env=env)
    ready = json.loads(p.stdout.readline())
    assert ready.get("ready"), ready
    p.library_mb = ready["library_mb"]
    return p


def ask(p):
    p.stdin.write("run\n")
    p.stdin.flush()
    return json.loads(p.stdout.readline())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs="+", default=[ROOT])
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--trace", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--problem", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a.worker, a.problem)
        return

    sys.path.insert(0, ROOT)
    from opensfm_b200 import synthetic as syn

    sc = syn.cube_scene(500, 200000, 1.0, seed=42, with_descriptors=True, max_obs_per_point=10)   # bench.py's C4
    pb = syn.scene_to_problem(sc)
    del sc
    report = {"card": card(), "trees": a.trees, "observations": int(pb.num_observations), "runs": {}}
    names = ["%d:%s" % (i, t) for i, t in enumerate(a.trees)]
    with tempfile.TemporaryDirectory() as tmp:
        problem_path = os.path.join(tmp, "c4.pkl")
        with open(problem_path, "wb") as f:
            pickle.dump(pb, f)
        procs = [spawn(t, problem_path) for t in a.trees]
        report["library_mb"] = {t: p.library_mb for t, p in zip(names, procs)}
        try:
            for r in range(a.runs):   # alternating: drifts of the card's clocks fall on every tree alike
                for t, p in zip(names, procs):
                    row = ask(p)
                    report["runs"].setdefault(t, []).append(row)
                    print("run %d %-40s schur %.3f ms/launch  pcg %.2f ms (%d its / %d solves)  device %.1f ms  value %.4e  its %d" % (
                        r, t, row["schur_ms_per_launch"], row["time_pcg_ms"], row["pcg_iterations"], row["linear_solves"],
                        row["time_device_ms"], row["value"], row["iterations"]), flush=True)
        finally:
            for p in procs:
                p.stdin.close()
                p.wait()
        report["card_after"] = card()
        summary = {}
        for t in names:
            rows = report["runs"][t]
            summary[t] = {k: {"median": statistics.median(x[k] for x in rows), "min": min(x[k] for x in rows),
                              "max": max(x[k] for x in rows)}
                          for k in ("schur_ms_per_launch", "time_device_ms", "value", "time_linearize_ms", "time_pcg_ms",
                                    "pcg_iterations", "linear_solves", "iterations")}
        report["summary"] = summary
        if a.trace:
            report["trace"] = {}
            for i, t in enumerate(a.trees):
                log = os.path.join(tmp, "trace%d.txt" % i)
                with open(log, "w") as ef:
                    p = spawn(t, problem_path, env=dict(os.environ, OSFM_BA_TRACE="1"), stderr=ef)
                    ask(p)
                    p.stdin.close()
                    p.wait()
                with open(log) as ef:
                    lines = ef.read().splitlines()
                report["trace"][names[i]] = ([ln for ln in lines if "schur" in ln or "consumer group" in ln][-8:] +
                                             [ln for ln in lines if "pcg" in ln])
        if a.profile:
            report["profile"] = {}
            for i, t in enumerate(a.trees):
                p = spawn(t, problem_path)
                p.stdin.write("profile\n")
                p.stdin.flush()
                prof = json.loads(p.stdout.readline())
                p.stdin.close()
                p.wait()
                report["profile"][names[i]] = prof
                print("profile %s (one bundle, %d LM iterations, %d linearisations, %d Schur builds; device %.2f ms without the profiler: %.2f)" % (
                    names[i], prof["iterations"], prof["linearize_launches"], prof["schur_launches"], prof["time_device_ms"],
                    summary[names[i]]["time_device_ms"]["median"]))
                for kname, (ms, cnt) in sorted(prof["kernels"].items(), key=lambda kv: -kv[1][0]):
                    print("  %9.3f ms %5d x  %s" % (ms, cnt, kname))
    print(json.dumps({"card": report["card"], "library_mb": report["library_mb"], "summary": report["summary"], "trace": report.get("trace")}, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
