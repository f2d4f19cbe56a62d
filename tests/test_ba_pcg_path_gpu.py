"""The flagship C4 scene (bench.py: 500 cameras, 200k points, 2M observations) on the PCG the solver is built around:
the gauge-deflated pipelined kernel, whose shared-memory plan (ba_pcg_plan.h) has to fit one CTA per SM.  Checks the
path and the solve of the captured system, then a full bundle() against the classic PCG (OSFM_BA_PCG_PIPELINED=0, in a
subprocess: the switches are read once per process)."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from opensfm_b200 import bundle, synthetic as syn

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PCG_BAR = 1.5e-8


@pytest.fixture(scope="module")
def c4_scene():
    return syn.cube_scene(500, 200000, 1.0, seed=42, max_obs_per_point=10)


def _capture(pb):
    pb.max_iterations = 1
    cap = bundle.solve(pb, capture_iteration=1)["capture"]
    res = float(np.linalg.norm(cap["S"] @ cap["y"] - cap["rhs"]) / np.linalg.norm(cap["rhs"]))
    print("nc %d: pcg %s, rescued %d, %d iterations, |S y - rhs| / |rhs| = %.3e" % (
        cap["nc"], cap["pcg_kernel"], cap["pcg_rescued"], cap["pcg_iterations"], res))
    return cap, res


def test_c4_runs_deflated_pipelined_pcg(c4_scene):
    cap, res = _capture(syn.scene_to_problem(c4_scene))
    assert cap["nc"] == 4500
    assert cap["pcg_kernel"] == "pipelined_deflated" and not cap["pcg_rescued"]
    assert res <= PCG_BAR


def test_c4_shared_intrinsics_pcg_path(c4_scene):
    """One 3-parameter camera for all shots: its group's rows span every column of S."""
    cap, res = _capture(syn.scene_to_problem(c4_scene, shared_intrinsics=True))
    assert res <= PCG_BAR


WORKER = r"""
import json, pickle, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from opensfm_b200 import bundle
with open(sys.argv[2], "rb") as f:
    pb = pickle.load(f)
r = bundle.solve(pb)
s = r["summary"]
np.savez(sys.argv[3], cam_params=r["cam_params"], inst=r["inst"], points=r["points"],
         summary=np.array(json.dumps({k: s[k] for k in ("iterations", "termination", "final_cost", "pcg_iterations")})))
"""


def test_c4_bundle_matches_classic_pcg(c4_scene, tmp_path):
    pb = syn.scene_to_problem(c4_scene)
    prob = str(tmp_path / "c4.pkl")
    with open(prob, "wb") as f:
        pickle.dump(pb, f)
    out = {}
    for name, pipelined in (("pipelined", "1"), ("classic", "0")):
        path = str(tmp_path / (name + ".npz"))
        env = dict(os.environ, OSFM_BA_PCG_PIPELINED=pipelined)
        subprocess.run([sys.executable, "-c", WORKER, ROOT, prob, path], env=env, check=True)
        d = np.load(path)
        out[name] = (json.loads(str(d["summary"])), d)
    (sp, dp), (sc, dc) = out["pipelined"], out["classic"]
    print("pipelined: %s | classic: %s" % (sp, sc))
    assert sp["iterations"] == sc["iterations"] and sp["termination"] == sc["termination"]
    assert abs(sp["final_cost"] - sc["final_cost"]) <= 1e-9 * sc["final_cost"]
    for k in ("cam_params", "inst", "points"):
        assert np.abs(dp[k] - dc[k]).max() <= 1e-6, k
    assert sp["pcg_iterations"] < sc["pcg_iterations"]
