"""The flagship C4 scene (bench.py: 500 cameras, 200k points, 2M observations) on the PCG the solver is built around:
the gauge-deflated pipelined kernel, whose shared-memory plan (ba_pcg_plan.h) has to fit one CTA per SM.  Checks the
path and the solve of the captured system, then a full bundle() against the classic PCG (the classic_pcg fallback
path)."""
import numpy as np
import pytest

from opensfm_b200 import bundle, synthetic as syn

pytestmark = pytest.mark.gpu

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


def test_c4_bundle_matches_classic_pcg_fallback(c4_scene):
    pb = syn.scene_to_problem(c4_scene)
    out = {}
    for name, fallbacks in (("pipelined", ()), ("classic", ("classic_pcg",))):
        r = bundle.solve(pb, fallbacks=fallbacks)
        out[name] = ({k: r["summary"][k] for k in ("iterations", "termination", "final_cost", "pcg_iterations")}, r)
    (sp, dp), (sc, dc) = out["pipelined"], out["classic"]
    print("pipelined: %s | classic: %s" % (sp, sc))
    assert sp["iterations"] == sc["iterations"] and sp["termination"] == sc["termination"]
    assert abs(sp["final_cost"] - sc["final_cost"]) <= 1e-9 * sc["final_cost"]
    for k in ("cam_params", "inst", "points"):
        assert np.abs(dp[k] - dc[k]).max() <= 1e-6, k
    assert sp["pcg_iterations"] < sc["pcg_iterations"]
