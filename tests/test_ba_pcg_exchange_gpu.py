"""The exchange of the pipelined PCG (pcg_pipelined): m = M^-1 w and the per-CTA dot products travel as flagged words
that carry a generation, zeroed before every solve.  Bundles of different sizes back to back on one pooled handle must
not see a word left by an earlier solve; small grids (fewer CTAs than SMs), the path without deflation, an exact start
and a one-iteration bundle must take the pipelined path without a rescue by the classic PCG.  Bundles run to the end
must agree with the classic_pcg fallback: iterations, termination, cost to 1e-9 relative, parameters to 1e-6 (the Schur
atomics are unordered, as in test_ba_pcg_path_gpu.py); the one-iteration bundle must solve its captured system to
|S y - rhs| <= 1.5e-8 |rhs| (tests/test_ba_linear_system_gpu.py)."""
import numpy as np
import pytest

import ba_linear_system_scenes as scenes
from opensfm_b200 import ba_problem as bp, bundle, synthetic as syn

pytestmark = pytest.mark.gpu

SUMMARY = ("iterations", "termination", "final_cost", "pcg_iterations", "linear_solves")


@pytest.fixture(scope="module")
def c4_problem():
    return syn.scene_to_problem(syn.cube_scene(500, 200000, 1.0, seed=42, max_obs_per_point=10))


def _ring16():
    return scenes.ring_problem([bp.PERSPECTIVE] * 16, n_points=300, seed=1)


def _solve(pb, fallbacks=()):
    r = bundle.solve(pb, fallbacks=fallbacks)
    return {k: r["summary"][k] for k in SUMMARY}, {k: r[k] for k in ("cam_params", "inst", "points")}


def _path(pb, fallbacks=()):
    """kernel and rescue of the first LM iteration's PCG"""
    cap = bundle.solve(pb, capture_iteration=1, fallbacks=fallbacks)["capture"]
    return cap["pcg_kernel"], cap["pcg_rescued"]


def _agrees_with_classic(pb, s, x, classic_path=()):
    sc, xc = _solve(pb, ("classic_pcg",) + tuple(classic_path))
    print("pipelined: %s | classic: %s" % (s, sc))
    assert s["iterations"] == sc["iterations"] and s["termination"] == sc["termination"]
    assert abs(s["final_cost"] - sc["final_cost"]) <= 1e-9 * abs(sc["final_cost"])
    for k in ("cam_params", "inst", "points"):
        assert np.abs(x[k] - xc[k]).max(initial=0.0) <= 1e-6 * max(1.0, np.abs(xc[k]).max(initial=0.0)), k


def test_bundles_back_to_back_on_one_handle(c4_problem):
    """C4, a 16-shot ring (9 CTAs), C4 again: the second C4 takes the steps of the first."""
    first, x_first = _solve(c4_problem)
    ring, x_ring = _solve(_ring16())
    again, x_again = _solve(c4_problem)
    print("C4: %s\nring: %s\nC4 again: %s" % (first, ring, again))
    for k in ("iterations", "termination", "pcg_iterations", "linear_solves"):
        assert again[k] == first[k], k
    assert abs(again["final_cost"] - first["final_cost"]) <= 1e-9 * first["final_cost"]
    assert first["iterations"] == 5 and first["pcg_iterations"] == 403
    _agrees_with_classic(c4_problem, again, x_again)
    _agrees_with_classic(_ring16(), ring, x_ring)


def test_small_grid_takes_pipelined_path():
    pb = _ring16()
    assert _path(pb) == ("pipelined_deflated", 0)
    s, x = _solve(pb)
    _agrees_with_classic(pb, s, x)


def test_undeflated_pipelined_path(c4_problem):
    """Three dot products per CTA in flagged words instead of the ten of the deflated solver."""
    for pb in (_ring16(), syn.scene_to_problem(syn.cube_scene(30, 4000, 1.0, seed=5))):
        assert _path(pb, ("undeflated_pcg",)) == ("pipelined", 0)
        s, x = _solve(pb, ("undeflated_pcg",))
        _agrees_with_classic(pb, s, x)


def test_exact_start():
    """Noise-free observations at the true parameters: the right-hand side is (nearly) zero."""
    pb = syn.scene_to_problem(syn.cube_scene(12, 1500, 0.0, seed=3), perturb_seed=None)
    s, x = _solve(pb)
    assert s["iterations"] <= 1 and s["termination"] == "CONVERGENCE"
    _agrees_with_classic(pb, s, x)


def test_one_iteration():
    """One LM step: its cost depends on the PCG's 1e-8 stopping point, so the check is the captured solve itself."""
    pb = syn.scene_to_problem(syn.cube_scene(20, 3000, 1.0, seed=9), max_iterations=1)
    r = bundle.solve(pb, capture_iteration=1)
    cap = r["capture"]
    assert (cap["pcg_kernel"], cap["pcg_rescued"]) == ("pipelined_deflated", 0)
    assert r["summary"]["iterations"] == 1
    res = np.linalg.norm(cap["S"] @ cap["y"] - cap["rhs"]) / np.linalg.norm(cap["rhs"])
    assert res <= 1.5e-8, res
