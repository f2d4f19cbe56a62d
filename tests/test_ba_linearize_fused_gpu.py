"""The linearisation that also forms the column norms, the gradient and the per-point sums (ba_linearize_fused, used
for perspective scenes with the segment chunk list) against the separate plane-reading kernels (the generic_linearize
fallback path).  Only summation orders differ: the captured Jacobi scale, LM diagonal and gradient agree to 1e-12 at
LM iteration 1 (iteration 2: see below), and a full bundle() takes the same iterations to the same termination, final
cost and parameters."""
import numpy as np
import pytest

import ba_linear_system_scenes as scenes
from opensfm_b200 import ba_problem as bp
from opensfm_b200 import bundle

pytestmark = pytest.mark.gpu


def _c4():
    return scenes.cube(500, 200000, max_obs=10)


def _many_shots():
    """16 perspective cameras on a ring, observations thinned: segments of 1 to 16 shots, many of them longer than
    one chunk of 8 points."""
    return scenes.ring_problem([bp.PERSPECTIVE] * 16, n_points=600, seed=11, keep=0.7)


def _odd_count():
    pb = scenes.cube(9, 301, max_obs=5)
    if len(pb.obs_shot) % 2 == 0:
        pb.obs_shot, pb.obs_point = pb.obs_shot[:-1].copy(), pb.obs_point[:-1].copy()
        pb.obs_xy, pb.obs_sigma = pb.obs_xy[:-1].copy(), pb.obs_sigma[:-1].copy()
    assert len(pb.obs_shot) % 2 == 1
    return pb


SCENES = {
    "c4": (_c4, 10),
    "many_shots": (_many_shots, 20),
    "constant_blocks": (scenes.constant_blocks, 20),    # constant cameras, instances and points
    "fast_and_prior_points": (scenes.point_priors_many_obs, 20),   # segment points next to per-point ba_schur points
    "odd_count": (_odd_count, 20),
}


def _run(pb, fallbacks, max_its):
    out = {}
    for it in (1, 2):
        pb.max_iterations = it
        cap = bundle.solve(pb, capture_iteration=it, fallbacks=fallbacks)["capture"]
        for k in ("scale", "diag", "grad"):
            out["%s%d" % (k, it)] = cap[k]
    pb.max_iterations = max_its
    r = bundle.solve(pb, fallbacks=fallbacks)
    out.update({k: r[k] for k in ("cam_params", "inst", "points")})
    return {k: r["summary"][k] for k in ("iterations", "termination", "final_cost")}, out


@pytest.mark.parametrize("name", sorted(SCENES))
def test_fused_linearisation_matches_plane_kernels(name):
    make, max_its = SCENES[name]
    pb = make()
    sf, df = _run(pb, (), max_its)
    sg, dg = _run(pb, ("generic_linearize",), max_its)
    # Iteration 1 linearises at the input parameters: only summation orders differ.  The Jacobi scale is fixed by that
    # linearisation.  Iteration 2 linearises after one step, whose parameters already differ by the rounding of the
    # Schur atomics and the PCG (two runs of the same build differ there too), so its diagonal and gradient get 1e-8.
    for it, tol in ((1, 1e-12), (2, 1e-8)):
        a, b = df["scale%d" % it], dg["scale%d" % it]
        assert np.max(np.abs(a - b) / np.abs(b)) <= 1e-12, ("scale", it)
        a, b = df["diag%d" % it], dg["diag%d" % it]
        assert np.max(np.abs(a - b) / np.abs(b)) <= tol, ("diag", it)
        a, b = df["grad%d" % it], dg["grad%d" % it]
        assert np.max(np.abs(a - b)) <= tol * np.max(np.abs(b)), ("grad", it)
    print("%s fused: %s | plane kernels: %s" % (name, sf, sg))
    assert sf["iterations"] == sg["iterations"] and sf["termination"] == sg["termination"]
    assert abs(sf["final_cost"] - sg["final_cost"]) <= 1e-9 * sg["final_cost"]
    for k in ("cam_params", "inst", "points"):
        assert np.abs(df[k] - dg[k]).max() <= 1e-6, k
