"""The engine's rig-instance covariances (bundle.solve(compute_covariances=True), ba_cov.cuh) against the CPU
restatement of tests/covariance_oracle.py, evaluated at the parameters the engine returned (LM trajectories do not
enter).  Per scene: equal validity and status; constant instances exactly zero; invalid runs exactly the default
matrix; valid runs |C_e - C_o|_ij <= 10 * 5e-12 * cond2(S_o) * sqrt(C_o,ii C_o,jj) -- the first-order bound from the
agreement of the reduced systems (5e-12, tests/test_ba_linear_system_gpu.py), S_o the oracle's scaled S.  The
solve is the same with covariances on and off (iterations, termination; cost and parameters within the run-to-run
spread of the Schur atomics that two unarmed solves show as well).  The scenes also
run on every fallback path (bundle.solve(fallbacks=...))."""
import json

import numpy as np
import pytest

import ba_linear_system_scenes as scenes
import covariance_oracle as co
from opensfm_b200 import bundle
from test_ba_linear_system_gpu import VARIANTS
from test_covariance_reference import gps_cube_constant_instances, point_seen_once

pytestmark = pytest.mark.gpu

S_TAU = 5e-12


def gps_cube(num_cameras=500, num_points=20000):
    """500 cameras with GPS priors on every instance, ~20k points: n_c = 4500, m = 3000 (not a multiple of the
    64-wide Cholesky blocks), 71 panels."""
    pb = scenes.cube(num_cameras, num_points, max_obs=8)
    rng = np.random.RandomState(11)
    pb.inst_has_prior[:] = 1
    pb.inst_prior_pos = pb.inst[:, 3:] + rng.normal(0, 0.02, (len(pb.inst), 3))
    pb.inst_prior_std = np.full((len(pb.inst), 3), 0.05)
    pb.max_iterations = 20
    return pb


# point_seen_once: the gauge is fixed, so the reduced system passes its pivot test; only the point-side rank rule
# makes the estimate invalid (and the engine must still return exactly the default matrices)
SCENES = dict(scenes.SCENES, gps_cube_constant_instances=gps_cube_constant_instances, point_seen_once=point_seen_once,
              gps_cube_500=gps_cube)
FULL_RANK = {"camera_and_position_priors", "fixed_instances", "point_priors_many_obs", "gps_cube_constant_instances",
             "gps_cube_500"}


def measure(name, fallbacks=()):
    pb = SCENES[name]()
    on = bundle.solve(pb, compute_covariances=True, fallbacks=fallbacks)
    off = bundle.solve(pb, fallbacks=fallbacks)
    off2 = bundle.solve(pb, fallbacks=fallbacks)

    def apart(a, b):
        return max(float(np.abs(a[k] - b[k]).max()) if np.size(a[k]) else 0.0
                   for k in ("cam_params", "inst", "rigcam", "points", "ext_values"))

    # the pass runs after the LM loop and writes none of the returned buffers, so on and off differ only by the
    # run-to-run spread of the Schur atomics, which two unarmed solves (off, off2) show as well.  Measured on an H100
    # over every scene and variant: equal iterations and termination; between two unarmed solves parameters up to
    # 9.0e-6 apart (gauge-free scenes drift along the gauge) and costs up to 3.8e-9 relative, on vs off the same.
    # The bars are twice that.
    diff, spread = apart(on, off), apart(off, off2)
    sm_on, sm_off = on["summary"], off["summary"]
    cost_rel = abs(sm_on["final_cost"] - sm_off["final_cost"]) / sm_off["final_cost"]
    same = (diff <= 2e-5 and sm_on["termination"] == sm_off["termination"]
            and sm_on["iterations"] == sm_off["iterations"] and cost_rel <= 1e-8)
    params = (on["cam_params"], on["inst"], on["rigcam"], on["points"], on["ext_values"])
    valid, status, C, info = co.covariances(pb, params, termination=on["summary"]["termination"])
    Ce = on["covariances"]
    m = {"name": name, "same_on_off": bool(same), "on_off_param_diff": diff, "off_off_param_diff": spread,
         "on_off_cost_rel": cost_rel, "iterations": [sm_on["iterations"], sm_off["iterations"], off2["summary"]["iterations"]],
         "valid": on["covariance_valid"],
         "status": on["covariance_status"], "valid_o": valid, "status_o": status, "termination": on["summary"]["termination"]}
    const = np.asarray(pb.inst_const) != 0
    pass_ms, chol_ms = on["covariance_ms"]   # device times of the pass and of its Cholesky factorisation
    m["timing_ok"] = bool(np.isfinite([pass_ms, chol_ms]).all() and pass_ms > 0.0 and chol_ms >= 0.0)
    m["const_zero"] = bool(np.all(Ce[const] == 0.0)) if valid else True
    m["default_exact"] = bool(np.array_equal(Ce, np.tile(co.DEFAULT, (len(pb.inst), 1, 1)))) if not on["covariance_valid"] else True
    m["ratio"] = 0.0
    if valid and on["covariance_valid"] and (~const).any():
        kappa = np.linalg.cond(info["S"])
        d = np.sqrt(np.abs(np.einsum("ijj->ij", C)))
        den = (d[:, :, None] * d[:, None, :])[~const]
        m["kappa"] = float(kappa)
        m["ratio"] = float((np.abs(Ce - C)[~const] / den).max() / (10 * S_TAU * kappa))
        m["worst_rel"] = float((np.abs(Ce - C)[~const] / den).max())
    return m


def _check(m):
    print(json.dumps(m))
    assert m["valid"] == m["valid_o"] and m["status"] == m["status_o"], m
    assert m["const_zero"] and m["default_exact"] and m["timing_ok"], m
    assert m["ratio"] <= 1.0, m
    if m["name"] in FULL_RANK:
        assert m["valid"], m
    assert m["same_on_off"], m


@pytest.mark.parametrize("name", sorted(SCENES))
def test_covariances_match_oracle(name):
    _check(measure(name))


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_covariances_under_kernel_variant(variant):
    for name in sorted(scenes.SCENES):
        _check(measure(name, VARIANTS[variant]))


def test_bundle_adjuster_end_to_end():
    """BundleAdjuster with GPS priors: get_covariance_estimation_valid / get_rig_instance_covariance against the
    restatement at the returned parameters; a free problem (no priors) reports the default, invalid."""
    from opensfm_b200 import types as T

    pb0 = scenes.cube(8, 300, max_obs=5)
    for gps in (True, False):
        ba = bundle.BundleAdjuster()
        off = pb0.cam_off
        for k in range(len(pb0.cam_type)):
            vals = pb0.cam_params[off[k]:off[k + 1]]
            ba.add_camera("c%d" % k, T.Camera("perspective", vals), T.Camera("perspective", vals), False)
        ba.add_rig_camera("rc", T.Pose(), T.Pose(), True)
        for i in range(len(pb0.inst)):
            ba.add_rig_instance("i%d" % i, T.Pose.from_ba_params(pb0.inst[i]), {"s%d" % i: "c%d" % i},
                                {"s%d" % i: "rc"}, i == 0)
            if gps:
                ba.add_rig_instance_position_prior("i%d" % i, pb0.inst[i, 3:] + 0.01, [0.05] * 3)
        ba.add_points_bulk(["p%d" % p for p in range(len(pb0.points))], pb0.points, False)
        ba.add_observations_bulk(["s%d" % s for s in pb0.obs_shot], ["p%d" % p for p in pb0.obs_point], pb0.obs_xy,
                                 pb0.obs_sigma)
        ba.set_compute_covariances(True)
        ba.run()
        pb, res = ba.results()
        valid, status, C, info = co.covariances(pb, (res["cam_params"], res["inst"], res["rigcam"], res["points"],
                                                     res["ext_values"]))
        assert ba.get_covariance_estimation_valid() == valid == gps   # free: the similarity scale stays in the null space
        got = np.array([ba.get_rig_instance_covariance("i%d" % i) for i in range(len(pb0.inst))])
        if not valid:
            assert np.array_equal(got, C)
            continue
        assert np.all(got[0] == 0.0)   # the constant instance
        d = np.sqrt(np.abs(np.einsum("ijj->ij", C[1:])))
        worst = (np.abs(got[1:] - C[1:]) / (d[:, :, None] * d[:, None, :])).max()
        assert worst <= 10 * S_TAU * np.linalg.cond(info["S"]), worst


def test_distributed_covariances_raise_before_any_allreduce():
    calls = []
    pb = scenes.camera_and_position_priors()
    with pytest.raises(ValueError, match="world == 1"):
        bundle.solve(pb, rank=0, world=2, allreduce=lambda ptr, count, strm: calls.append(count),
                     compute_covariances=True)
    assert calls == []
