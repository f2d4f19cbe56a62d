"""Rig-instance covariances through BundleAdjuster on the reference's own bundle scenes (opensfm/test/test_bundle.py:
test_pair, test_pair_with_points_priors, test_four_cams_one_fixed; built as in tests/test_bundle_reference.py).
These add what the synthetic covariance scenes lack: relative motions with reconstruction-scale ext blocks, point
priors, problems with no points at all.

Oracle backend (CPU): the CPU restatement (tests/covariance_oracle.py) fed through BundleAdjuster.apply_results; its
instance blocks are checked against a dense numpy inverse of the scaled normal equations formed from the oracle's
undamped reduced system.  CUDA backend (GPU): get_covariance_estimation_valid / get_rig_instance_covariance against
the restatement at the engine's own parameters, to 10 * 5e-12 * cond2(S) of sqrt(C_ii C_jj) (as in
tests/test_ba_covariance_gpu.py), and against the oracle backend's getters."""
import numpy as np
import pytest

import covariance_oracle as co
from opensfm_b200 import bundle
from opensfm_b200 import types as T
from opensfm_b200.bundle import RelativeMotion
from test_bundle_reference import _four_cams, create_shots

IDS = {"pair": "12", "pair_with_points_priors": "12", "four_cams_one_fixed": "1234"}
# the free pair keeps the rotation about its baseline in the null space of J: the reference's default, invalid
VALID = {"pair": False, "pair_with_points_priors": True, "four_cams_one_fixed": True}


def build(name):
    ba = bundle.BundleAdjuster()
    camera = T.Camera.create_perspective(1.0, 0.0, 0.0)
    ba.add_camera("cam1", camera, camera, True)
    ba.add_rig_camera("rig_cam1", T.Pose(), T.Pose(), True)
    if name == "pair":
        create_shots(ba, 2)
        ba.add_reconstruction("12", False)
        ba.add_reconstruction_instance("12", 4, "1")
        ba.add_reconstruction_instance("12", 4, "2")
        ba.set_scale_sharing("12", True)
        ba.add_relative_motion(RelativeMotion("1", "2", np.array([0, 0, 0]), np.array([-1, 0, 0]), 1, 1, False))
        ba.add_rig_instance_position_prior("1", np.array([0, 0, 0]), np.array([1, 1, 1]), "")
        ba.add_rig_instance_position_prior("2", np.array([2, 0, 0]), np.array([1, 1, 1]), "")
    elif name == "pair_with_points_priors":
        for i in range(2):
            iid = str(i + 1)
            ba.add_rig_instance(iid, T.Pose(np.array([1e-3, 1e-3, 1e-3]), np.array([1e-3, 1e-3, 1e-3])), {iid: "cam1"},
                                {iid: "rig_cam1"}, False)
        ba.add_point("p1", np.array([0, 0, 0]), False)
        ba.add_point("p2", np.array([0, 0, 0]), False)
        ba.add_reconstruction("12", False)
        ba.add_reconstruction_instance("12", 4, "1")
        ba.add_reconstruction_instance("12", 4, "2")
        ba.add_absolute_roll("1", np.radians(90), 1)
        ba.add_absolute_pan("1", -np.radians(90), 1)
        ba.add_absolute_tilt("1", -np.radians(90), 1)
        ba.set_scale_sharing("12", True)
        ba.add_relative_motion(RelativeMotion("1", "2", np.array([0, 0, 0]), np.array([-1, 0, 0]), 1, 1, False))
        sd = np.array([1, 1, 1])
        ba.add_point_projection_observation(shot="1", point="p1", observation=np.array([0, 0]), std_deviation=1)
        ba.add_point_projection_observation(shot="2", point="p1", observation=np.array([-0.5, 0]), std_deviation=1)
        ba.add_point_prior("p1", np.array([-0.5, 2, 2]), sd, True)
        ba.add_point_projection_observation(shot="2", point="p2", observation=np.array([0, 0]), std_deviation=1)
        ba.add_point_projection_observation(shot="1", point="p2", observation=np.array([0.5, 0]), std_deviation=1)
        ba.add_point_prior("p2", np.array([1.5, 2, 2]), sd, True)
    else:
        for i in range(4):
            iid = str(i + 1)
            ba.add_rig_instance(iid, T.Pose(np.array([0, 0, 0]), np.array([0, 0, 0])), {iid: "cam1"}, {iid: "rig_cam1"},
                                i == 0)
        _four_cams(ba, [100, 0, 0])
    ba.set_compute_covariances(True)
    return ba


def run_oracle(ba):
    pb = ba.to_problem()
    ba.apply_results(pb, co.solve(pb))
    return pb


def getters(ba, name):
    return ba.get_covariance_estimation_valid(), np.array([ba.get_rig_instance_covariance(i) for i in IDS[name]])


def dense_reference(pb, params):
    """Instance blocks of the inverse of the oracle's undamped, scaled S (numpy.linalg.inv, no pivot rule)."""
    valid, _, C, info = co.covariances(pb, params)
    assert valid
    S, s = info["S"], info["scale"]
    m = 6 * int(np.sum(np.asarray(pb.inst_const) == 0))
    Ci = np.linalg.inv(S)[-m:, -m:] * s[-m:, None] * s[None, -m:]
    ref = np.zeros_like(C)
    for q, i in enumerate(np.flatnonzero(np.asarray(pb.inst_const) == 0)):
        ref[i] = Ci[6 * q:6 * q + 6, 6 * q:6 * q + 6]
    return C, ref, np.linalg.cond(S)


@pytest.mark.parametrize("name", sorted(IDS))
def test_oracle_backend(name):
    ba = build(name)
    pb = run_oracle(ba)
    valid, C = getters(ba, name)
    assert valid == VALID[name]
    if not valid:
        assert np.array_equal(C, np.tile(co.DEFAULT, (len(C), 1, 1)))
        return
    pb_, res = ba.results()
    Cr, ref, kappa = dense_reference(pb, (res["cam_params"], res["inst"], res["rigcam"], res["points"], res["ext_values"]))
    assert np.array_equal(C, Cr)
    free = np.asarray(pb.inst_const) == 0
    d = np.sqrt(np.abs(np.einsum("ijj->ij", ref)))
    worst = (np.abs(C - ref) / (d[:, :, None] * d[:, None, :]))[free].max()
    print("%s: cond2(S) %.2e, worst |C - C_ref| / sqrt(C_ii C_jj) %.2e" % (name, kappa, worst))
    assert worst <= 1e-10
    for i in np.flatnonzero(pb.inst_const):
        assert np.all(C[i] == 0.0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(IDS))
def test_cuda_backend_matches_oracle(name):
    ba = build(name)
    ba.run()
    valid, C = getters(ba, name)
    pb, res = ba.results()
    valid_o, status_o, C_o, info = co.covariances(pb, (res["cam_params"], res["inst"], res["rigcam"], res["points"],
                                                       res["ext_values"]))
    assert valid == valid_o == VALID[name] and res["covariance_status"] == status_o
    ob = build(name)
    run_oracle(ob)
    valid_b, C_b = getters(ob, name)
    assert valid_b == valid
    if not valid:
        assert np.array_equal(C, C_o) and np.array_equal(C, C_b)
        return
    free = np.asarray(pb.inst_const) == 0
    assert np.all(C[~free] == 0.0)
    d = np.sqrt(np.abs(np.einsum("ijj->ij", C_o)))
    den = d[:, :, None] * d[:, None, :]
    kappa = np.linalg.cond(info["S"])
    worst = (np.abs(C - C_o) / den)[free].max()
    # the two backends converge to the same solution within the reference's 1e-6 pose tolerance; the covariance
    # moves with it at first order
    worst_b = (np.abs(C - C_b) / den)[free].max()
    print("%s: cond2(S) %.2e, engine vs restatement %.2e (bound %.2e), vs oracle backend %.2e"
          % (name, kappa, worst, 10 * 5e-12 * kappa, worst_b))
    assert worst <= 10 * 5e-12 * kappa
    assert worst_b <= 1e-4
