"""The reference's own known-answer tests of `pybundle.BundleAdjuster` (opensfm/test/test_bundle.py), ported
assertion for assertion (same inputs, same tolerances) and run twice: against the BA oracle on the CPU and
against the CUDA engine.  These are the only vectors the reference holds that pin the *solver* end to end
(pose / scale recovery to 1e-6), so they are what ties the oracle's restated Levenberg-Marquardt and its
secondary residual functors to the reference (SURVEY.md §8c), and the CUDA path to both.

Reference test -> test here (file:line in OpenSfM's opensfm/test/test_bundle.py):
  test_unicode_strings_in_bundle :20-34, test_sigleton :46-72, test_singleton_pan_tilt_roll :75-106,
  test_pair :181-219, test_pair_with_points_priors :222-316, test_pair_non_rigid :319-352,
  test_four_cams_single_reconstruction :355-417, test_four_cams_double_reconstruction :420-500,
  test_four_cams_one_fixed :503-574, test_linear_motion_prior_position :577-600,
  test_linear_motion_prior_rotation :603-638.
(test_heatmaps_position needs ceres::BiCubicInterpolator: not part of this engine; the three tests that go through
reconstruction.bundle() are in tests/test_reconstruction_bundle.py.)"""
import numpy as np
import pytest

from oracle import ba_lm as oracle
from opensfm_b200 import bundle
from opensfm_b200 import types as T
from opensfm_b200.bundle import RelativeMotion

BACKENDS = [pytest.param("oracle", id="oracle"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


def run(ba: bundle.BundleAdjuster, backend: str):
    """`ba.run()` on the chosen backend."""
    if backend == "cuda":
        ba.run()
        return
    pb = ba.to_problem()
    res = oracle.solve(pb)
    res["summary"] = {"iterations": res["iterations"], "initial_cost": res["initial_cost"],
                      "final_cost": res["final_cost"], "termination": res["termination"]}
    ba.apply_results(pb, res)


def ptr_from_rotation(R):
    """opensfm/geometry.py ptr_from_rotation (pan, tilt, roll of a world-to-camera rotation matrix)."""
    Rt_ex, Rt_ez = R.T @ [1.0, 0, 0], R.T @ [0, 0, 1.0]
    pan = np.arctan2(Rt_ez[0], Rt_ez[1])
    tilt = -np.arctan2(Rt_ez[2], np.hypot(Rt_ez[0], Rt_ez[1]))
    a = np.array([Rt_ez[1], -Rt_ez[0], 0.0])
    a /= np.linalg.norm(a)
    roll = np.arcsin(np.dot(Rt_ez, np.cross(Rt_ex, a)))
    return pan, tilt, roll


def test_unicode_strings_in_bundle():
    ba = bundle.BundleAdjuster()
    camera = T.Camera.create_perspective(0.4, 0.1, -0.01)
    ba.add_camera("A\xb2", camera, camera, True)
    ba.add_camera(b"A_2", camera, camera, True)


@pytest.fixture()
def bundle_adjuster():
    ba = bundle.BundleAdjuster()
    camera = T.Camera.create_perspective(1.0, 0.0, 0.0)
    ba.add_camera("cam1", camera, camera, True)
    ba.add_rig_camera("rig_cam1", T.Pose(), T.Pose(), True)
    return ba


@pytest.mark.parametrize("backend", BACKENDS)
def test_sigleton(bundle_adjuster, backend):
    sa = bundle_adjuster
    sa.add_rig_instance("1", T.Pose(np.array([0.5, 0, 0]), np.array([0, 0, 0])), {"1": "cam1"}, {"1": "rig_cam1"}, False)
    sa.add_rig_instance_position_prior("1", np.array([1, 0, 0]), np.array([1, 1, 1]), "")
    sa.add_absolute_up_vector("1", np.array([0, -1, 0]), 1)
    sa.add_absolute_pan("1", np.radians(180), 1)
    run(sa, backend)
    s1 = sa.get_rig_instance_pose("1")
    assert np.allclose(s1.translation, [1, 0, 0], atol=1e-6)


@pytest.mark.parametrize("backend", BACKENDS)
def test_singleton_pan_tilt_roll(bundle_adjuster, backend):
    pan, tilt, roll = 1, 0.3, 0.2
    sa = bundle_adjuster
    sa.add_rig_instance("1", T.Pose(np.array([0.5, 0, 0]), np.array([0, 0, 0])), {"1": "cam1"}, {"1": "rig_cam1"}, False)
    sa.add_rig_instance_position_prior("1", np.array([1, 0, 0]), np.array([1, 1, 1]), "")
    sa.add_absolute_pan("1", pan, 1)
    sa.add_absolute_tilt("1", tilt, 1)
    sa.add_absolute_roll("1", roll, 1)
    run(sa, backend)
    pose = sa.get_rig_instance_pose("1")
    assert np.allclose(pose.get_origin(), [1, 0, 0], atol=1e-6)
    assert np.allclose(ptr_from_rotation(pose.get_rotation_matrix()), (pan, tilt, roll))


def create_shots(ba, num_shots):
    for i in range(num_shots):
        instance_id = str(i + 1)
        ba.add_rig_instance(instance_id, T.Pose(np.array([0, 0, 0]), np.array([0, 0, 0])), {instance_id: "cam1"},
                            {instance_id: "rig_cam1"}, False)


@pytest.mark.parametrize("backend", BACKENDS)
def test_pair(bundle_adjuster, backend):
    sa = bundle_adjuster
    create_shots(sa, 2)
    sa.add_reconstruction("12", False)
    sa.add_reconstruction_instance("12", 4, "1")
    sa.add_reconstruction_instance("12", 4, "2")
    sa.set_scale_sharing("12", True)
    sa.add_relative_motion(RelativeMotion("1", "2", np.array([0, 0, 0]), np.array([-1, 0, 0]), 1, 1, False))
    std_dev = np.array([1, 1, 1])
    sa.add_rig_instance_position_prior("1", np.array([0, 0, 0]), std_dev, "")
    sa.add_rig_instance_position_prior("2", np.array([2, 0, 0]), std_dev, "")
    run(sa, backend)
    s1, s2 = sa.get_rig_instance_pose("1"), sa.get_rig_instance_pose("2")
    r12 = sa.get_reconstruction("12")
    assert np.allclose(s1.translation, [0, 0, 0], atol=1e-6)
    assert np.allclose(s2.translation, [-2, 0, 0], atol=1e-6)
    assert np.allclose(r12.get_scale("1"), 0.5)
    assert np.allclose(r12.get_scale("2"), 0.5)


@pytest.mark.parametrize("backend", BACKENDS)
def test_pair_with_points_priors(bundle_adjuster, backend):
    sa = bundle_adjuster
    for i in range(2):
        instance_id = str(i + 1)
        sa.add_rig_instance(instance_id, T.Pose(np.array([1e-3, 1e-3, 1e-3]), np.array([1e-3, 1e-3, 1e-3])),
                            {instance_id: "cam1"}, {instance_id: "rig_cam1"}, False)
    sa.add_point("p1", np.array([0, 0, 0]), False)
    sa.add_point("p2", np.array([0, 0, 0]), False)
    sa.add_reconstruction("12", False)
    sa.add_reconstruction_instance("12", 4, "1")
    sa.add_reconstruction_instance("12", 4, "2")
    # identity rotation with pan/tilt/roll
    sa.add_absolute_roll("1", np.radians(90), 1)
    sa.add_absolute_pan("1", -np.radians(90), 1)
    sa.add_absolute_tilt("1", -np.radians(90), 1)
    sa.set_scale_sharing("12", True)
    sa.add_relative_motion(RelativeMotion("1", "2", np.array([0, 0, 0]), np.array([-1, 0, 0]), 1, 1, False))
    std_dev = np.array([1, 1, 1])
    sa.add_point_projection_observation(shot="1", point="p1", observation=np.array([0, 0]), std_deviation=1)
    sa.add_point_projection_observation(shot="2", point="p1", observation=np.array([-0.5, 0]), std_deviation=1)
    sa.add_point_prior("p1", np.array([-0.5, 2, 2]), std_dev, True)
    sa.add_point_projection_observation(shot="2", point="p2", observation=np.array([0, 0]), std_deviation=1)
    sa.add_point_projection_observation(shot="1", point="p2", observation=np.array([0.5, 0]), std_deviation=1)
    sa.add_point_prior("p2", np.array([1.5, 2, 2]), std_dev, True)
    run(sa, backend)
    s1, s2 = sa.get_rig_instance_pose("1"), sa.get_rig_instance_pose("2")
    r12 = sa.get_reconstruction("12")
    p1, p2 = sa.get_point("p1"), sa.get_point("p2")
    assert np.allclose(s1.translation, [0.5, -2, 2], atol=1e-2)
    assert np.allclose(s2.translation, [-1.5, -2, 2], atol=1e-2)
    assert np.allclose(p1.p, [-0.5, 2, 2], atol=1e-6)
    assert np.allclose(p2.p, [1.5, 2, 2], atol=1e-6)
    assert np.allclose(r12.get_scale("1"), 0.5)
    assert np.allclose(r12.get_scale("2"), 0.5)


@pytest.mark.parametrize("backend", BACKENDS)
def test_pair_non_rigid(bundle_adjuster, backend):
    sa = bundle_adjuster
    create_shots(sa, 2)
    sa.add_reconstruction("12", False)
    sa.add_reconstruction_instance("12", 4, "1")
    sa.add_reconstruction_instance("12", 4, "2")
    sa.set_scale_sharing("12", False)
    sa.add_relative_motion(RelativeMotion("1", "2", np.array([0, 0, 0]), np.array([-1, 0, 0]), 1, 1, False))
    std_dev = np.array([1, 1, 1])
    sa.add_rig_instance_position_prior("1", np.array([0, 0, 0]), std_dev, "")
    sa.add_rig_instance_position_prior("2", np.array([2, 0, 0]), std_dev, "")
    run(sa, backend)
    s1, s2 = sa.get_rig_instance_pose("1"), sa.get_rig_instance_pose("2")
    r12 = sa.get_reconstruction("12")
    assert np.allclose(s1.translation, [0, 0, 0], atol=1e-6)
    assert np.allclose(s2.translation, [-2, 0, 0], atol=1e-6)
    assert np.allclose(r12.get_scale("1"), 4.0)
    assert np.allclose(r12.get_scale("2"), 0.5)


def _four_cams(sa, origin_prior):
    sa.add_reconstruction("1234", False)
    for i in "1234":
        sa.add_reconstruction_instance("1234", 1, i)
    sa.set_scale_sharing("1234", True)
    for j, t in (("2", [-1, 0, 0]), ("3", [0, -1, 0]), ("4", [0, 0, -1])):
        sa.add_relative_motion(RelativeMotion("1", j, np.array([0, 0, 0]), np.array(t), 1, 1, False))
    std_dev = np.array([1, 1, 1])
    sa.add_rig_instance_position_prior("1", np.array(origin_prior), std_dev, "")
    sa.add_rig_instance_position_prior("2", np.array([2, 0, 0]), std_dev, "")
    sa.add_rig_instance_position_prior("3", np.array([0, 2, 0]), std_dev, "")


def _check_four(sa):
    s = [sa.get_rig_instance_pose(i) for i in "1234"]
    assert np.allclose(s[0].translation, [0, 0, 0], atol=1e-6)
    assert np.allclose(s[1].translation, [-2, 0, 0], atol=1e-6)
    assert np.allclose(s[2].translation, [0, -2, 0], atol=1e-6)
    assert np.allclose(s[3].translation, [0, 0, -2], atol=1e-6)


@pytest.mark.parametrize("backend", BACKENDS)
def test_four_cams_single_reconstruction(bundle_adjuster, backend):
    sa = bundle_adjuster
    create_shots(sa, 4)
    _four_cams(sa, [0, 0, 0])
    run(sa, backend)
    _check_four(sa)


@pytest.mark.parametrize("backend", BACKENDS)
def test_four_cams_double_reconstruction(bundle_adjuster, backend):
    sa = bundle_adjuster
    create_shots(sa, 4)
    sa.add_reconstruction("12", False)
    sa.add_reconstruction_instance("12", 1, "1")
    sa.add_reconstruction_instance("12", 1, "2")
    sa.set_scale_sharing("12", False)
    sa.add_reconstruction("34", False)
    sa.add_reconstruction_instance("34", 1, "3")
    sa.add_reconstruction_instance("34", 1, "4")
    sa.set_scale_sharing("34", False)
    z = np.array([0, 0, 0])
    sa.add_relative_motion(RelativeMotion("1", "2", z, np.array([-0.5, -0.5, -0.5]), 1, 1, True))
    sa.add_relative_motion(RelativeMotion("3", "2", z, np.array([0.5, 0.5, 0.5]), 1, 1, False))
    sa.add_relative_motion(RelativeMotion("3", "4", z, np.array([-2, -2, -2]), 1, 1, True))
    sa.add_relative_motion(RelativeMotion("2", "3", z, np.array([-2, -2, -2]), 1, 1, False))
    std_dev = np.array([1, 1, 1])
    sa.add_rig_instance_position_prior("1", np.array([0, 0, 0]), std_dev, "")
    sa.add_rig_instance_position_prior("4", np.array([3, 3, 3]), std_dev, "")
    run(sa, backend)
    s = [sa.get_rig_instance_pose(i) for i in "1234"]
    for k in range(4):
        assert np.allclose(s[k].get_origin(), [k, k, k], atol=1e-6)
    r12 = sa.get_reconstruction("12")
    assert np.allclose(r12.get_scale("1"), 0.5)
    assert np.allclose(r12.get_scale("2"), 0.5)
    r34 = sa.get_reconstruction("34")
    assert np.allclose(r34.get_scale("3"), 2.0)
    assert np.allclose(r34.get_scale("4"), 2.0)


@pytest.mark.parametrize("backend", BACKENDS)
def test_four_cams_one_fixed(bundle_adjuster, backend):
    sa = bundle_adjuster
    for i in range(4):
        instance_id = str(i + 1)
        sa.add_rig_instance(instance_id, T.Pose(np.array([0, 0, 0]), np.array([0, 0, 0])), {instance_id: "cam1"},
                            {instance_id: "rig_cam1"}, i == 0)
    _four_cams(sa, [100, 0, 0])
    run(sa, backend)
    _check_four(sa)


@pytest.mark.parametrize("backend", BACKENDS)
def test_linear_motion_prior_position(bundle_adjuster, backend):
    sa = bundle_adjuster
    create_shots(sa, 3)
    sa.add_reconstruction("123", False)
    for i in "123":
        sa.add_reconstruction_instance("123", 1, i)
    sa.set_scale_sharing("123", True)
    std_dev = np.array([1, 1, 1])
    sa.add_rig_instance_position_prior("1", np.array([0, 0, 0]), std_dev, "")
    sa.add_rig_instance_position_prior("3", np.array([2, 0, 0]), std_dev, "")
    sa.add_linear_motion("1", "2", "3", 0.5, 0.1, 0.1)
    run(sa, backend)
    s1, s2, s3 = (sa.get_rig_instance_pose(i) for i in "123")
    assert np.allclose(s1.translation, [0, 0, 0], atol=1e-6)
    assert np.allclose(s2.translation, [-1, 0, 0], atol=1e-6)
    assert np.allclose(s3.translation, [-2, 0, 0], atol=1e-6)


@pytest.mark.parametrize("backend", BACKENDS)
def test_linear_motion_prior_rotation(bundle_adjuster, backend):
    sa = bundle_adjuster
    sa.add_rig_instance("1", T.Pose(np.array([0, 0, 0]), np.array([0, 0, 0])), {"1": "cam1"}, {"1": "rig_cam1"}, True)
    sa.add_rig_instance("2", T.Pose(np.array([0, 0, 0]), np.array([0, 0, 0])), {"2": "cam1"}, {"2": "rig_cam1"}, False)
    sa.add_rig_instance("3", T.Pose(np.array([0, 1, 0]), np.array([0, 0, 0])), {"3": "cam1"}, {"3": "rig_cam1"}, True)
    sa.add_reconstruction("123", False)
    for i in "123":
        sa.add_reconstruction_instance("123", 1, i)
    sa.set_scale_sharing("123", True)
    sa.add_linear_motion("1", "2", "3", 0.3, 0.1, 0.1)
    run(sa, backend)
    s2 = sa.get_rig_instance_pose("2")
    assert np.allclose(s2.rotation, [0, 0.3, 0], atol=1e-6)


# ---- terms the reference tests do not reach: CUDA vs oracle on the same problem -------------------------------
def _rig_scene():
    """Two-camera rig, free rig camera with its pose prior, GPS priors through a free camera bias with an adjusted
    std-deviation group, a gauge fix, common-position and relative-rotation terms, a DUAL camera (barrier)."""
    rng = np.random.RandomState(7)
    ba = bundle.BundleAdjuster()
    cam = T.Camera.create_perspective(0.9, -0.05, 0.01)
    dual = T.Camera.create_dual(0.4, 0.8, -0.03, 0.005)
    ba.add_camera("c0", cam, cam, False)
    ba.add_camera("c1", dual, dual, False)
    ba.set_internal_parameters_prior_sd(0.01, 0.01, 0.01, 0.01, 0.01, 0.01, 0.01, 0.01, 0.01)
    ba.add_rig_camera("rc0", T.Pose(), T.Pose(), True)
    rc1 = T.Pose.from_ba_params([0.02, -0.03, 0.01, 0.2, 0.0, 0.02])
    ba.add_rig_camera("rc1", rc1, T.Pose.from_ba_params([0.0, 0.0, 0.0, 0.2, 0.0, 0.0]), False)
    ba.set_rig_parameters_prior_sd(0.1, 0.1)
    pts = rng.uniform(-0.5, 0.5, (150, 3))
    NI = 5
    truth = []
    for i in range(NI):
        ang = 2 * np.pi * i / NI
        origin = 2.5 * np.array([np.cos(ang), np.sin(ang), 0.1 * i])
        ez = -origin / np.linalg.norm(origin)
        ex = np.cross(ez, [0, 0, 1.0]); ex /= np.linalg.norm(ex)
        ey = np.cross(ez, ex)
        pose = T.Pose()
        pose.set_rotation_matrix(np.array([ex, ey, ez]))
        pose.set_origin(origin)
        truth.append(pose)
        noisy = T.Pose.from_ba_params(pose.to_ba_params() + rng.normal(0, 0.01, 6))
        ba.add_rig_instance("i%d" % i, noisy, {"s%da" % i: "c0", "s%db" % i: "c1"}, {"s%da" % i: "rc0", "s%db" % i: "rc1"}, False)
        ba.add_rig_instance_position_prior("i%d" % i, origin + rng.normal(0, 0.02, 3) + [0.05, 0, 0], np.full(3, 0.05), "g")
    ba.set_camera_bias("c0", [0, 0, 0], [0, 0, 0], 1.0)
    ba.set_adjust_absolute_position_std(True)
    for p in range(len(pts)):
        ba.add_point("p%d" % p, pts[p] + rng.normal(0, 0.01, 3), False)
    from oracle import ba_lm
    for i in range(NI):
        for suffix, camobj, ctype, rcp in (("a", cam, 0, np.zeros(6)), ("b", dual, 7, rc1.to_ba_params())):
            for p in range(len(pts)):
                xi = truth[i].get_rotation_matrix() @ pts[p] + truth[i].translation
                R = T.Pose.from_ba_params(rcp)
                xc = R.get_rotation_matrix() @ xi + R.translation
                if xc[2] < 0.5:
                    continue
                px = ba_lm.project(ctype, camobj.get_parameters_values(), xc)
                ba.add_point_projection_observation("s%d%s" % (i, suffix), "p%d" % p, px + rng.normal(0, 5e-4, 2), 0.004)
    ba.add_common_position("s0a", "s0b", 0.01, 0.05)
    rr = bundle.RelativeRotation("s1a", "s2b", [0.0, 0.0, 0.3])
    ba.add_relative_rotation(rr)
    ba.add_absolute_up_vector("s3b", [0, 0, -1], 0.5)
    ba.set_gauge_fix_shots("s0a", "s2a")
    ba.set_point_projection_loss_function("SoftLOneLoss", 1.0)
    ba.set_max_num_iterations(50)
    return ba


@pytest.mark.gpu
def test_rig_bias_scale_group_gauge_terms_match_oracle():
    ba = _rig_scene()
    pb = ba.to_problem()
    types = sorted({t.type for t in pb.side_terms})
    assert len(types) >= 6
    ref = oracle.solve(pb)
    got = bundle.solve(pb)
    s = got["summary"]
    assert abs(s["initial_cost"] - ref["initial_cost"]) <= 1e-9 * ref["initial_cost"]
    assert abs(s["final_cost"] - ref["final_cost"]) <= 1e-6 * ref["final_cost"], (s["final_cost"], ref["final_cost"])
    for k in ("points", "inst", "cam_params", "rigcam", "ext_values"):
        assert np.abs(got[k] - ref[k]).max() < 5e-5, k
