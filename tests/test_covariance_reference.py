"""Rig-instance covariances of the CPU restatement (tests/covariance_oracle.py) against a dense numpy (J^T J)^-1,
scene by scene, plus the host logic of the covariance interface.  The dense J is the one of
tests/test_reduced_system_reference.py (dual-number observation blocks, prior rows)."""
import numpy as np
import pytest

import ba_linear_system_scenes as scenes
import covariance_oracle as co
from oracle import ba_lm as oracle
from test_reduced_system_reference import _layout, reference_system


def gps_cube_constant_instances():
    """A cube with GPS priors on every instance and three constant instances."""
    pb = scenes.camera_and_position_priors()
    pb.inst_const[[0, 4, 7]] = 1
    return pb


def point_seen_once():
    """A full-rank scene in which one free point keeps a single observation: its V has rank 2."""
    pb = scenes.camera_and_position_priors()
    p = int(np.bincount(pb.obs_point).argmax())
    idx = np.flatnonzero(pb.obs_point == p)
    keep = np.ones(len(pb.obs_point), dtype=bool)
    keep[idx[1:]] = False
    pb.obs_shot, pb.obs_point = pb.obs_shot[keep], pb.obs_point[keep]
    pb.obs_xy, pb.obs_sigma = pb.obs_xy[keep], pb.obs_sigma[keep]
    return pb


def rig_fixed_instances():
    pb = scenes.rig_with_priors()
    pb.inst_const[:] = 1
    return pb


EXTRA = {"gps_cube_constant_instances": gps_cube_constant_instances, "point_seen_once": point_seen_once,
         "rig_free_rigcam_priors_fixed_instances": rig_fixed_instances}
SCENES = dict(scenes.SCENES, **EXTRA)
NAMES = scenes.CPU_SCENES + list(EXTRA)
FULL_RANK = {"camera_and_position_priors", "fixed_instances", "point_priors_many_obs", "gps_cube_constant_instances",
             "rig_free_rigcam_priors_fixed_instances"}


def dense_covariances(pb):
    """(sigma_min / sigma_max of the scaled J, expected status, C[NI, 6, 6]) from the dense numpy J."""
    _, _, J, _, _, _, scale, _ = reference_system(pb)
    nc, n, _, inst_col, _, pt_col = _layout(pb)
    Js = J * scale
    sv = np.linalg.svd(Js, compute_uv=False)
    ratio = sv[-1] / sv[0] if len(sv) == n else 0.0
    C = np.zeros((len(pb.inst), 6, 6))
    if ratio < 1e-12:
        pts = [c for c in pt_col if c >= 0]
        point_bad = any(np.linalg.svd(Js[:, c:c + 3], compute_uv=False)[-1] <= 1e-12 * np.linalg.norm(Js[:, c:c + 3])
                        for c in pts)
        return ratio, "point_rank_deficient" if point_bad else "camera_rank_deficient", np.tile(co.DEFAULT, (len(pb.inst), 1, 1))
    Ci = np.linalg.inv(Js.T @ Js)
    for i, c in enumerate(inst_col):
        if c >= 0:
            C[i] = Ci[c:c + 6, c:c + 6] * scale[c:c + 6, None] * scale[None, c:c + 6]
    return ratio, "ok", C


def test_full_rank_scenes_are_covered():
    assert FULL_RANK <= set(NAMES)


@pytest.mark.parametrize("at", ["start", "solution"])
@pytest.mark.parametrize("name", NAMES)
def test_covariances_match_dense_inverse(name, at):
    pb = SCENES[name]()
    if at == "solution":
        r = oracle.solve(pb)
        pb = co.with_params(pb, r["cam_params"], r["inst"], r["rigcam"], r["points"], r["ext_values"])
    ratio, status_ref, C_ref = dense_covariances(pb)
    print("%s at %s: sigma_min / sigma_max of the scaled J %.2e, %s" % (name, at, ratio, status_ref))
    assert ratio < 1e-12 or ratio > 1e-5, "rank verdict on a knife edge"
    if name in FULL_RANK:
        assert status_ref == "ok"
    if name == "point_seen_once":
        assert status_ref == "point_rank_deficient"
    valid, status, C, _ = co.covariances(pb)
    assert status == status_ref
    assert valid == (status_ref == "ok")
    if not valid:
        assert np.array_equal(C, np.tile(co.DEFAULT, (len(pb.inst), 1, 1)))
        return
    for i in np.flatnonzero(pb.inst_const):
        assert np.all(C[i] == 0.0)
    d = np.sqrt(np.abs(np.einsum("ijj->ij", C_ref)))
    den = d[:, :, None] * d[:, None, :]
    free = pb.inst_const == 0
    worst = (np.abs(C - C_ref)[free] / den[free]).max() if free.any() else 0.0
    print("  worst |C - C_ref| / sqrt(C_ii C_jj) %.2e" % worst)
    assert worst <= 1e-10


def test_failure_gives_default_matrices():
    pb = scenes.camera_and_position_priors()
    valid, status, C, _ = co.covariances(pb, termination="FAILURE")
    assert not valid and status == "solver_failure"
    assert np.array_equal(C, np.tile(co.DEFAULT, (len(pb.inst), 1, 1)))


def test_bundle_adjuster_covariance_host_logic():
    from opensfm_b200 import bundle
    from opensfm_b200 import types as T

    ba = bundle.BundleAdjuster()
    ba.set_compute_covariances(True)   # no longer raises
    assert ba.get_covariance_estimation_valid() is False
    ba.add_camera("c", T.Camera("perspective", [1.0, 0.0, 0.0]), T.Camera("perspective", [1.0, 0.0, 0.0]), False)
    ba.add_rig_camera("rc", T.Pose(), T.Pose(), True)
    ba.add_rig_instance("i0", T.Pose(), {"s0": "c"}, {"s0": "rc"}, False)
    with pytest.raises(RuntimeError, match="Rig instance nope doesn't exist."):
        ba.get_rig_instance_covariance("nope")
    with pytest.raises(RuntimeError, match="i0 hasn't any covariance"):
        ba.get_rig_instance_covariance("i0")
