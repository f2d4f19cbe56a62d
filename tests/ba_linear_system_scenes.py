"""Small seeded bundle-adjustment scenes for the reduced-camera-system tests, each built to reach one kernel path
of the engine's Schur complement / PCG (tests/test_ba_linear_system_gpu.py) and, where it has no side terms, the
numpy restatement of the oracle's Schur complement (tests/test_reduced_system_reference.py).

Not a test module: the test files import it (pytest puts tests/ on sys.path)."""
from __future__ import annotations

import numpy as np

from opensfm_b200 import ba_problem as bp
from opensfm_b200 import synthetic as syn

PRIOR_SD = dict(focal_sd=0.01, aspect_ratio_sd=0.01, c_sd=0.01, k1_sd=0.01, k2_sd=0.01, p1_sd=0.01, p2_sd=0.01,
                k3_sd=0.01, k4_sd=0.01)

RING_PARAMS = {
    bp.PERSPECTIVE: [-0.05, 0.01, 0.8], bp.BROWN: [-0.05, 0.01, 0.001, 0.001, -0.001, 0.8, 1.0, 0.01, -0.01],
    bp.FISHEYE: [-0.02, 0.005, 0.7], bp.FISHEYE_OPENCV: [-0.02, 0.005, 0.001, 0.0, 0.7, 1.0, 0.0, 0.01],
    bp.RADIAL: [-0.05, 0.01, 0.8, 1.0, 0.0, 0.0], bp.SPHERICAL: [0.0], bp.DUAL: [0.4, -0.03, 0.005, 0.75],
    bp.SIMPLE_RADIAL: [-0.04, 0.8, 1.0, 0.0, 0.0],
    bp.FISHEYE62: [-0.02, 0.005, 0.0, 0.0, 0.0, 0.0, 0.001, -0.001, 0.7, 1.0, 0.0, 0.0],
    bp.FISHEYE624: [-0.02, 0.005, 0.0, 0.0, 0.0, 0.0, 0.001, -0.001, 0.001, 0.0, -0.001, 0.0, 0.7, 1.0, 0.0, 0.0],
}
ALL_TYPES = [bp.PERSPECTIVE, bp.BROWN, bp.FISHEYE, bp.FISHEYE_OPENCV, bp.RADIAL, bp.SPHERICAL, bp.DUAL,
             bp.SIMPLE_RADIAL, bp.FISHEYE62, bp.FISHEYE624]


def ring_problem(types, n_points=300, seed=0, rig=False, free_rig=False, keep=1.0, loss="SoftLOneLoss"):
    """len(types) rig instances on a ring around a point cloud, one camera each (the types given); with `rig`, a
    second shot per instance through a free (or constant) rig camera.  `keep` < 1 drops observations at random so
    that points see different numbers of shots."""
    from scipy.spatial.transform import Rotation

    rng = np.random.RandomState(seed)
    K = NI = len(types)
    pts = rng.uniform(-0.5, 0.5, (n_points, 3))
    inst = np.zeros((NI, 6))
    for i in range(NI):
        ang = 2 * np.pi * i / NI
        origin = 2.5 * np.array([np.cos(ang), np.sin(ang), 0.2 * np.sin(3 * ang)])
        ez = -origin / np.linalg.norm(origin)
        ex = np.cross(ez, [0, 0, 1.0]); ex /= np.linalg.norm(ex)
        ey = np.cross(ez, ex)
        inst[i] = np.concatenate([Rotation.from_matrix(np.array([ex, ey, ez]).T).as_rotvec(), origin])
    if rig:
        rigcam = np.array([[0.0] * 6, [0.02, -0.03, 0.01, 0.1, 0.0, 0.02]])
        shot_inst, shot_cam = np.repeat(np.arange(NI), 2), np.repeat(np.arange(K), 2)
        shot_rc, shot_use = np.tile([0, 1], NI), np.tile([0, 1], NI)
    else:
        rigcam = np.zeros((1, 6))
        shot_inst, shot_cam = np.arange(NI), np.arange(K)
        shot_rc, shot_use = np.zeros(NI, int), np.zeros(NI, int)
    obs_shot, obs_point, obs_xy = [], [], []
    for s in range(len(shot_inst)):
        i, t = shot_inst[s], types[shot_cam[s]]
        R = Rotation.from_rotvec(-inst[i, :3])
        for p in range(n_points):
            xc = R.apply(pts[p] - inst[i, 3:])
            if shot_use[s]:
                rc = rigcam[shot_rc[s]]
                xc = Rotation.from_rotvec(-rc[:3]).apply(xc - rc[3:])
            if (t != bp.SPHERICAL and xc[2] < 0.5) or rng.uniform() > keep:
                continue
            if t == bp.SPHERICAL:
                lon, lat = np.arctan2(xc[0], xc[2]), np.arctan2(-xc[1], np.hypot(xc[0], xc[2]))
                px = np.array([lon / (2 * np.pi), -lat / (2 * np.pi)])
            else:
                from oracle import ba_lm

                px = ba_lm.project(t, RING_PARAMS[t], xc)
            obs_shot.append(s); obs_point.append(p); obs_xy.append(px + rng.normal(0, 5e-4, 2))
    pb = bp.make_problem(types, [RING_PARAMS[t] for t in types], inst, pts + rng.normal(0, 0.01, pts.shape), obs_shot,
                         obs_point, np.array(obs_xy), np.full(len(obs_shot), 0.004), shot_inst=shot_inst,
                         shot_cam=shot_cam, rigcam=rigcam, shot_rc=shot_rc, shot_use_rc=shot_use,
                         rigcam_const=[1, 0 if free_rig else 1] if rig else None, prior_sd=PRIOR_SD,
                         loss_name=loss, loss_threshold=1.0, max_iterations=50)
    pb.inst[:, 3:] += rng.normal(0, 0.01, (NI, 3))
    return pb


def cube(num_cameras, num_points, max_obs=None, seed=42, **kw):
    sc = syn.cube_scene(num_cameras, num_points, 1.0, seed=seed, with_descriptors=False, max_obs_per_point=max_obs)
    return syn.scene_to_problem(sc, **kw)


def constant_blocks():
    pb = cube(12, 600, max_obs=6)
    pb.cam_const[::3] = 1         # every third camera constant
    pb.inst_const[1::4] = 1       # some instances constant
    pb.point_const[::5] = 1       # every fifth point constant: segments of constant points carry U only
    return pb


def camera_and_position_priors():
    pb = cube(10, 500, max_obs=6)
    rng = np.random.RandomState(5)
    # priors away from the start, so that the prior rows have non-zero residuals (log rows on the focal)
    pb.cam_prior = pb.cam_prior * (1.0 + 0.02 * rng.standard_normal(pb.cam_prior.shape))
    pb.inst_has_prior[:] = 1
    pb.inst_prior_pos = pb.inst[:, 3:] + rng.normal(0, 0.02, (len(pb.inst), 3))
    pb.inst_prior_std = np.full((len(pb.inst), 3), 0.05)
    return pb


def point_priors_many_obs():
    """20 perspective cameras seeing (almost) every point: more than 16 observations per point (two staging chunks of
    the per-point ba_schur), GCP priors with and without altitude on every seventh point."""
    pb = ring_problem([bp.PERSPECTIVE] * 20, n_points=200, seed=4)
    q = np.arange(0, len(pb.points), 7)
    rng = np.random.RandomState(6)
    pb.pp_point = q.astype(np.int32)
    pb.pp_prior = pb.points[q] + rng.normal(0, 0.02, (len(q), 3))
    pb.pp_sigma = np.full((len(q), 3), 0.05)
    pb.pp_alt = (np.arange(len(q)) % 2).astype(np.int32)
    return pb


def rig_with_priors():
    pb = ring_problem([bp.PERSPECTIVE, bp.FISHEYE, bp.PERSPECTIVE, bp.BROWN, bp.PERSPECTIVE, bp.FISHEYE], seed=2,
                      rig=True, free_rig=True)
    pb.rigcam_prior = pb.rigcam + np.array([0.01, -0.01, 0.005, 0.02, 0.01, -0.01])
    pb.rigcam_prior_sigma = np.full((len(pb.rigcam), 6), 0.05)
    return pb


def robust(loss):
    pb = cube(10, 500, max_obs=6, loss_name=loss)
    rng = np.random.RandomState(8)
    bad = rng.uniform(size=len(pb.obs_xy)) < 0.1   # about 10 % gross outliers, far beyond the loss threshold
    pb.obs_xy = pb.obs_xy.copy()
    pb.obs_xy[bad] += rng.normal(0, 0.05, (int(bad.sum()), 2))
    return pb


def duplicate_observations():
    """Some points observed twice by the same shot (different measurements): Ceres adds both residuals."""
    pb = cube(8, 400, max_obs=5)
    rng = np.random.RandomState(9)
    dup = rng.choice(len(pb.obs_shot), 40, replace=False)
    pb.obs_shot = np.concatenate([pb.obs_shot, pb.obs_shot[dup]]).astype(np.int32)
    pb.obs_point = np.concatenate([pb.obs_point, pb.obs_point[dup]]).astype(np.int32)
    pb.obs_xy = np.concatenate([pb.obs_xy, pb.obs_xy[dup] + rng.normal(0, 5e-4, (40, 2))])
    pb.obs_sigma = np.concatenate([pb.obs_sigma, pb.obs_sigma[dup]])
    return pb


def rig_segments():
    """Perspective / fisheye rig (wc = 3 + 6 + 6 = 15): observations with three parameter blocks in the SIMT segment
    kernels; thinned so that points see between 0 and 12 shots (two free points end up with no observation at all:
    empty columns, damped only)."""
    pb = ring_problem([bp.PERSPECTIVE, bp.FISHEYE] * 3, n_points=300, seed=7, rig=True, free_rig=True, keep=0.35)
    pb.rigcam_prior = pb.rigcam + np.array([0.01, -0.01, 0.005, 0.02, 0.01, -0.01])
    pb.rigcam_prior_sigma = np.full((len(pb.rigcam), 6), 0.05)
    return pb


def instances_sharing_no_point(pb):
    """Pairs (i, j), i < j, of rig instances whose shots observe no common point."""
    NI = len(pb.inst)
    seen = np.zeros((NI, len(pb.points)), dtype=bool)
    seen[pb.shot_inst[pb.obs_shot], pb.obs_point] = True
    common = seen.astype(np.int64) @ seen.T.astype(np.int64)
    return [(i, j) for i in range(NI) for j in range(i + 1, NI) if common[i, j] == 0]


def side_terms():
    """Side terms through BundleAdjuster (side_enum_pairs structure discovery, side_system): relative motions with
    per-instance reconstruction scales (1-parameter ext blocks bounded below by 0, so the problem is constrained), one of
    them between two instances that share no point, common position, up vector and linear motion."""
    from opensfm_b200 import bundle
    from opensfm_b200 import types as T

    pb0 = cube(8, 400, max_obs=4)
    # shot 4 loses its observations of the points shot 0 sees (those points keep shot 0): instances 0 and 4 share none
    drop = (pb0.obs_shot == 4) & np.isin(pb0.obs_point, pb0.obs_point[pb0.obs_shot == 0])
    pb0.obs_shot, pb0.obs_point = pb0.obs_shot[~drop], pb0.obs_point[~drop]
    pb0.obs_xy, pb0.obs_sigma = pb0.obs_xy[~drop], pb0.obs_sigma[~drop]
    ba = bundle.BundleAdjuster()
    off = pb0.cam_off
    for k in range(len(pb0.cam_type)):
        vals = pb0.cam_params[off[k]:off[k + 1]]
        ba.add_camera("c%d" % k, T.Camera("perspective", vals), T.Camera("perspective", vals), False)
    ba.add_rig_camera("rc", T.Pose(), T.Pose(), True)
    NI = len(pb0.inst)
    poses = [T.Pose.from_ba_params(pb0.inst[i]) for i in range(NI)]
    for i in range(NI):
        ba.add_rig_instance("i%d" % i, poses[i], {"s%d" % i: "c%d" % i}, {"s%d" % i: "rc"}, False)
    ba.add_points_bulk(["p%d" % p for p in range(len(pb0.points))], pb0.points, False)
    ba.add_observations_bulk(["s%d" % s for s in pb0.obs_shot], ["p%d" % p for p in pb0.obs_point], pb0.obs_xy,
                             pb0.obs_sigma)
    ba.set_point_projection_loss_function("SoftLOneLoss", 1.0)
    ba.set_internal_parameters_prior_sd(0.01, 0.01, 0.01, 0.01, 0.01, 0.01, 0.01, 0.01, 0.01)
    ba.add_reconstruction("r", False)
    for i in range(NI):
        ba.add_reconstruction_instance("r", 1.0 + 0.05 * i, "i%d" % i)
    ba.set_scale_sharing("r", False)

    def relative(i, j):
        Ri, Rj = poses[i].get_rotation_matrix(), poses[j].get_rotation_matrix()
        from scipy.spatial.transform import Rotation

        Rij = Rj @ Ri.T
        tij = poses[j].translation - Rij @ poses[i].translation
        return bundle.RelativeMotion("i%d" % i, "i%d" % j, Rotation.from_matrix(Rij).as_rotvec(), tij, 1.0, 1.0, True)

    pairs = [(i, i + 1) for i in range(NI - 1)]
    apart = instances_sharing_no_point(pb0)
    assert apart, "the scene needs two instances that share no point"
    a, b = apart[0]
    pairs.append((a, b))
    for i, j in pairs:
        ba.add_relative_motion(relative(i, j))
    ba.add_common_position("s%d" % a, "s%d" % b, 0.5, 0.2)
    ba.add_absolute_up_vector("s1", [0.0, 0.0, 1.0], 0.5)
    ba.add_linear_motion("s2", "s3", "s4", 0.5, 0.2, 0.2)
    pb = ba.to_problem()
    pb.max_iterations = 50
    return pb


def fixed_instances():
    pb = cube(12, 600, max_obs=6)
    pb.inst_const[:] = 1
    return pb


def _keep_observations(pb, keep):
    pb.obs_shot, pb.obs_point = pb.obs_shot[keep], pb.obs_point[keep]
    pb.obs_xy, pb.obs_sigma = pb.obs_xy[keep], pb.obs_sigma[keep]
    return pb


def pipe_long_runs():
    """4 cameras that all see all 400 points; 64 points (at random places of the point list) lose shot 3 and 65 lose
    shot 2: runs of 64, 65 and 271 identical shot lists, cut into 1, 2 and 5 segments of ba_schur_pipe."""
    pb = cube(4, 400)
    rng = np.random.RandomState(11)
    order = rng.permutation(len(pb.points))
    drop = np.full(len(pb.points), -1)
    drop[order[:64]], drop[order[64:129]] = 3, 2
    return _keep_observations(pb, pb.obs_shot != drop[pb.obs_point])


def pipe_k_edge():
    """12 perspective cameras (wc = 9); 150 points keep 10 of their 12 shots (90 camera-side columns: segments of
    ba_schur_pipe) and 150 keep 11 (99 > 96: the per-point ba_schur), on one solve."""
    pb = cube(12, 300)
    rng = np.random.RandomState(12)
    keep = np.zeros(len(pb.obs_shot), dtype=bool)
    for p in range(len(pb.points)):
        mine = np.nonzero(pb.obs_point == p)[0]
        keep[rng.choice(mine, 10 if p % 2 else 11, replace=False)] = True
    return _keep_observations(pb, keep)


def unobserved_and_idle():
    """A cube scene with 20 free points that no shot observes, at random places of the point list, and a shot whose
    rig instance (free, no prior) is used by nothing else and which observes nothing, in the middle of the shot and
    instance lists.  Their parameter blocks appear in no residual (see test_ba_input_order_gpu.py)."""
    pb = cube(10, 500, max_obs=6)
    rng = np.random.RandomState(13)
    P, extra = len(pb.points), 20
    idle = np.sort(rng.choice(P + extra, extra, replace=False))
    observed = np.setdiff1d(np.arange(P + extra), idle)
    pts = np.zeros((P + extra, 3))
    pts[observed] = pb.points
    pts[idle] = rng.uniform(-0.5, 0.5, (extra, 3))
    pb.points, pb.point_const = pts, np.zeros(P + extra, dtype=np.int32)
    pb.obs_point = observed[pb.obs_point].astype(np.int32)
    # the idle instance at index 3, its shot at index 4 (camera 0)
    ins, sh = 3, 4
    pb.inst = np.insert(pb.inst, ins, pb.inst[ins] + rng.normal(0, 0.05, 6), axis=0)
    pb.inst_const = np.insert(pb.inst_const, ins, 0)
    pb.inst_has_prior = np.insert(pb.inst_has_prior, ins, 0)
    pb.inst_prior_pos = np.insert(pb.inst_prior_pos, ins, 0.0, axis=0)
    pb.inst_prior_std = np.insert(pb.inst_prior_std, ins, 1.0, axis=0)
    shot_inst = pb.shot_inst + (pb.shot_inst >= ins)
    pb.shot_inst = np.insert(shot_inst, sh, ins).astype(np.int32)
    pb.shot_cam = np.insert(pb.shot_cam, sh, 0).astype(np.int32)
    pb.shot_rc = np.insert(pb.shot_rc, sh, 0).astype(np.int32)
    pb.shot_use_rc = np.insert(pb.shot_use_rc, sh, 0).astype(np.int32)
    pb.obs_shot = (pb.obs_shot + (pb.obs_shot >= sh)).astype(np.int32)
    pb.validate()
    return pb


# name -> builder; CPU_SCENES are the ones the numpy restatement covers (all but side_terms, which has no simple numpy
# restatement, and the two large cube scenes)
SCENES = {
    "pipe_many_chunks": lambda: cube(30, 4000, max_obs=8),
    "pipe_few_chunks": lambda: cube(6, 150, max_obs=4),
    "c2_size": lambda: cube(50, 20000, max_obs=8),   # C2: 50 cameras, 160k observations, nc = 450
    "shared_intrinsics": lambda: cube(10, 600, max_obs=6, shared_intrinsics=True),
    "constant_blocks": constant_blocks,
    "brown_simt_segments": lambda: ring_problem([bp.BROWN] * 10, n_points=300, seed=3, keep=0.6),
    "rig_free_rigcam_priors": rig_with_priors,
    "rig_segments": rig_segments,
    "side_terms": side_terms,
    "spherical": lambda: ring_problem([bp.SPHERICAL] * 6, n_points=200, seed=5),
    "all_ten_models": lambda: ring_problem(ALL_TYPES, n_points=250, seed=0),
    "point_priors_many_obs": point_priors_many_obs,
    "camera_and_position_priors": camera_and_position_priors,
    "cauchy_outliers": lambda: robust("CauchyLoss"),
    "huber_outliers": lambda: robust("HuberLoss"),
    "duplicate_observations": duplicate_observations,
    "fixed_instances": fixed_instances,
    "pipe_long_runs": pipe_long_runs,
    "pipe_k_edge": pipe_k_edge,
    "unobserved_and_idle": unobserved_and_idle,
}
CPU_SCENES = ["pipe_few_chunks", "shared_intrinsics", "constant_blocks", "brown_simt_segments", "rig_free_rigcam_priors",
              "rig_segments", "spherical", "all_ten_models", "point_priors_many_obs", "camera_and_position_priors", "cauchy_outliers",
              "huber_outliers", "duplicate_observations", "fixed_instances", "pipe_long_runs", "pipe_k_edge",
              "unobserved_and_idle"]
