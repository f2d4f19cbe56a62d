"""Host-side SoA description of one bundle-adjustment problem.

This is the bulk ("structure of arrays") form of what the reference builds one
string-keyed call at a time through `bundle::BundleAdjuster::Add*`
(opensfm/src/bundle/src/bundle_adjuster.cc:94-260) and keeps in
`std::map<std::string, ...>` AoS containers (bundle/bundle_adjuster.h:306-313,
bundle/data/*.h).  The CUDA engine uploads these arrays as they are; nothing
here computes.

Parameter conventions follow the reference:
* camera parameters are stored [PROJ | DISTO | AFFINE]
  (opensfm/src/geometry/src/camera.cc:9-178), e.g. perspective = [k1, k2, focal];
* a pose is [rx, ry, rz, tx, ty, tz] = angle-axis of R(camera->world) and the
  camera origin (bundle/data/pose.h:17,34-43);
* a shot references (rig instance, camera, rig camera); the rig camera is used
  only when it is non-trivial (`IsRigCameraUseful`, bundle_adjuster.cc:17-20).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

# geometry::ProjectionType order (opensfm/src/geometry/camera_instances.h:8-20)
PERSPECTIVE, BROWN, FISHEYE, FISHEYE_OPENCV, FISHEYE62, FISHEYE624, SPHERICAL, DUAL, RADIAL, SIMPLE_RADIAL = range(10)

PROJECTION_NAMES = {
    "perspective": PERSPECTIVE, "brown": BROWN, "fisheye": FISHEYE, "fisheye_opencv": FISHEYE_OPENCV,
    "fisheye62": FISHEYE62, "fisheye624": FISHEYE624, "spherical": SPHERICAL, "equirectangular": SPHERICAL,
    "dual": DUAL, "radial": RADIAL, "simple_radial": SIMPLE_RADIAL,
}

# Parameter names per model in storage order (geometry/src/camera.cc:9-178).
CAMERA_PARAM_NAMES = {
    PERSPECTIVE: ["k1", "k2", "focal"],
    BROWN: ["k1", "k2", "k3", "p1", "p2", "focal", "aspect_ratio", "cx", "cy"],
    FISHEYE: ["k1", "k2", "focal"],
    FISHEYE_OPENCV: ["k1", "k2", "k3", "k4", "focal", "aspect_ratio", "cx", "cy"],
    FISHEYE62: ["k1", "k2", "k3", "k4", "k5", "k6", "p1", "p2", "focal", "aspect_ratio", "cx", "cy"],
    FISHEYE624: ["k1", "k2", "k3", "k4", "k5", "k6", "p1", "p2", "s0", "s1", "s2", "s3",
                 "focal", "aspect_ratio", "cx", "cy"],
    SPHERICAL: ["none"],
    DUAL: ["transition", "k1", "k2", "focal"],
    RADIAL: ["k1", "k2", "focal", "aspect_ratio", "cx", "cy"],
    SIMPLE_RADIAL: ["k1", "focal", "aspect_ratio", "cx", "cy"],
}

LOSS_NAMES = ("TrivialLoss", "HuberLoss", "SoftLOneLoss", "CauchyLoss", "ArctanLoss")
LOSS_IDS = {n: i for i, n in enumerate(LOSS_NAMES)}
LOSS_NONE, LOSS_CAUCHY, LOSS_TUKEY = -1, 3, 5

# block kinds of a side term / ids of the side-term types (include/opensfm_b200.h)
SB_CAM, SB_INST, SB_RIGCAM, SB_EXT = 0, 1, 2, 3
(SIDE_UP_VECTOR, SIDE_PAN, SIDE_TILT, SIDE_ROLL, SIDE_RELATIVE_MOTION, SIDE_RELATIVE_ROTATION, SIDE_COMMON_POSITION,
 SIDE_LINEAR_MOTION, SIDE_TRANSLATION_PRIOR, SIDE_PARAMETER_BARRIER, SIDE_STD_DEVIATION, SIDE_POSITION_PRIOR,
 SIDE_RA_RELATIVE_MOTION, SIDE_RA_ABSOLUTE_POSITION, SIDE_RA_RELATIVE_ABSOLUTE_POSITION, SIDE_RA_COMMON_POINT,
 SIDE_RA_COMMON_CAMERA) = range(17)
LOSS_SOFTLONE = 2


@dataclass
class SideTerm:
    """One secondary residual block: its type, the parameter blocks it reads ((kind, index) pairs, at most 6),
    its constants and its ceres loss (LOSS_NONE = nullptr in the reference).  The constructors below restate the
    reference functors' constructors (argument checks and pre-computed constants included)."""
    type: int
    nres: int
    blocks: List[Tuple[int, int]]
    consts: np.ndarray
    loss: int = LOSS_NONE
    loss_a: float = 1.0
    aux: Tuple[int, ...] = ()


def up_vector_term(inst: int, rigcam: int, up_vector, std_deviation: float) -> SideTerm:
    """UpVectorError (absolute_motion_errors.h:12-39) under CauchyLoss(1) (bundle_adjuster.cc:956-971)."""
    a = np.asarray(up_vector, dtype=np.float64)
    n = float(np.linalg.norm(a))
    if n < 1e-10:
        raise RuntimeError("UpVectorError: acceleration vector has near-zero magnitude")
    return SideTerm(SIDE_UP_VECTOR, 3, [(SB_INST, inst), (SB_RIGCAM, rigcam)],
                    np.concatenate([a / n, [1.0 / std_deviation]]), LOSS_CAUCHY, 1.0)


def angle_term(which: int, inst: int, rigcam: int, angle: float, std_deviation: float) -> SideTerm:
    """Pan / Tilt / RollAngleError (absolute_motion_errors.h:41-136) under CauchyLoss(1) (:973-1022)."""
    assert which in (SIDE_PAN, SIDE_TILT, SIDE_ROLL)
    return SideTerm(which, 1, [(SB_INST, inst), (SB_RIGCAM, rigcam)], np.array([angle, 1.0 / std_deviation]),
                    LOSS_CAUCHY, 1.0)


def relative_motion_term(inst_i: int, inst_j: int, scale_i_ext: int, scale_j_ext: int, rts7, scale_matrix7x7,
                         observed_scale: bool, loss: int, loss_a: float) -> SideTerm:
    """RelativeMotionError (relative_motion_errors.h:14-72; blocks bundle_adjuster.cc:817-856)."""
    blocks = [(SB_INST, inst_i), (SB_INST, inst_j), (SB_EXT, scale_i_ext)]
    sj = 2
    if scale_j_ext != scale_i_ext:
        blocks.append((SB_EXT, scale_j_ext))
        sj = 3
    c = np.concatenate([np.asarray(rts7, dtype=np.float64).reshape(7),
                        np.asarray(scale_matrix7x7, dtype=np.float64).reshape(49), [1.0 if observed_scale else 0.0]])
    return SideTerm(SIDE_RELATIVE_MOTION, 7, blocks, c, loss, loss_a, (sj,))


def _with_rigcams(insts: Sequence[int], rigcams: Sequence[Optional[int]]):
    """Block list [instances..., distinct useful rig cameras...] and, per shot, the block of its rig camera or -1
    (the de-duplication of bundle_adjuster.cc:880-898 / 1048-1081: a rig camera shared by two shots is one block)."""
    blocks = [(SB_INST, i) for i in insts]
    where = {}
    aux = []
    for rc in rigcams:
        if rc is None:
            aux.append(-1)
            continue
        if rc not in where:
            where[rc] = len(blocks)
            blocks.append((SB_RIGCAM, rc))
        aux.append(where[rc])
    return blocks, tuple(aux)


def relative_rotation_term(inst_i, inst_j, rigcam_i, rigcam_j, rij3, scale_matrix3x3, loss, loss_a) -> SideTerm:
    """RelativeRotationError (relative_motion_errors.h:74-103); rigcam_* = None when not 'useful'."""
    blocks, aux = _with_rigcams([inst_i, inst_j], [rigcam_i, rigcam_j])
    c = np.concatenate([np.asarray(rij3, dtype=np.float64).reshape(3), np.asarray(scale_matrix3x3, dtype=np.float64).reshape(9)])
    return SideTerm(SIDE_RELATIVE_ROTATION, 3, blocks, c, loss, loss_a, aux)


def common_position_term(inst_i, inst_j, rigcam_i, rigcam_j, margin: float, std_deviation: float) -> SideTerm:
    """CommonPositionError under TukeyLoss(1) (relative_motion_errors.h:105-138, bundle_adjuster.cc:902-944)."""
    blocks, aux = _with_rigcams([inst_i, inst_j], [rigcam_i, rigcam_j])
    return SideTerm(SIDE_COMMON_POSITION, 3, blocks, np.array([margin, 1.0 / std_deviation]), LOSS_TUKEY, 1.0, aux)


def linear_motion_term(insts3, rigcams3, alpha: float, position_std: float, orientation_std: float) -> SideTerm:
    """LinearMotionError under CauchyLoss(1) (motion_prior_errors.h:13-76, bundle_adjuster.cc:1024-1084)."""
    blocks, aux = _with_rigcams(list(insts3), list(rigcams3))
    return SideTerm(SIDE_LINEAR_MOTION, 6, blocks, np.array([alpha, 1.0 / position_std, 1.0 / orientation_std]),
                    LOSS_CAUCHY, 1.0, aux)


def translation_prior_term(inst1: int, inst2: int, prior_norm: float) -> SideTerm:
    """TranslationPriorError: the gauge-fix scale constraint (absolute_motion_errors.h:180-202)."""
    return SideTerm(SIDE_TRANSLATION_PRIOR, 1, [(SB_INST, inst1), (SB_INST, inst2)], np.array([max(prior_norm, 1e-20)]))


def parameter_barrier_term(cam: int, index: int, lower: float = 0.0, upper: float = 1.0) -> SideTerm:
    """ParameterBarrier on the DUAL transition (parameters_errors.h:20-36, bundle_adjuster.cc:610-625)."""
    return SideTerm(SIDE_PARAMETER_BARRIER, 1, [(SB_CAM, cam)], np.array([lower, upper]), aux=(index,))


def std_deviation_term(ext: int) -> SideTerm:
    """StdDeviationConstraint (parameters_errors.h:7-18, bundle_adjuster.cc:727-736)."""
    return SideTerm(SIDE_STD_DEVIATION, 1, [(SB_EXT, ext)], np.zeros(0))


def position_prior_term(inst: int, bias_ext: int, std_ext: int, position, std_deviation, adjust_scales: bool) -> SideTerm:
    """DataPriorError<Pose, SimilarityPriorTransform> on TX, TY, TZ (bundle_adjuster.cc:745-778)."""
    sig = np.maximum(np.asarray(std_deviation, dtype=np.float64).reshape(3), np.finfo(np.float64).eps)
    c = np.concatenate([np.asarray(position, dtype=np.float64).reshape(3), 1.0 / sig, [1.0 if adjust_scales else 0.0]])
    return SideTerm(SIDE_POSITION_PRIOR, 3, [(SB_INST, inst), (SB_EXT, bias_ext), (SB_EXT, std_ext)], c)


def camera_num_params(ptype: int) -> int:
    return len(CAMERA_PARAM_NAMES[int(ptype)])


def default_prior_sigma(ptype: int, focal_sd=1.0, aspect_ratio_sd=1.0, c_sd=1.0, k1_sd=1.0, k2_sd=1.0,
                        p1_sd=1.0, p2_sd=1.0, k3_sd=1.0, k4_sd=1.0) -> np.ndarray:
    """BundleAdjuster::GetDefaultCameraSigma (bundle_adjuster.cc:46-67): one sigma per stored
    parameter.  The reference's map holds focal, aspect ratio, cx, cy, k1, k2, k3, p1, p2 and
    transition (=1); every other parameter (k4, k5, k6, s0..s3, none) reads a default-inserted
    0.0 from `std_dev_map[...]` (:64), i.e. scale 1/eps in DataPriorError (prior_error.h:31-35):
    those parameters are pinned to their prior.  k4_sd is accepted and unused, as in the reference."""
    del k4_sd
    table = {"focal": focal_sd, "aspect_ratio": aspect_ratio_sd, "cx": c_sd, "cy": c_sd, "k1": k1_sd,
             "k2": k2_sd, "k3": k3_sd, "p1": p1_sd, "p2": p2_sd, "transition": 1.0}
    return np.array([table.get(n, 0.0) for n in CAMERA_PARAM_NAMES[int(ptype)]], dtype=np.float64)


def prior_log_mask(ptype: int) -> np.ndarray:
    """Focal and aspect ratio use a logarithmic prior (bundle_adjuster.cc:574-583)."""
    return np.array([1 if n in ("focal", "aspect_ratio") else 0 for n in CAMERA_PARAM_NAMES[int(ptype)]],
                    dtype=np.int32)


@dataclass
class BAProblem:
    # cameras (K); parameters flattened, camera k owns cam_params[cam_off[k]:cam_off[k+1]]
    cam_type: np.ndarray
    cam_params: np.ndarray
    cam_const: np.ndarray
    cam_prior: np.ndarray
    cam_prior_sigma: np.ndarray
    cam_prior_log: np.ndarray
    # rig instances (NI x 6)
    inst: np.ndarray
    inst_const: np.ndarray
    inst_has_prior: np.ndarray
    inst_prior_pos: np.ndarray
    inst_prior_std: np.ndarray
    # rig cameras (NR x 6)
    rigcam: np.ndarray
    rigcam_const: np.ndarray
    # shots (S)
    shot_inst: np.ndarray
    shot_cam: np.ndarray
    shot_rc: np.ndarray
    shot_use_rc: np.ndarray
    # points (P x 3)
    points: np.ndarray
    point_const: np.ndarray
    # observations (N)
    obs_shot: np.ndarray
    obs_point: np.ndarray
    obs_xy: np.ndarray
    obs_sigma: np.ndarray
    # solver options (defaults of bundle::BundleAdjuster(), bundle_adjuster.cc:24-44)
    loss_name: str = "CauchyLoss"
    loss_threshold: float = 1.0
    max_iterations: int = 500
    linear_solver_type: str = "SPARSE_SCHUR"
    num_threads: int = 1
    # --- secondary residuals (SURVEY.md §8a); all optional -------------------------------------
    # rig-camera pose priors DataPriorError<Pose> (bundle_adjuster.cc:779-790): NR x 6 each, or None
    rigcam_prior: Optional[np.ndarray] = None
    rigcam_prior_sigma: Optional[np.ndarray] = None
    # point priors (AddPointPrior): point index, prior xyz, sigma xyz, has_altitude
    pp_point: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int32))
    pp_prior: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))
    pp_sigma: np.ndarray = field(default_factory=lambda: np.ones((0, 3)))
    pp_alt: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int32))
    # ext blocks: camera biases (7), reconstruction scales (1), std-deviation scales (1)
    ext_size: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int32))
    ext_values: np.ndarray = field(default_factory=lambda: np.zeros(0))
    ext_const: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int32))
    ext_lower: np.ndarray = field(default_factory=lambda: np.zeros(0))
    side_terms: List[SideTerm] = field(default_factory=list)

    def add_ext_block(self, values, constant: bool, lower: Optional[Sequence[float]] = None) -> int:
        v = np.atleast_1d(np.asarray(values, dtype=np.float64))
        lo = np.full(len(v), -np.inf) if lower is None else np.atleast_1d(np.asarray(lower, dtype=np.float64))
        self.ext_size = np.append(self.ext_size, len(v)).astype(np.int32)
        self.ext_values = np.concatenate([self.ext_values, v])
        self.ext_const = np.append(self.ext_const, int(constant)).astype(np.int32)
        self.ext_lower = np.concatenate([self.ext_lower, lo])
        return len(self.ext_size) - 1

    @property
    def ext_off(self) -> np.ndarray:
        return np.concatenate([[0], np.cumsum(self.ext_size)]).astype(np.int32)

    def packed_side_terms(self):
        """(records, constants): per term (type, nres, nblocks, kind[6], idx[6], loss, loss_a, cofs, aux[4])."""
        recs, consts, cofs = [], [], 0
        for t in self.side_terms:
            if len(t.blocks) > 6 or len(t.aux) > 4:
                raise ValueError("side term with too many blocks")
            kind = [b[0] for b in t.blocks] + [0] * (6 - len(t.blocks))
            idx = [b[1] for b in t.blocks] + [0] * (6 - len(t.blocks))
            aux = list(t.aux) + [-1] * (4 - len(t.aux))
            recs.append((int(t.type), int(t.nres), len(t.blocks), kind, idx, int(t.loss), float(t.loss_a), cofs, aux))
            c = np.asarray(t.consts, dtype=np.float64).ravel()
            consts.append(c)
            cofs += len(c)
        return recs, (np.concatenate(consts) if consts else np.zeros(0))

    def block_size(self, kind: int, idx: int) -> int:
        if kind == SB_CAM:
            return camera_num_params(self.cam_type[idx])
        return int(self.ext_size[idx]) if kind == SB_EXT else 6

    def side_row_sizes(self) -> Tuple[np.ndarray, np.ndarray]:
        """Per side term: its residual count and the size nres x np of its Jacobian block (np = the sizes of the blocks
        it lists, in that order), the layout of the captured side rows."""
        nres = np.array([t.nres for t in self.side_terms], dtype=np.int64)
        npar = np.array([sum(self.block_size(k, i) for k, i in t.blocks) for t in self.side_terms], dtype=np.int64)
        return nres, nres * npar

    @property
    def cam_off(self) -> np.ndarray:
        sizes = np.array([camera_num_params(t) for t in self.cam_type], dtype=np.int32)
        return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)

    @property
    def num_observations(self) -> int:
        return int(self.obs_shot.shape[0])

    def copy(self) -> "BAProblem":
        kw = {}
        for k, v in self.__dict__.items():
            kw[k] = v.copy() if isinstance(v, np.ndarray) else (list(v) if isinstance(v, list) else v)
        return BAProblem(**kw)

    def validate(self, check_indices: bool = True) -> None:
        """Shape / range checks.  bundle.solve passes check_indices=False: the observation indices are range-checked
        on the device while the sort keys are built (ba_order.cuh, "observation references a shot / point that does
        not exist"), and four numpy passes over 2M entries cost more than the whole device-side ordering."""
        K = len(self.cam_type)
        ncp = int(self.cam_off[-1])
        assert self.cam_params.shape == (ncp,)
        assert self.cam_prior.shape == (ncp,) and self.cam_prior_sigma.shape == (ncp,)
        assert self.cam_prior_log.shape == (ncp,)
        assert len(self.cam_const) == K
        NI, NR, S, P, N = len(self.inst), len(self.rigcam), len(self.shot_inst), len(self.points), len(self.obs_shot)
        assert self.inst.shape == (NI, 6) and self.rigcam.shape == (NR, 6) and self.points.shape == (P, 3)
        assert self.obs_xy.shape == (N, 2) and self.obs_sigma.shape == (N,)
        if N and check_indices:
            assert self.obs_shot.min() >= 0 and self.obs_shot.max() < S
            assert self.obs_point.min() >= 0 and self.obs_point.max() < P
        if S:
            assert self.shot_inst.max() < NI and self.shot_cam.max() < K and self.shot_rc.max() < max(NR, 1)
        if self.loss_name not in LOSS_NAMES:
            # bundle_adjuster.cc:427
            raise RuntimeError("ceres::LossFunction with name %s not found." % self.loss_name)


def make_problem(cam_type, cam_params_list, inst, points, obs_shot, obs_point, obs_xy, obs_sigma,
                 shot_inst=None, shot_cam=None, rigcam=None, shot_rc=None, shot_use_rc=None,
                 cam_const=None, inst_const=None, rigcam_const=None, point_const=None,
                 cam_prior_list=None, prior_sd=None, inst_prior_pos=None, inst_prior_std=None,
                 **options) -> BAProblem:
    """Convenience builder: one camera/instance per shot unless told otherwise."""
    cam_type = np.asarray(cam_type, dtype=np.int32)
    K = len(cam_type)
    inst = np.ascontiguousarray(inst, dtype=np.float64).reshape(-1, 6)
    NI = len(inst)
    if shot_inst is None:
        shot_inst = np.arange(NI, dtype=np.int32)
    S = len(shot_inst)
    if shot_cam is None:
        shot_cam = np.arange(S, dtype=np.int32) if K == S else np.zeros(S, dtype=np.int32)
    if rigcam is None:
        rigcam = np.zeros((1, 6))
    rigcam = np.ascontiguousarray(rigcam, dtype=np.float64).reshape(-1, 6)
    NR = len(rigcam)
    if shot_rc is None:
        shot_rc = np.zeros(S, dtype=np.int32)
    if shot_use_rc is None:
        shot_use_rc = np.zeros(S, dtype=np.int32)
    cam_params = np.concatenate([np.asarray(p, dtype=np.float64) for p in cam_params_list])
    cam_prior = cam_params.copy() if cam_prior_list is None else np.concatenate(
        [np.asarray(p, dtype=np.float64) for p in cam_prior_list])
    sd = prior_sd or {}
    cam_prior_sigma = np.concatenate([default_prior_sigma(t, **sd) for t in cam_type])
    cam_prior_log = np.concatenate([prior_log_mask(t) for t in cam_type])
    points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
    P = len(points)
    has_prior = np.zeros(NI, dtype=np.int32)
    if inst_prior_pos is None:
        inst_prior_pos = np.zeros((NI, 3))
        inst_prior_std = np.ones((NI, 3))
    else:
        has_prior[:] = 1
    z = lambda n, a: np.zeros(n, dtype=np.int32) if a is None else np.asarray(a, dtype=np.int32)
    pb = BAProblem(
        cam_type=cam_type, cam_params=cam_params, cam_const=z(K, cam_const), cam_prior=cam_prior,
        cam_prior_sigma=cam_prior_sigma, cam_prior_log=cam_prior_log,
        inst=inst, inst_const=z(NI, inst_const), inst_has_prior=has_prior,
        inst_prior_pos=np.ascontiguousarray(inst_prior_pos, dtype=np.float64),
        inst_prior_std=np.ascontiguousarray(inst_prior_std, dtype=np.float64),
        rigcam=rigcam, rigcam_const=np.ones(NR, dtype=np.int32) if rigcam_const is None else np.asarray(rigcam_const, dtype=np.int32),
        shot_inst=np.asarray(shot_inst, dtype=np.int32), shot_cam=np.asarray(shot_cam, dtype=np.int32),
        shot_rc=np.asarray(shot_rc, dtype=np.int32), shot_use_rc=np.asarray(shot_use_rc, dtype=np.int32),
        points=points, point_const=z(P, point_const),
        obs_shot=np.asarray(obs_shot, dtype=np.int32), obs_point=np.asarray(obs_point, dtype=np.int32),
        obs_xy=np.ascontiguousarray(obs_xy, dtype=np.float64).reshape(-1, 2),
        obs_sigma=np.ascontiguousarray(obs_sigma, dtype=np.float64),
        **options)
    pb.validate()
    return pb
