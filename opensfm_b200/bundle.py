"""Drop-in bundle adjustment: the `opensfm.pybundle.BundleAdjuster` surface and a bulk
SoA entry, both running on the CUDA engine (opensfm_b200/csrc/ba.cu) through the C ABI.

Reference interfaces mirrored here:
* class `pybundle.BundleAdjuster` (opensfm/src/bundle/python/pybind.cc:45-117,
  stub opensfm/src/bundle/pybundle.pyi:34-187): same method names, argument
  meaning, defaults (CauchyLoss(1), 500 iterations, SPARSE_SCHUR,
  bundle_adjuster.cc:24-44) and error behaviour (missing ids ->
  RuntimeError "... doesn't exist.", unknown loss / solver names -> RuntimeError).
* `solve(problem)`: the bulk path that replaces O(N) string-keyed Add* calls
  (SURVEY.md §7 "String-keyed API"), fed by opensfm_b200.ba_problem.BAProblem.

No CPU fallback: every `run()` goes to the GPU library.
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, List, Optional, Sequence

import numpy as np

from . import _lib
from . import ba_problem as bp
from . import types as T
from ._lib import ptr

_TERMINATION = {0: "CONVERGENCE", 1: "NO_CONVERGENCE", 2: "FAILURE"}


def solve(pb: bp.BAProblem, device: int = 0, rank: int = 0, world: int = 1, allreduce=None,
          stream: Optional[int] = None, compute_reprojection_errors: bool = True,
          out: Optional[Dict[str, np.ndarray]] = None, pinned_inputs: bool = False,
          capture_iteration: Optional[int] = None, compute_covariances: bool = False,
          fallbacks: Sequence[str] = ()) -> Dict[str, Any]:
    """Run the GPU bundle adjustment on a BAProblem.  Returns updated parameter arrays,
    unscaled reprojection errors (bundle_adjuster.cc:1196-1208) and the run summary.

    Multi-GPU: pass rank/world and either allreduce="nccl" (the library opens its own NCCL
    communicator; torch.distributed must be initialised, it only carries the 128-byte id once) or a
    callable `allreduce(ptr:int, count:int, stream:int) -> None` that sums `count` float64 at device
    pointer `ptr` across ranks (see opensfm_b200.dist; used with gloo in the CPU tests).

    `out` may hold preallocated C-contiguous float64 arrays "points" (P, 3) and "reprojection_errors"
    (N, 3) to receive the results (page-locked buffers make the device->host copy a plain DMA).
    `pinned_inputs`: the observation arrays of `pb` are page-locked; their upload then overlaps the device-side
    ordering (osfm_ba_set_observations_async; the arrays are kept alive here until the solve returns).
    `capture_iteration` (single GPU, tests): result["capture"] holds the damped reduced system of that LM iteration
    (1-based) as the PCG received it, the PCG solution, the Jacobi scale, the LM diagonal, the gradient and the
    kernel paths that ran (osfm_ba_get_captured_system); raises if the solve ended before that iteration.
    `compute_covariances` (single GPU): the result gains "covariances" (NI x 6 x 6, the rig-instance pose covariances
    in the problem's instance order, zeros for constant instances), "covariance_valid", "covariance_status" (one of
    _lib.COVARIANCE_STATUS) and "covariance_ms", the device times (ms) of the covariance pass and of its Cholesky
    factorisation (osfm_ba_get_covariance_timing).  As in the reference, an invalid estimate leaves every instance with
    the default diag(1e-5, 1e-5, 1e-5, 1e-2, 1e-2, 1e-2).
    `fallbacks` (tests, A/B runs): names from _lib.BA_FALLBACKS of kernel paths this solve takes instead of the product
    path (osfm_ba_set_fallbacks); each is a path some inputs take anyway."""
    pb.validate(check_indices=False)
    unknown = sorted(set(fallbacks) - set(_lib.BA_FALLBACKS))
    if unknown:
        raise ValueError("unknown fallback paths %s; known: %s" % (unknown, sorted(_lib.BA_FALLBACKS)))
    fallback_mask = sum(_lib.BA_FALLBACKS[f] for f in set(fallbacks))
    with _lib.pooled("ba", device) as hd:
        L, h = hd.L, hd.h
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        K, NI, NR = len(pb.cam_type), len(pb.inst), len(pb.rigcam)
        S, P, N = len(pb.shot_inst), len(pb.points), len(pb.obs_shot)
        keep = [i32(pb.cam_type), f64(pb.cam_params), i32(pb.cam_const), f64(pb.cam_prior), f64(pb.cam_prior_sigma),
                i32(pb.cam_prior_log)]
        _lib.check(L.osfm_ba_set_cameras(h, K, *[ptr(a) for a in keep]))
        k2 = [f64(pb.inst), i32(pb.inst_const), i32(pb.inst_has_prior), f64(pb.inst_prior_pos), f64(pb.inst_prior_std)]
        _lib.check(L.osfm_ba_set_rig_instances(h, NI, *[ptr(a) for a in k2]))
        k3 = [f64(pb.rigcam), i32(pb.rigcam_const)]
        _lib.check(L.osfm_ba_set_rig_cameras(h, NR, *[ptr(a) for a in k3]))
        k4 = [i32(pb.shot_inst), i32(pb.shot_cam), i32(pb.shot_rc), i32(pb.shot_use_rc)]
        _lib.check(L.osfm_ba_set_shots(h, S, *[ptr(a) for a in k4]))
        k5 = [f64(pb.points), i32(pb.point_const)]
        _lib.check(L.osfm_ba_set_points(h, P, *[ptr(a) for a in k5]))
        k6 = [i32(pb.obs_shot), i32(pb.obs_point), f64(pb.obs_xy), f64(pb.obs_sigma)]
        set_obs = L.osfm_ba_set_observations_async if pinned_inputs else L.osfm_ba_set_observations
        _lib.check(set_obs(h, N, *[ptr(a) for a in k6]))
        # secondary residuals: always (re)set, the handle is reused between solves
        if pb.rigcam_prior is not None:
            k7 = [f64(pb.rigcam_prior), f64(pb.rigcam_prior_sigma)]
            if k7[0].shape != (NR, 6) or k7[1].shape != (NR, 6):
                raise ValueError("rigcam_prior / rigcam_prior_sigma must be NR x 6")
            _lib.check(L.osfm_ba_set_rig_camera_priors(h, ptr(k7[0]), ptr(k7[1])))
        else:
            _lib.check(L.osfm_ba_set_rig_camera_priors(h, None, None))
        k8 = [i32(pb.pp_point), f64(pb.pp_prior), f64(pb.pp_sigma), i32(pb.pp_alt)]
        _lib.check(L.osfm_ba_set_point_priors(h, len(k8[0]), *[ptr(a) for a in k8]))
        k9 = [i32(pb.ext_size), f64(pb.ext_values), i32(pb.ext_const), f64(pb.ext_lower)]
        _lib.check(L.osfm_ba_set_ext_blocks(h, len(k9[0]), *[ptr(a) for a in k9]))
        recs, consts = pb.packed_side_terms()
        terms = (_lib.SideTerm * max(len(recs), 1))()
        for t, (ty, nres, nb, kind, idx, loss, loss_a, cofs, aux) in zip(terms, recs):
            t.type, t.nres, t.nblocks, t.loss, t.loss_a, t.cofs = ty, nres, nb, loss, loss_a, cofs
            t.kind[:] = kind
            t.idx[:] = idx
            t.aux[:] = aux
        consts = f64(consts)
        _lib.check(L.osfm_ba_set_side_terms(h, len(recs), ctypes.cast(terms, ctypes.c_void_p), len(consts),
                                            ptr(consts)))
        if pb.loss_name not in _lib.LOSS_IDS:
            raise RuntimeError("ceres::LossFunction with name %s not found." % pb.loss_name)  # bundle_adjuster.cc:427
        _lib.check(L.osfm_ba_set_options(h, _lib.LOSS_IDS[pb.loss_name], float(pb.loss_threshold),
                                         int(pb.max_iterations), pb.linear_solver_type.encode(),
                                         int(compute_reprojection_errors)))
        cb = None
        if world > 1:
            if allreduce is None:
                raise ValueError("world > 1 needs allreduce: a callable or the string 'nccl'")
            if isinstance(allreduce, str):
                if allreduce != "nccl":
                    raise ValueError("allreduce must be a callable or 'nccl'")
                # the library's own NCCL communicator (one per handle; the 128-byte id travels over torch.distributed)
                if getattr(hd, "nccl", None) != (int(rank), int(world)):
                    import torch.distributed as tdist

                    buf = ctypes.create_string_buffer(128)
                    if rank == 0:
                        _lib.check(L.osfm_nccl_unique_id(buf))
                    box = [buf.raw]
                    tdist.broadcast_object_list(box, src=0)
                    idb = ctypes.create_string_buffer(box[0], 128)
                    _lib.check(L.osfm_ba_set_nccl(h, int(rank), int(world), idb))
                    hd.nccl = (int(rank), int(world))
                _lib.check(L.osfm_ba_set_distributed(h, int(rank), int(world), ctypes.cast(None, _lib.ALLREDUCE_FN), None))
            else:
                def _cb(buf, count, strm, user):
                    try:
                        allreduce(int(buf), int(count), int(strm or 0))
                        return 0
                    except Exception:  # surfaces as RuntimeError from run()
                        import traceback

                        traceback.print_exc()
                        return 1

                cb = _lib.ALLREDUCE_FN(_cb)
                _lib.check(L.osfm_ba_set_distributed(h, int(rank), int(world), cb, None))
        else:
            # the handle is reused between calls: reset whatever a previous distributed solve left
            _lib.check(L.osfm_ba_set_distributed(h, 0, 1, ctypes.cast(None, _lib.ALLREDUCE_FN), None))
        _lib.check(L.osfm_ba_set_stream(h, ctypes.c_void_p(stream) if stream is not None else None))
        _lib.check(L.osfm_ba_set_compute_covariances(h, int(bool(compute_covariances))))
        # set on every call, 0 included: the handle is reused, and one caller's paths must not reach another's solve
        _lib.check(L.osfm_ba_set_fallbacks(h, fallback_mask))
        if capture_iteration is not None:
            if int(capture_iteration) < 1:
                raise ValueError("capture_iteration must be >= 1")
            _lib.check(L.osfm_ba_capture_linear_system(h, int(capture_iteration)))
        try:
            _lib.check(L.osfm_ba_run(h))
        finally:
            if capture_iteration is not None:   # the handle is reused: later solves run unarmed
                _lib.check(L.osfm_ba_capture_linear_system(h, 0))
        capture = _get_capture(L, h, len(keep[1]), NI, NR, P, len(k9[1])) if capture_iteration is not None else None
        cam = np.zeros_like(keep[1])
        inst = np.zeros((NI, 6))
        rc = np.zeros((NR, 6))
        def _out(name, shape):
            a = out.get(name) if out else None
            if a is None:
                return np.empty(shape)
            if a.shape != shape or a.dtype != np.float64 or not a.flags.c_contiguous:
                raise ValueError("out[%r] must be a C-contiguous float64 array of shape %r" % (name, shape))
            return a

        pts = _out("points", (P, 3))
        rep = _out("reprojection_errors", (N, 3))
        if not compute_reprojection_errors:
            rep[:] = 0.0
        _lib.check(L.osfm_ba_get_cameras(h, ptr(cam)))
        _lib.check(L.osfm_ba_get_rig_instances(h, ptr(inst)))
        _lib.check(L.osfm_ba_get_rig_cameras(h, ptr(rc)))
        _lib.check(L.osfm_ba_get_points(h, ptr(pts)))
        if compute_reprojection_errors:
            _lib.check(L.osfm_ba_get_reprojection_errors(h, ptr(rep)))
        ext = np.zeros(len(k9[1]))
        if len(ext):
            _lib.check(L.osfm_ba_get_ext_blocks(h, ptr(ext)))
        s = _lib.BASummary()
        _lib.check(L.osfm_ba_get_summary(h, ctypes.byref(s)))
        summary = {f[0]: getattr(s, f[0]) for f in s._fields_}
        summary["message"] = s.message.decode()
        summary["termination"] = _TERMINATION[s.termination]
        res = {"cam_params": cam, "inst": inst, "rigcam": rc, "points": pts, "reprojection_errors": rep,
               "ext_values": ext, "summary": summary}
        if capture is not None:
            res["capture"] = capture
        if compute_covariances:
            cov = np.zeros((NI, 6, 6))
            valid, status = ctypes.c_int(0), ctypes.c_int(0)
            _lib.check(L.osfm_ba_get_covariances(h, ctypes.byref(valid), ctypes.byref(status), ptr(cov)))
            res["covariances"] = cov
            res["covariance_valid"] = bool(valid.value)
            res["covariance_status"] = _lib.COVARIANCE_STATUS[status.value]
            pass_ms, chol_ms = ctypes.c_double(), ctypes.c_double()
            _lib.check(L.osfm_ba_get_covariance_timing(h, ctypes.byref(pass_ms), ctypes.byref(chol_ms)))
            res["covariance_ms"] = (pass_ms.value, chol_ms.value)
        return res


def _get_capture(L, h, ncam: int, NI: int, NR: int, P: int, next_: int) -> Dict[str, Any]:
    info = _lib.BACapture()
    _lib.check(L.osfm_ba_get_captured_system(h, ctypes.byref(info), None, None, None, None, None, None))
    nc, n = info.nc, info.n
    cap = {f[0]: getattr(info, f[0]) for f in info._fields_}
    cap["schur_kernel"] = _lib.SCHUR_KERNELS[info.schur_kernel]
    cap["pcg_kernel"] = _lib.PCG_KERNELS[info.pcg_kernel]
    arrs = {"S": np.zeros((nc, nc)), "rhs": np.zeros(nc), "y": np.zeros(nc), "scale": np.zeros(n), "diag": np.zeros(n),
            "grad": np.zeros(n)}
    _lib.check(L.osfm_ba_get_captured_system(h, None, *[ptr(arrs[k]) for k in ("S", "rhs", "y", "scale", "diag",
                                                                                 "grad")]))
    # the linearisation point of the captured iteration
    x = {"cam_params": np.zeros(ncam), "inst": np.zeros((NI, 6)), "rigcam": np.zeros((NR, 6)), "points": np.zeros((P, 3)),
         "ext_values": np.zeros(next_)}
    _lib.check(L.osfm_ba_get_captured_parameters(h, *[ptr(x[k]) for k in ("cam_params", "inst", "rigcam", "points",
                                                                        "ext_values")]))
    cap.update(arrs)
    cap["x"] = x
    return cap


def eval_observation(projection_type: int, camera, rig_instance, rig_camera, use_rig_camera: bool, point, observed,
                     std_deviation: float, device: int = 0):
    """Residual and Jacobian blocks of one observation computed on the GPU (test hook)."""
    L = _lib.load()
    C = bp.camera_num_params(projection_type)
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    cam, ri, pt, ob = f64(camera), f64(rig_instance), f64(point), f64(observed)
    rc = f64(rig_camera if rig_camera is not None else np.zeros(6))
    r, jc, ji, jrc, jp = np.zeros(3), np.zeros(3 * 16), np.zeros(18), np.zeros(18), np.zeros(9)
    n = ctypes.c_int()
    _lib.check(L.osfm_ba_eval_observation(device, int(projection_type), ptr(cam), ptr(ri), ptr(rc),
                                          int(bool(use_rig_camera)), ptr(pt), ptr(ob), float(std_deviation), ptr(r),
                                          ptr(jc), ptr(ji), ptr(jrc), ptr(jp), ctypes.byref(n)))
    k = n.value
    return (r[:k].copy(), jc[:k * C].reshape(k, C).copy(), ji[:k * 6].reshape(k, 6).copy(),
            jrc[:k * 6].reshape(k, 6).copy(), jp[:k * 3].reshape(k, 3).copy())


class Point:
    """bundle::Point as exposed by pybundle (pybind.cc:34-43)."""

    def __init__(self, pid: str, p: np.ndarray):
        self.id = pid
        self.p = p
        self.reprojection_errors: Dict[str, np.ndarray] = {}


class RelativeMotion:
    """bundle::RelativeMotion (bundle_adjuster.h:80-109, pybind.cc:12-20)."""

    def __init__(self, rig_instance_i, rig_instance_j, rotation, translation, scale: float, robust_multiplier: float,
                 observed_scale: bool):
        self.rig_instance_i = rig_instance_i
        self.rig_instance_j = rig_instance_j
        self.parameters = np.concatenate([np.asarray(rotation, dtype=np.float64).reshape(3),
                                          np.asarray(translation, dtype=np.float64).reshape(3), [float(scale)]])
        self.scale_matrix = np.eye(7)
        self.robust_multiplier = float(robust_multiplier)
        self.observed_scale = bool(observed_scale)

    def set_scale_matrix(self, s) -> None:
        self.scale_matrix = np.asarray(s, dtype=np.float64).reshape(7, 7).copy()


class RelativeRotation:
    """bundle::RelativeRotation (bundle_adjuster.h:111-129, pybind.cc:22-29)."""

    def __init__(self, shot_i, shot_j, r):
        self.shot_i = shot_i
        self.shot_j = shot_j
        self.r = np.asarray(r, dtype=np.float64).reshape(3).copy()
        self.scale_matrix = np.eye(3)

    def set_scale_matrix(self, s) -> None:
        self.scale_matrix = np.asarray(s, dtype=np.float64).reshape(3, 3).copy()


class Reconstruction:
    """bundle::Reconstruction (bundle_adjuster.h:25-78, pybind.cc:31-35): per-instance scales; when `shared`,
    every instance reads the first entry of the (sorted) scale map."""

    def __init__(self):
        self.id = ""
        self.scales: Dict[str, float] = {}
        self.constant = False
        self.shared = True

    def _shared_key(self) -> str:
        if not self.scales:
            raise RuntimeError("Shared scale requested but no scale entries exist")
        return min(self.scales)  # std::map::begin()

    def get_scale(self, shot) -> float:
        if self.shared:
            return self.scales[self._shared_key()]
        try:
            return self.scales[_key(shot)]
        except KeyError:
            raise IndexError("map::at")

    def set_scale(self, shot, v: float) -> None:
        if self.shared:
            self.scales[self._shared_key()] = float(v)
        else:
            self.scales[_key(shot)] = float(v)


def _key(s) -> str:
    # ids may be bytes or unicode (opensfm/test/test_bundle.py:20-34)
    return s.decode("utf-8", "replace") if isinstance(s, bytes) else str(s)


_IDENTITY_BIAS = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])


class BundleAdjuster:
    """`pybundle.BundleAdjuster` backed by the GPU engine: same methods, argument meaning, defaults and errors
    (opensfm/src/bundle/python/pybind.cc:45-117, bundle_adjuster.cc:24-44, 94-412).  `run()` turns the collected
    blocks into one BAProblem (numpy index arrays, no per-observation Python work) and calls `solve()`.

    Covariances (set_compute_covariances, bundle_adjuster.cc:1123-1194): run() ends with the rig-instance pose
    covariances of every shot's instance, read with get_rig_instance_covariance; get_covariance_estimation_valid()
    says whether the estimate of the last run is valid (the default matrices otherwise).

    Not available (raise NotImplementedError): heat maps (ceres::BiCubicInterpolator) and relative depth priors."""

    def __init__(self, device: int = 0):
        self.device = device
        self._cams: Dict[str, Dict[str, Any]] = {}
        self._bias: Dict[str, Dict[str, Any]] = {}
        self._rig_cameras: Dict[str, Dict[str, Any]] = {}
        self._instances: Dict[str, Dict[str, Any]] = {}
        self._shots: Dict[str, Dict[str, str]] = {}
        self._shot_index: Dict[str, int] = {}
        # points and observations are kept as growing index / value lists
        self._pt_index: Dict[str, int] = {}
        self._pt_ids: List[str] = []
        self._pt_pos: List[np.ndarray] = []
        self._pt_const: List[int] = []
        self._pt_prior: Dict[int, Any] = {}
        self._pt_errors: Optional[Dict[int, Dict[str, np.ndarray]]] = None
        self._obs_shot: List[Any] = []    # chunks: int lists / arrays
        self._obs_point: List[Any] = []
        self._obs_xy: List[Any] = []
        self._obs_sd: List[Any] = []
        self._cur = ([], [], [], [])      # the chunk add_point_projection_observation appends to
        self._reconstructions: Dict[str, Reconstruction] = {}
        self._assignments: Dict[str, str] = {}
        self._relative_motions: List[RelativeMotion] = []
        self._relative_rotations: List[RelativeRotation] = []
        self._common_positions: List[Any] = []
        self._up_vectors: List[Any] = []
        self._pans: List[Any] = []
        self._tilts: List[Any] = []
        self._rolls: List[Any] = []
        self._linear_motions: List[Any] = []
        self._gauge_fix: Optional[Any] = None
        # defaults of bundle::BundleAdjuster() (bundle_adjuster.cc:24-44, bundle_adjuster.h:315,350-351)
        self._loss = ("CauchyLoss", 1.0)
        self._rm_loss = ("CauchyLoss", 1.0)
        self._prior_sd = dict(focal_sd=1.0, aspect_ratio_sd=1.0, c_sd=1.0, k1_sd=1.0, k2_sd=1.0, p1_sd=1.0,
                              p2_sd=1.0, k3_sd=1.0, k4_sd=1.0)
        self._rig_translation_sd = 1.0
        self._rig_rotation_sd = 1.0
        self._adjust_std = False
        self._max_iterations = 500
        self._num_threads = 1
        self._linear_solver = "SPARSE_SCHUR"
        self._compute_reprojection_errors = True
        self._compute_covariances = False
        self._covariance_valid = False
        self._use_analytic = False
        self._summary: Optional[Dict[str, Any]] = None

    # -- cameras ---------------------------------------------------------
    def add_camera(self, cid, camera, prior, constant: bool) -> None:
        cid = _key(cid)
        self._cams[cid] = dict(type=T.camera_type_id(camera), values=T.camera_values(camera),
                               prior=T.camera_values(prior), constant=bool(constant), proto=camera)
        # identity bias, constant (bundle_adjuster.cc:93-101)
        self._bias[cid] = dict(values=_IDENTITY_BIAS.copy(), constant=True)

    def get_camera(self, cid):
        c = self._cams.get(_key(cid))
        if c is None:
            raise RuntimeError("Camera %s doesn't exist." % _key(cid))  # bundle_adjuster.cc:104
        names = {v: k for k, v in bp.PROJECTION_NAMES.items() if k != "equirectangular"}
        out = T.Camera(names[c["type"]], c["values"])
        out.id = _key(cid)
        return out

    def set_camera_bias(self, cid, rotation, translation, scale: float) -> None:
        """BundleAdjuster::SetCameraBias (bundle_adjuster.cc:103-111; C++-only in the reference, used by
        BAHelpers::Bundle with bundle_compensate_gps_bias): the bias similarity becomes a free 7-parameter block."""
        if _key(cid) not in self._bias:
            raise RuntimeError("Camera %s doesn't exist." % _key(cid))
        self._bias[_key(cid)] = dict(values=np.concatenate([np.asarray(rotation, dtype=np.float64).reshape(3),
                                                            np.asarray(translation, dtype=np.float64).reshape(3),
                                                            [float(scale)]]), constant=False)

    def get_camera_bias(self, cid) -> np.ndarray:
        """[rotation(3) | translation(3) | scale] of the camera's bias (BundleAdjuster::GetBias)."""
        b = self._bias.get(_key(cid))
        if b is None:
            raise RuntimeError("Camera %s doesn't exist." % _key(cid))
        return b["values"].copy()

    # -- rig cameras / instances ------------------------------------------
    def add_rig_camera(self, rid, pose, prior_pose, fixed: bool) -> None:
        rid = _key(rid)
        if rid in self._rig_cameras:
            raise RuntimeError("Rig model %s already exist." % rid)  # bundle_adjuster.cc:155-158
        self._rig_cameras[rid] = dict(params=T.pose_to_ba_params(pose), prior=T.pose_to_ba_params(prior_pose),
                                      constant=bool(fixed))

    def get_rig_camera_pose(self, rid):
        r = self._rig_cameras.get(_key(rid))
        if r is None:
            raise RuntimeError("Rig camera %s doesn't exist." % _key(rid))
        return T.Pose.from_ba_params(r["params"])

    def add_rig_instance(self, iid, pose, shot_cameras: Dict[str, str], shot_rig_cameras: Dict[str, str],
                         fixed: bool) -> None:
        iid = _key(iid)
        if iid not in self._instances:  # std::map::emplace keeps an existing entry
            self._instances[iid] = dict(params=T.pose_to_ba_params(pose), constant=bool(fixed), prior=None,
                                        scale_group=None, cameras=[])
        elif fixed:
            self._instances[iid]["constant"] = True
        for shot_id, cam_id in shot_cameras.items():
            if _key(cam_id) not in self._cams:
                raise RuntimeError("Camera %s doesn't exist." % _key(cam_id))  # bundle_adjuster.cc:130
            try:
                rc_id = _key(shot_rig_cameras[shot_id])
            except KeyError:
                raise IndexError("unordered_map::at")
            if rc_id not in self._rig_cameras:
                raise RuntimeError("Rig camera %s doesn't exist." % rc_id)
            sid = _key(shot_id)
            if sid not in self._shots:
                self._shot_index[sid] = len(self._shots)
                self._shots[sid] = dict(instance=iid, camera=_key(cam_id), rig_camera=rc_id)
                self._instances[iid]["cameras"].append(_key(cam_id))

    def get_rig_instance_pose(self, iid):
        r = self._instances.get(_key(iid))
        if r is None:
            raise RuntimeError("Rig instance %s doesn't exist." % _key(iid))
        return T.Pose.from_ba_params(r["params"])

    def add_rig_instance_position_prior(self, iid, position, std_deviation, scale_group: str = "") -> None:
        r = self._instances.get(_key(iid))
        if r is None:
            raise RuntimeError("Rig instance %s doesn't exist." % _key(iid))  # bundle_adjuster.cc:170
        r["prior"] = (np.asarray(position, dtype=np.float64).reshape(3).copy(),
                      np.asarray(std_deviation, dtype=np.float64).reshape(3).copy())
        r["scale_group"] = _key(scale_group)

    # -- reconstructions (per-instance scales of relative motions) -----------
    def add_reconstruction(self, rid, constant: bool) -> None:
        r = Reconstruction()
        r.id = _key(rid)
        r.constant = bool(constant)
        r.shared = True
        self._reconstructions[r.id] = r

    def add_reconstruction_instance(self, rid, scale: float, instance_id) -> None:
        r = self._reconstructions.get(_key(rid))
        if r is None:
            return
        r.scales[_key(instance_id)] = float(scale)
        self._assignments[_key(instance_id)] = r.id

    def set_scale_sharing(self, rid, share: bool) -> None:
        r = self._reconstructions.get(_key(rid))
        if r is not None:
            r.shared = bool(share)

    def get_reconstruction(self, rid) -> Reconstruction:
        r = self._reconstructions.get(_key(rid))
        if r is None:
            raise RuntimeError("Reconstruction %s doesn't exist." % _key(rid))
        return r

    # -- points / observations --------------------------------------------
    def add_point(self, pid, position, constant: bool) -> None:
        pid = _key(pid)
        if pid in self._pt_index:  # emplace keeps the existing point
            if constant:
                self._pt_const[self._pt_index[pid]] = 1
            return
        self._pt_index[pid] = len(self._pt_ids)
        self._pt_ids.append(pid)
        self._pt_pos.append(np.asarray(position, dtype=np.float64).reshape(3).copy())
        self._pt_const.append(int(bool(constant)))

    def add_points_bulk(self, ids: Sequence[Any], positions: np.ndarray, constant) -> None:
        """Bulk form of add_point: `positions` n x 3, `constant` a bool or an array of n."""
        positions = np.asarray(positions, dtype=np.float64).reshape(-1, 3)
        const = np.broadcast_to(np.asarray(constant, dtype=bool), (len(positions),))
        base = len(self._pt_ids)
        keys = [_key(i) for i in ids]
        fresh = [k not in self._pt_index for k in keys]
        if not all(fresh):
            for k, p, c in zip(keys, positions, const):
                self.add_point(k, p, bool(c))
            return
        self._pt_index.update(zip(keys, range(base, base + len(keys))))
        self._pt_ids.extend(keys)
        self._pt_pos.extend(positions)
        self._pt_const.extend(int(c) for c in const)

    def add_point_prior(self, pid, position, std_deviation, has_altitude_prior: bool) -> None:
        i = self._pt_index.get(_key(pid))
        if i is None:
            raise RuntimeError("Point %s doesn't exist." % _key(pid))  # bundle_adjuster.cc:229
        self._pt_prior[i] = (np.asarray(position, dtype=np.float64).reshape(3).copy(),
                             np.asarray(std_deviation, dtype=np.float64).reshape(3).copy(), bool(has_altitude_prior))

    def has_point(self, pid) -> bool:
        return _key(pid) in self._pt_index

    def get_point(self, pid) -> Point:
        i = self._pt_index.get(_key(pid))
        if i is None:
            raise RuntimeError("Point %s doesn't exist." % _key(pid))
        pt = Point(_key(pid), np.asarray(self._pt_pos[i]).copy())
        if self._pt_errors is not None:
            pt.reprojection_errors = dict(self._pt_errors.get(i, {}))
        return pt

    def add_point_projection_observation(self, shot, point, observation, std_deviation, depth_prior=None) -> None:
        si = self._shot_index.get(_key(shot))
        pi = self._pt_index.get(_key(point))
        if si is None or pi is None:
            # the reference uses std::map::at (bundle_adjuster.cc:242-244) -> IndexError in Python
            raise IndexError("map::at")
        if depth_prior is not None:
            raise NotImplementedError("relative depth priors are outside this engine's scope (SURVEY.md §8a)")
        c = self._cur
        c[0].append(si); c[1].append(pi); c[2].append((float(observation[0]), float(observation[1])))
        c[3].append(float(std_deviation))

    def add_observations_bulk(self, shots: Sequence[Any], points: Sequence[Any], xy: np.ndarray,
                              std_deviation) -> None:
        """Bulk form of add_point_projection_observation (SURVEY.md §7 'String-keyed API'): one dictionary
        lookup per id in C speed, arrays kept as they are (no per-observation Python objects)."""
        try:
            si = np.fromiter((self._shot_index[_key(s)] for s in shots), dtype=np.int32)
            pi = np.fromiter((self._pt_index[_key(p)] for p in points), dtype=np.int32)
        except KeyError:
            raise IndexError("map::at")
        xy = np.asarray(xy, dtype=np.float64).reshape(-1, 2)
        sd = np.broadcast_to(np.asarray(std_deviation, dtype=np.float64), (len(si),))
        if not (len(si) == len(pi) == len(xy)):
            raise ValueError("shots, points and xy differ in length")
        self._flush_obs()
        self._obs_shot.append(si); self._obs_point.append(pi); self._obs_xy.append(xy); self._obs_sd.append(np.array(sd))

    def _flush_obs(self) -> None:
        c = self._cur
        if c[0]:
            self._obs_shot.append(np.asarray(c[0], dtype=np.int32))
            self._obs_point.append(np.asarray(c[1], dtype=np.int32))
            self._obs_xy.append(np.asarray(c[2], dtype=np.float64).reshape(-1, 2))
            self._obs_sd.append(np.asarray(c[3], dtype=np.float64))
            self._cur = ([], [], [], [])

    # -- secondary residual blocks ------------------------------------------------
    def add_relative_motion(self, rm: RelativeMotion) -> None:
        self._relative_motions.append(rm)

    def add_relative_rotation(self, rr: RelativeRotation) -> None:
        self._relative_rotations.append(rr)

    def add_common_position(self, shot_i, shot_j, margin: float, std_deviation: float) -> None:
        self._common_positions.append((_key(shot_i), _key(shot_j), float(margin), float(std_deviation)))

    def add_absolute_up_vector(self, shot_id, up_vector, std_deviation: float) -> None:
        self._up_vectors.append((_key(shot_id), np.asarray(up_vector, dtype=np.float64).reshape(3).copy(),
                                 float(std_deviation)))

    def add_absolute_pan(self, shot_id, angle: float, std_deviation: float) -> None:
        self._pans.append((_key(shot_id), float(angle), float(std_deviation)))

    def add_absolute_tilt(self, shot_id, angle: float, std_deviation: float) -> None:
        self._tilts.append((_key(shot_id), float(angle), float(std_deviation)))

    def add_absolute_roll(self, shot_id, angle: float, std_deviation: float) -> None:
        self._rolls.append((_key(shot_id), float(angle), float(std_deviation)))

    def add_linear_motion(self, shot0, shot1, shot2, alpha: float, position_std_deviation: float,
                          orientation_std_deviation: float) -> None:
        self._linear_motions.append((_key(shot0), _key(shot1), _key(shot2), float(alpha),
                                     float(position_std_deviation), float(orientation_std_deviation)))

    def set_gauge_fix_shots(self, shot_origin, shot_scale) -> None:
        try:
            s = self._shots[_key(shot_origin)]
        except KeyError:
            raise IndexError("map::at")
        self._instances[s["instance"]]["constant"] = True  # bundle_adjuster.cc:330-335
        self._gauge_fix = (_key(shot_origin), _key(shot_scale))

    def add_heatmap(self, *a, **k):
        raise NotImplementedError("heat-map position priors (ceres::BiCubicInterpolator) are not part of this engine")

    add_absolute_position_heatmap = add_heatmap

    # -- options -----------------------------------------------------------
    def set_point_projection_loss_function(self, name: str, threshold: float) -> None:
        self._loss = (name, float(threshold))

    def set_relative_motion_loss_function(self, name: str, threshold: float) -> None:
        self._rm_loss = (name, float(threshold))

    def set_internal_parameters_prior_sd(self, focal_sd, aspect_ratio_sd, c_sd, k1_sd, k2_sd, p1_sd, p2_sd, k3_sd,
                                         k4_sd) -> None:
        self._prior_sd = dict(focal_sd=focal_sd, aspect_ratio_sd=aspect_ratio_sd, c_sd=c_sd, k1_sd=k1_sd,
                              k2_sd=k2_sd, p1_sd=p1_sd, p2_sd=p2_sd, k3_sd=k3_sd, k4_sd=k4_sd)

    def set_rig_parameters_prior_sd(self, rig_translation_sd: float, rig_rotation_sd: float) -> None:
        """BundleAdjuster::SetRigParametersPriorSD (bundle_adjuster.cc:394-402; C++-only in the reference)."""
        self._rig_translation_sd = float(rig_translation_sd)
        self._rig_rotation_sd = float(rig_rotation_sd)

    def set_max_num_iterations(self, n: int) -> None:
        self._max_iterations = int(n)

    def set_num_threads(self, n: int) -> None:
        self._num_threads = int(n)

    def set_use_analytic_derivatives(self, use: bool) -> None:
        self._use_analytic = bool(use)  # the GPU engine is always analytic

    def set_linear_solver_type(self, name: str) -> None:
        self._linear_solver = name

    def set_compute_reprojection_errors(self, v: bool) -> None:
        self._compute_reprojection_errors = bool(v)

    def set_compute_covariances(self, v: bool) -> None:
        self._compute_covariances = bool(v)

    def get_covariance_estimation_valid(self) -> bool:
        return self._covariance_valid

    def get_rig_instance_covariance(self, iid) -> np.ndarray:
        """RigInstance::GetCovariance of the reference (bundle/data/data.h:62-66): the 6 x 6 covariance of the
        instance's [rx, ry, rz, tx, ty, tz] from the last run with covariances on."""
        r = self._instances.get(_key(iid))
        if r is None:
            raise RuntimeError("Rig instance %s doesn't exist." % _key(iid))
        # only instances of shots get one (ComputeCovariances walks the shots)
        if r.get("covariance") is None or not r["cameras"]:
            raise RuntimeError("%s hasn't any covariance" % _key(iid))
        return r["covariance"].copy()

    def set_adjust_absolute_position_std(self, v: bool) -> None:
        self._adjust_std = bool(v)

    # -- run ---------------------------------------------------------------
    def _rm_loss_id(self) -> int:
        if self._rm_loss[0] not in bp.LOSS_IDS:
            raise RuntimeError("ceres::LossFunction with name %s not found." % self._rm_loss[0])
        return bp.LOSS_IDS[self._rm_loss[0]]

    def to_problem(self) -> bp.BAProblem:
        self._flush_obs()
        cam_ids = list(self._cams)
        cam_index = {c: i for i, c in enumerate(cam_ids)}
        inst_ids = list(self._instances)
        inst_index = {c: i for i, c in enumerate(inst_ids)}
        rc_ids = list(self._rig_cameras)
        rc_index = {c: i for i, c in enumerate(rc_ids)}
        shot_ids = list(self._shots)
        self._order = (cam_ids, inst_ids, rc_ids, shot_ids)
        NI = len(inst_ids)
        rigcam = np.array([self._rig_cameras[r]["params"] for r in rc_ids]).reshape(-1, 6) if rc_ids else np.zeros((1, 6))
        rc_const = np.array([self._rig_cameras[r]["constant"] for r in rc_ids], dtype=np.int32) if rc_ids else np.ones(1, dtype=np.int32)
        # IsRigCameraUseful (bundle_adjuster.cc:17-20): free parameters or a non-zero pose
        useful = {r: (not self._rig_cameras[r]["constant"]) or bool(np.any(self._rig_cameras[r]["params"] != 0.0))
                  for r in rc_ids}
        n_obs = sum(len(a) for a in self._obs_shot)
        cat = lambda chunks, shape, dt: (np.concatenate(chunks) if chunks else np.zeros(shape, dtype=dt))
        obs_shot = cat(self._obs_shot, 0, np.int32)
        obs_point = cat(self._obs_point, 0, np.int32)
        obs_xy = cat(self._obs_xy, (0, 2), np.float64)
        obs_sigma = cat(self._obs_sd, 0, np.float64)
        assert len(obs_shot) == n_obs
        pb = bp.make_problem(
            [self._cams[c]["type"] for c in cam_ids], [self._cams[c]["values"] for c in cam_ids],
            np.array([self._instances[i]["params"] for i in inst_ids]).reshape(-1, 6),
            np.array(self._pt_pos).reshape(-1, 3),
            obs_shot, obs_point, obs_xy, obs_sigma,
            shot_inst=[inst_index[self._shots[s]["instance"]] for s in shot_ids],
            shot_cam=[cam_index[self._shots[s]["camera"]] for s in shot_ids],
            rigcam=rigcam, shot_rc=[rc_index[self._shots[s]["rig_camera"]] for s in shot_ids],
            shot_use_rc=[int(useful[self._shots[s]["rig_camera"]]) for s in shot_ids],
            cam_const=[int(self._cams[c]["constant"]) for c in cam_ids],
            inst_const=[int(self._instances[i]["constant"]) for i in inst_ids],
            rigcam_const=rc_const, point_const=np.asarray(self._pt_const, dtype=np.int32),
            cam_prior_list=[self._cams[c]["prior"] for c in cam_ids], prior_sd=self._prior_sd,
            loss_name=self._loss[0], loss_threshold=self._loss[1], max_iterations=self._max_iterations,
            linear_solver_type=self._linear_solver, num_threads=self._num_threads)

        # rig-camera pose priors with sigma GetDefaultRigPoseSigma (bundle_adjuster.cc:69-74, 779-790)
        if rc_ids:
            pb.rigcam_prior = np.array([self._rig_cameras[r]["prior"] for r in rc_ids]).reshape(-1, 6)
            pb.rigcam_prior_sigma = np.tile([self._rig_rotation_sd] * 3 + [self._rig_translation_sd] * 3, (len(rc_ids), 1))
        # point priors
        if self._pt_prior:
            idx = sorted(self._pt_prior)
            pb.pp_point = np.array(idx, dtype=np.int32)
            pb.pp_prior = np.array([self._pt_prior[i][0] for i in idx])
            pb.pp_sigma = np.array([self._pt_prior[i][1] for i in idx])
            pb.pp_alt = np.array([int(self._pt_prior[i][2]) for i in idx], dtype=np.int32)

        # DUAL transition barrier (bundle_adjuster.cc:610-625)
        for c in cam_ids:
            if self._cams[c]["type"] == bp.DUAL:
                pb.side_terms.append(bp.parameter_barrier_term(cam_index[c], bp.CAMERA_PARAM_NAMES[bp.DUAL].index("transition")))

        # position priors (bundle_adjuster.cc:710-778): plain rows when the bias is the constant identity and the
        # std-deviation scale is locked (the common case), the general term otherwise
        self._ext_of: Dict[Any, int] = {}
        groups: Dict[str, int] = {}
        has_prior = np.zeros(NI, dtype=np.int32)
        ppos = np.zeros((NI, 3))
        pstd = np.ones((NI, 3))
        for i, iid in enumerate(inst_ids):
            inst = self._instances[iid]
            if inst["prior"] is None:
                continue
            if not inst["cameras"]:
                raise RuntimeError("Reference camera of RigInstance %s doesn't have associated Bias" % iid)
            # shot_cameras is an unordered_map in the reference (begin() is unspecified); first shot added here
            bias_cam = inst["cameras"][0]
            bias = self._bias[bias_cam]
            simple = bias["constant"] and np.array_equal(bias["values"], _IDENTITY_BIAS) and not self._adjust_std
            if simple:
                has_prior[i] = 1
                ppos[i], pstd[i] = inst["prior"]
                continue
            kb = ("bias", bias_cam)
            if kb not in self._ext_of:
                self._ext_of[kb] = pb.add_ext_block(bias["values"], bias["constant"])
            g = inst["scale_group"] or ""
            kg = ("std", g)
            if kg not in self._ext_of:
                self._ext_of[kg] = pb.add_ext_block([1.0], not self._adjust_std, [1e-10])
                groups[g] = self._ext_of[kg]
            pb.side_terms.append(bp.position_prior_term(i, self._ext_of[kb], self._ext_of[kg], inst["prior"][0],
                                                        inst["prior"][1], self._adjust_std))
        if self._adjust_std:
            for g, e in groups.items():
                pb.side_terms.append(bp.std_deviation_term(e))
        pb.inst_has_prior = has_prior
        pb.inst_prior_pos = ppos
        pb.inst_prior_std = pstd

        def shot(sid):
            try:
                s = self._shots[sid]
            except KeyError:
                raise IndexError("map::at")
            return inst_index[s["instance"]], rc_index[s["rig_camera"]], useful[s["rig_camera"]]

        # reconstruction scales (bundle_adjuster.cc:672-685): one 1-parameter block per scale entry, lower bound 0
        def scale_block(iid):
            try:
                r = self._reconstructions[self._assignments[iid]]
            except KeyError:
                raise IndexError("map::at")
            entry = r._shared_key() if r.shared else iid
            k = ("scale", r.id, entry)
            if k not in self._ext_of:
                self._ext_of[k] = pb.add_ext_block([r.scales[entry]], r.constant, [0.0])
            return self._ext_of[k]

        for rm in self._relative_motions:
            try:
                ii, ij = inst_index[_key(rm.rig_instance_i)], inst_index[_key(rm.rig_instance_j)]
            except KeyError:
                raise IndexError("map::at")
            pb.side_terms.append(bp.relative_motion_term(
                ii, ij, scale_block(_key(rm.rig_instance_i)), scale_block(_key(rm.rig_instance_j)), rm.parameters,
                rm.scale_matrix, rm.observed_scale, self._rm_loss_id(), self._rm_loss[1] * rm.robust_multiplier))
        for rr in self._relative_rotations:
            (ii, ri, ui), (ij, rj, uj) = shot(_key(rr.shot_i)), shot(_key(rr.shot_j))
            pb.side_terms.append(bp.relative_rotation_term(ii, ij, ri if ui else None, rj if uj else None, rr.r,
                                                           rr.scale_matrix, self._rm_loss_id(), self._rm_loss[1]))
        for si, sj, margin, sd in self._common_positions:
            (ii, ri, ui), (ij, rj, uj) = shot(si), shot(sj)
            pb.side_terms.append(bp.common_position_term(ii, ij, ri if ui else None, rj if uj else None, margin, sd))
        for sid, up, sd in self._up_vectors:
            if sd > 0:
                i, r, _ = shot(sid)
                pb.side_terms.append(bp.up_vector_term(i, r, up, sd))
        for which, lst in ((bp.SIDE_PAN, self._pans), (bp.SIDE_TILT, self._tilts), (bp.SIDE_ROLL, self._rolls)):
            for sid, angle, sd in lst:
                if sd > 0:
                    i, r, _ = shot(sid)
                    pb.side_terms.append(bp.angle_term(which, i, r, angle, sd))
        for s0, s1, s2, alpha, psd, osd in self._linear_motions:
            t = [shot(s0), shot(s1), shot(s2)]
            pb.side_terms.append(bp.linear_motion_term([x[0] for x in t], [x[1] if x[2] else None for x in t], alpha, psd, osd))
        if self._gauge_fix is not None:
            i1, i2 = shot(self._gauge_fix[0])[0], shot(self._gauge_fix[1])[0]
            norm = float(np.linalg.norm(pb.inst[i1, 3:] - pb.inst[i2, 3:]))
            pb.side_terms.append(bp.translation_prior_term(i1, i2, norm))
        return pb

    def run(self) -> None:
        pb = self.to_problem()
        self.apply_results(pb, solve(pb, device=self.device,
                                     compute_reprojection_errors=self._compute_reprojection_errors,
                                     compute_covariances=self._compute_covariances))

    def apply_results(self, pb: bp.BAProblem, res: Dict[str, Any]) -> None:
        """Write the arrays of a solve of `pb` (= self.to_problem()) back into the per-id containers the getters
        read.  Separate from run() so that the parity tests can push the same problem through the oracle."""
        cam_ids, inst_ids, rc_ids, shot_ids = self._order
        off = pb.cam_off
        for i, c in enumerate(cam_ids):
            self._cams[c]["values"] = res["cam_params"][off[i]:off[i + 1]].copy()
        for i, iid in enumerate(inst_ids):
            self._instances[iid]["params"] = res["inst"][i].copy()
        for i, r in enumerate(rc_ids):
            self._rig_cameras[r]["params"] = res["rigcam"][i].copy()
        self._pt_pos = list(res["points"])
        eo = pb.ext_off
        for k, e in self._ext_of.items():
            vals = res["ext_values"][eo[e]:eo[e + 1]]
            if k[0] == "bias":
                self._bias[k[1]]["values"] = vals.copy()
            elif k[0] == "scale":
                self._reconstructions[k[1]].scales[k[2]] = float(vals[0])
        if "covariances" in res:
            for i, iid in enumerate(inst_ids):
                self._instances[iid]["covariance"] = np.asarray(res["covariances"][i], dtype=np.float64).copy()
            self._covariance_valid = bool(res["covariance_valid"])
        self._pt_errors = None
        if self._compute_reprojection_errors:
            # Point::reprojection_errors: shot id -> 2-vector (3 for spherical cameras), bundle_adjuster.cc:531-566
            rep = res["reprojection_errors"]
            sph = np.array([self._cams[self._shots[s]["camera"]]["type"] == bp.SPHERICAL for s in shot_ids], dtype=bool)
            errs: Dict[int, Dict[str, np.ndarray]] = {}
            for k, (si, pi) in enumerate(zip(pb.obs_shot.tolist(), pb.obs_point.tolist())):
                errs.setdefault(pi, {})[shot_ids[si]] = rep[k, :3].copy() if sph[si] else rep[k, :2].copy()
            self._pt_errors = errs
        self._last = (pb, res)
        self._summary = res["summary"]

    def results(self):
        """(BAProblem, result arrays of solve()) of the last run: the bulk read-back for callers that do not want
        per-id getters (SURVEY.md §8f.2)."""
        return self._last

    def brief_report(self) -> str:
        s = self._summary
        if s is None:
            return "Solver has not run."
        return ("opensfm_b200 BA Report: Iterations: %d, Initial cost: %e, Final cost: %e, Termination: %s"
                % (s["iterations"], s["initial_cost"], s["final_cost"], s["termination"]))

    def full_report(self) -> str:
        s = self._summary
        if s is None:
            return "Solver has not run."
        return self.brief_report() + "\n" + "\n".join("%s: %s" % kv for kv in s.items())
