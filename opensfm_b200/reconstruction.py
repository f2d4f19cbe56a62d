"""Drop-in replacements of `opensfm.reconstruction.bundle`, `bundle_shot_poses`, `bundle_local` (and
`remove_outliers`) on the GPU engine  --  boundary B-py-1 of SURVEY.md §8b.

The reference implements them in C++ (`sfm::BAHelpers`, opensfm/src/sfm/src/ba_helpers.cc) on top of its own copy
of `bundle::BundleAdjuster`; replacing `pybundle` alone would not change them, so the same logic lives here on top
of `opensfm_b200.bundle.BundleAdjuster`:

  bundle             ba_helpers.cc:581-763   global BA: everything free (cameras iff optimize_camera_parameters),
                                             GPS position priors, up-vector alignment prior, GCP, camera biases
  bundle_shot_poses  ba_helpers.cc:408-579   only the poses of the given shots' rig instances
  bundle_local       ba_helpers.cc:117-311   interior of the shot neighbourhood free, its boundary fixed
  shot_neighborhood  ba_helpers.cc:37-115    interior / boundary by co-visibility
  add_gcp_to_bundle  ba_helpers.cc:349-406 ; bundle_to_map :765-819 (NaN guards) ; report keys :287-309, 743-762

`reconstruction` is duck-typed: `opensfm.types.Reconstruction` or `opensfm_b200.map_types.Reconstruction` (same
attribute names).  To re-point OpenSfM:  `opensfm.reconstruction.bundle = opensfm_b200.reconstruction.bundle`, etc.
(INTEGRATION.md §2).  Every call runs on the GPU; there is no CPU fallback.

The ranking of image pairs that `incremental_reconstruction` bootstraps from is here too, batched over all pairs
by the rotation-only RANSAC of opensfm_b200/rotation_ransac.py:

  compute_image_pairs                     reconstruction.py:208-244
  compute_image_pairs_sequential          reconstruction.py:1684-1709
  two_view_reconstruction_rotation_only   reconstruction.py:387-412
  compute_image_pairs_from_tracks         this engine's fast path: bearings once per image, rows from the device's
                                          common-track lists

and the triangulation of tracks after each shot the incremental loop adds, from opensfm_b200/triangulation.py:

  triangulate_shot_features               reconstruction.py:1143-1183
  retriangulate                           reconstruction.py:1186-1226

and the resection of the incremental loop, batched over every candidate image by the absolute-pose RANSAC of
opensfm_b200/resection.py:

  reconstructed_points_for_images         reconstruction.py:677-692  (ties in the order of tracks_manager.images)
  add_shot                                reconstruction.py:247-285
  resect                                  reconstruction.py:695-762
  resect_candidates                       the inner `for image, _ in candidates` loop of grow_reconstruction
                                          (:1495-1575): every candidate in one launch, the first success applied
  exif_to_metadata, get_image_metadata    reconstruction_helpers.py:129-185
  rig_assignments_per_image               rig.py:39-52
"""
from __future__ import annotations

import logging
import time
from typing import Any, Dict, Iterable, List, Optional, Sequence, Set, Tuple

import numpy as np

from . import bundle as _bundle
from . import resection as _rs
from . import rotation_ransac as _rr
from . import types as T
from .map_types import RigInstance, ShotMeasurements
from .triangulation import retriangulate, triangulate_shot_features  # noqa: F401

logger = logging.getLogger(__name__)


# ---------------------------------------------------------------------------------------------------------------
# small accessors over the duck-typed map
# ---------------------------------------------------------------------------------------------------------------
def _items(view) -> Iterable[Tuple[str, Any]]:
    return view.items()


def _shot_observations(shot) -> List[Tuple[Any, Any]]:
    """[(landmark, observation)] of a shot (Shot::GetLandmarkObservations)."""
    return [(lm, shot.get_landmark_observation(lm)) for lm in shot.get_valid_landmarks()]


def _instance_shots(instance) -> Dict[str, str]:
    """shot id -> rig camera id of a rig instance (RigInstance::GetRigCameras)."""
    return dict(instance.rig_camera_ids)


def _bias_values(bias) -> np.ndarray:
    if isinstance(bias, np.ndarray):
        return bias
    return np.concatenate([np.asarray(bias.rotation, dtype=np.float64), np.asarray(bias.translation, dtype=np.float64),
                           [float(bias.scale)]])


def _write_pose(holder, attr: str, ba_params: np.ndarray, what: str) -> None:
    """holder.<attr> <- pose given as [angle-axis camera->world | origin]; raises like BundleToMap on NaN/Inf."""
    if not np.all(np.isfinite(ba_params)):
        raise RuntimeError("%s has either NaN or INF values." % what)
    pose = getattr(holder, attr)
    new = T.Pose.from_ba_params(ba_params)
    pose.set_rotation_matrix(new.get_rotation_matrix())
    pose.set_origin(new.get_origin())
    setattr(holder, attr, pose)


def _configure(ba: _bundle.BundleAdjuster, config: Dict[str, Any]) -> None:
    ba.set_use_analytic_derivatives(config["bundle_analytic_derivatives"])
    ba.set_point_projection_loss_function(config["loss_function"], config["loss_function_threshold"])
    ba.set_internal_parameters_prior_sd(
        config["exif_focal_sd"], config["aspect_ratio_sd"], config["principal_point_sd"],
        config["radial_distortion_k1_sd"], config["radial_distortion_k2_sd"], config["tangential_distortion_p1_sd"],
        config["tangential_distortion_p2_sd"], config["radial_distortion_k3_sd"], config["radial_distortion_k4_sd"])
    ba.set_rig_parameters_prior_sd(config["rig_translation_sd"], config["rig_rotation_sd"])
    ba.set_num_threads(config["processes"])


def _report(ba, t0, t1, t2, t3) -> Dict[str, Any]:
    return {"brief_report": ba.brief_report(),
            "wall_times": {"setup": t1 - t0, "run": t2 - t1, "teardown": t3 - t2}}


def _add_observations(ba, triples: List[Tuple[str, str, Any]]) -> int:
    """AddPointProjectionObservation for (shot id, landmark id, observation) triples, in one bulk call."""
    if not triples:
        return 0
    if any(getattr(o, "depth_prior", None) is not None for _, _, o in triples):
        raise NotImplementedError("relative depth priors are outside this engine's scope (SURVEY.md §8a)")
    ba.add_observations_bulk([t[0] for t in triples], [t[1] for t in triples],
                             np.array([t[2].point for t in triples], dtype=np.float64).reshape(-1, 2),
                             np.array([t[2].scale for t in triples], dtype=np.float64))
    return len(triples)


# ---------------------------------------------------------------------------------------------------------------
# shot neighbourhood (ba_helpers.cc:37-115)
# ---------------------------------------------------------------------------------------------------------------
def _direct_shot_neighbors(reconstruction, shot_ids: Set[str], min_common_points: int, max_neighbors: int) -> Set[str]:
    points = {}
    for sid in shot_ids:
        for lm in reconstruction.shots[sid].get_valid_landmarks():
            points[lm.id] = lm
    common: Dict[str, int] = {}
    for lm in points.values():
        for shot in lm.get_observations():
            if shot.id not in shot_ids:
                common[shot.id] = common.get(shot.id, 0) + 1
    pairs = sorted(common.items(), key=lambda kv: -kv[1])
    neighbors: Set[str] = set()
    for idx, (sid, n) in enumerate(pairs):
        if n >= min_common_points and idx < min(max_neighbors, len(pairs)):
            inst = reconstruction.rig_instances[reconstruction.shots[sid].rig_instance_id]
            neighbors.update(_instance_shots(inst))
        else:
            break
    return neighbors


def shot_neighborhood_ids(reconstruction, central_shot_id: str, radius: int, min_common_points: int,
                          max_interior_size: int) -> Tuple[Set[str], Set[str]]:
    """(interior, boundary) shot ids: the central shot (and its rig instance) is at distance 0; shots at distance
    n + 1 share at least min_common_points points with shots at distance n; the boundary shares at least one point
    with the interior."""
    central = reconstruction.shots[central_shot_id]
    interior = set(_instance_shots(reconstruction.rig_instances[central.rig_instance_id]))
    interior.add(central_shot_id)
    distance = 1
    while distance < radius and len(interior) < max_interior_size:
        remaining = max_interior_size - len(interior)
        interior |= _direct_shot_neighbors(reconstruction, interior, min_common_points, remaining)
        distance += 1
    boundary = _direct_shot_neighbors(reconstruction, interior, 1, 1000000)
    return interior, boundary


# ---------------------------------------------------------------------------------------------------------------
# ground control points (ba_helpers.cc:313-406)
# ---------------------------------------------------------------------------------------------------------------
def _angle(u, v) -> float:
    c = float(np.dot(u, v) / np.sqrt(np.dot(u, u) * np.dot(v, v)))
    return 0.0 if abs(c) >= 1.0 else float(np.arccos(c))


def triangulate_bearings_midpoint(centers: np.ndarray, bearings: np.ndarray, thresholds: Sequence[float],
                                  min_angle: float, min_depth: float) -> Tuple[bool, np.ndarray]:
    """geometry::TriangulateBearingsMidpoint (geometry/src/triangulation.cc:137-177, solve triangulation.h:58-82)."""
    n = len(centers)
    if len(thresholds) < n:
        return False, np.zeros(3)
    if not any(min_angle <= _angle(bearings[i], bearings[j]) <= np.pi - min_angle for i in range(n) for j in range(i)):
        return False, np.zeros(3)
    BBt = bearings.T @ bearings
    BBtA = sum(np.outer(bearings[i], bearings[i]) @ centers[i] for i in range(n))
    A = centers.sum(axis=0)
    Cinv = np.linalg.inv(n * np.eye(3) - BBt)
    X = (np.eye(3) + BBt @ Cinv) @ A / n - Cinv @ BBtA
    for i in range(n):
        projected = X - centers[i]
        if _angle(projected, bearings[i]) > thresholds[i] or float(np.dot(projected, bearings[i])) < min_depth:
            return False, np.zeros(3)
    return True, X


def triangulate_gcp(point, shots) -> Tuple[bool, np.ndarray]:
    """BAHelpers::TriangulateGCP: needs `camera.pixel_bearing` on the shots' cameras (pygeometry.Camera has it)."""
    os_, bs = [], []
    for obs in point.observations:
        shot = shots.get(obs.shot_id) if hasattr(shots, "get") else (shots[obs.shot_id] if obs.shot_id in shots else None)
        if shot is None:
            continue
        if not hasattr(shot.camera, "pixel_bearing"):
            return False, np.zeros(3)
        b = np.asarray(shot.camera.pixel_bearing(obs.projection), dtype=np.float64)
        bs.append(shot.pose.get_rotation_matrix().T @ b)
        os_.append(shot.pose.get_origin())
    if len(os_) >= 2:
        return triangulate_bearings_midpoint(np.array(os_), np.array(bs), [1.0] * len(os_), 0.1 * np.pi / 180.0, 1e-3)
    return False, np.zeros(3)


def _gcp_topocentric(reconstruction, point) -> np.ndarray:
    ref = getattr(reconstruction, "reference", None)
    if ref is None:
        raise RuntimeError("ground control points with lla need reconstruction.reference (TopocentricConverter)")
    lla = point.lla
    return np.asarray(ref.to_topocentric(lla["latitude"], lla["longitude"], lla.get("altitude", 0.0)), dtype=np.float64)


def add_gcp_to_bundle(ba: _bundle.BundleAdjuster, reconstruction, gcp, config: Dict[str, Any], dominant_terms: int) -> int:
    """BAHelpers::AddGCPToBundle: a free point per GCP ("gcp-<id>"), its prior from the lla, its observations with
    std 0.001 / global_weight."""
    shots = reconstruction.shots
    total_terms = 0
    tri = {}
    for point in gcp:
        tri[point.id] = triangulate_gcp(point, shots)
        if tri[point.id][0] or point.lla:
            total_terms += 1
        total_terms += sum(1 for o in point.observations if o.shot_id in shots)
    global_weight = config["gcp_global_weight"] * dominant_terms / max(1, total_terms)
    added = 0
    for point in gcp:
        pid = "gcp-" + point.id
        ok, coordinates = tri[point.id]
        if not ok:
            if point.lla:
                coordinates = _gcp_topocentric(reconstruction, point)
            else:
                continue
        ba.add_point(pid, coordinates, False)
        if point.lla:
            std = np.array([config["gcp_horizontal_sd"], config["gcp_horizontal_sd"], config["gcp_vertical_sd"]])
            ba.add_point_prior(pid, _gcp_topocentric(reconstruction, point), std / global_weight, bool(point.has_altitude))
        for obs in point.observations:
            if obs.shot_id in shots:
                ba.add_point_projection_observation(obs.shot_id, pid, obs.projection, 0.001 / global_weight)
                added += 1
    return added


# ---------------------------------------------------------------------------------------------------------------
# alignment constraints (ba_helpers.cc:821-891)
# ---------------------------------------------------------------------------------------------------------------
def detect_alignment_constraints(reconstruction, config: Dict[str, Any], gcp) -> str:
    X = []
    if gcp and config["bundle_use_gcp"]:
        for point in gcp:
            if point.lla:
                ok, c = triangulate_gcp(point, reconstruction.shots)
                if ok:
                    X.append(c)
    if config["bundle_use_gps"]:
        for _, shot in _items(reconstruction.shots):
            if shot.metadata.gps_position.has_value:
                X.append(np.asarray(shot.pose.get_origin(), dtype=np.float64))
    if len(X) < 3:
        return "orientation_prior"
    X = np.array(X)
    Xz = X - X.mean(axis=0)
    evals = np.linalg.eigvalsh(Xz.T @ Xz)
    ratio = abs(evals[2] / evals[1]) if evals[1] != 0 else np.inf
    is_line = int((evals < 1e-10).sum()) > 1 or ratio > 5e3
    return "orientation_prior" if is_line else "naive"


# ---------------------------------------------------------------------------------------------------------------
# instances with their averaged GPS prior (shared by the three flavours)
# ---------------------------------------------------------------------------------------------------------------
def _add_instance(ba, reconstruction, instance_id: str, instance, config, fixed_if, use_gps_of, check_accuracy: bool):
    """AddRigInstance + the position prior averaged over the instance's shots (ba_helpers.cc:170-216, 467-516,
    641-683).  fixed_if(shot_id) -> the whole instance is fixed; use_gps_of(shot_id) -> its GPS counts."""
    shot_cameras, shot_rig_cameras = {}, {}
    avg = np.zeros(3)
    avg_std, count = 0.0, 0
    fix = False
    for shot_id, rig_camera_id in _instance_shots(instance).items():
        shot = reconstruction.shots[shot_id]
        shot_cameras[shot_id] = shot.camera.id
        shot_rig_cameras[shot_id] = rig_camera_id
        if fixed_if(shot_id):
            fix = True
        elif config["bundle_use_gps"] and use_gps_of(shot_id):
            pos, acc = shot.metadata.gps_position, shot.metadata.gps_accuracy
            if pos.has_value and acc.has_value:
                if check_accuracy and acc.value <= 0:
                    raise RuntimeError("Shot %s has an accuracy <= 0: %f. Try modifying your input parser to filter such "
                                       "values." % (shot_id, acc.value))
                avg += np.asarray(pos.value, dtype=np.float64)
                avg_std += float(acc.value)
                count += 1
    ba.add_rig_instance(instance_id, instance.pose, shot_cameras, shot_rig_cameras, fix)
    if not fix and count > 0:
        ba.add_rig_instance_position_prior(instance_id, avg / count, np.full(3, avg_std / count), "dummy")


# ---------------------------------------------------------------------------------------------------------------
# the three entry points
# ---------------------------------------------------------------------------------------------------------------
def bundle(reconstruction, camera_priors: Dict[str, Any], rig_camera_priors: Dict[str, Any], gcp: Optional[List[Any]],
           config: Dict[str, Any]) -> Dict[str, Any]:
    """opensfm.reconstruction.bundle (reconstruction.py:69-86) = BAHelpers::Bundle."""
    t0 = time.perf_counter()
    gcp = gcp if gcp is not None else []
    ba = _bundle.BundleAdjuster()
    fix_cameras = not config["optimize_camera_parameters"]
    for cam_id, cam in _items(reconstruction.cameras):
        ba.add_camera(cam_id, cam, camera_priors[cam_id], fix_cameras)
    pts = list(_items(reconstruction.points))
    ba.add_points_bulk([p for p, _ in pts], np.array([lm.coordinates for _, lm in pts], dtype=np.float64).reshape(-1, 3), False)

    align_method = config["align_method"]
    if align_method == "auto":
        align_method = detect_alignment_constraints(reconstruction, config, gcp)
    up_vector = None
    if align_method == "orientation_prior":
        if config["align_orientation_prior"] == "vertical":
            up_vector = np.array([0.0, 0.0, -1.0])
        elif config["align_orientation_prior"] == "horizontal":
            up_vector = np.array([0.0, -1.0, 0.0])

    n_rc = len(reconstruction.rig_cameras)
    shots_per_rig_camera = len(reconstruction.shots) // n_rc if n_rc > 0 else 1
    lock_rig_camera = shots_per_rig_camera <= 10
    for rc_id, rc in _items(reconstruction.rig_cameras):
        is_leverarm = rc_id in reconstruction.cameras
        ba.add_rig_camera(rc_id, rc.pose, rig_camera_priors[rc_id].pose, is_leverarm or lock_rig_camera)

    for inst_id, inst in _items(reconstruction.rig_instances):
        _add_instance(ba, reconstruction, inst_id, inst, config, lambda s: False, lambda s: True, True)

    triples = []
    for shot_id, shot in _items(reconstruction.shots):
        if up_vector is not None:
            ba.add_absolute_up_vector(shot_id, up_vector, 1e-3)
        triples.extend((shot_id, lm.id, obs) for lm, obs in _shot_observations(shot))
    added = _add_observations(ba, triples)

    if config["bundle_use_gcp"] and gcp:
        add_gcp_to_bundle(ba, reconstruction, gcp, config, len(reconstruction.rig_instances) + added)
    if config["bundle_compensate_gps_bias"]:
        for cam_id in reconstruction.cameras:
            b = _bias_values(reconstruction.biases[cam_id])
            ba.set_camera_bias(cam_id, b[:3], b[3:6], b[6])

    _configure(ba, config)
    ba.set_max_num_iterations(config["bundle_max_iterations"])
    ba.set_linear_solver_type("SPARSE_SCHUR")
    t1 = time.perf_counter()
    ba.run()
    t2 = time.perf_counter()
    bundle_to_map(ba, reconstruction, not fix_cameras)
    t3 = time.perf_counter()
    report = _report(ba, t0, t1, t2, t3)
    report["num_images"] = len(reconstruction.shots)
    report["num_points"] = len(reconstruction.points)
    report["num_reprojections"] = added
    return report


def bundle_to_map(ba: _bundle.BundleAdjuster, reconstruction, update_cameras: bool) -> None:
    """BAHelpers::BundleToMap (ba_helpers.cc:765-819): cameras, biases, rig instances, rig cameras, points and their
    reprojection errors; non-finite results raise RuntimeError."""
    pb, res = ba.results()
    cam_ids, inst_ids, rc_ids, _ = ba._order
    if update_cameras:
        off = pb.cam_off
        for i, cid in enumerate(cam_ids):
            cam = reconstruction.cameras[cid]
            vals = res["cam_params"][off[i]:off[i + 1]]
            if hasattr(cam, "set_parameter_value"):
                for name, v in zip(cam.get_parameters_types(), vals):
                    cam.set_parameter_value(name, float(v))
            else:
                cam.set_parameters_values(vals)
    biases = getattr(reconstruction, "biases", None)
    if biases is not None:
        for cid in list(biases):
            if cid not in ba._bias:
                continue
            b = ba.get_camera_bias(cid)
            if not np.all(np.isfinite(b)):
                raise RuntimeError("Bias %s has either NaN or INF values." % cid)
            if isinstance(biases[cid], np.ndarray):
                biases[cid] = b
            else:
                biases[cid].rotation, biases[cid].translation, biases[cid].scale = b[:3], b[3:6], float(b[6])
    for i, iid in enumerate(inst_ids):
        if iid in reconstruction.rig_instances:
            _write_pose(reconstruction.rig_instances[iid], "pose", res["inst"][i], "Rig Instance %s" % iid)
    for i, rid in enumerate(rc_ids):
        if rid in reconstruction.rig_cameras:
            _write_pose(reconstruction.rig_cameras[rid], "pose", res["rigcam"][i], "Rig Camera %s" % rid)
    _points_to_map(ba, reconstruction, [p for p in ba._pt_ids if p in reconstruction.points], True)


def _points_to_map(ba, reconstruction, point_ids: Sequence[str], check: bool) -> None:
    errors = ba._pt_errors or {}
    for pid in point_ids:
        i = ba._pt_index[pid]
        x = np.asarray(ba._pt_pos[i])
        if check and not np.all(np.isfinite(x)):
            raise RuntimeError("Point %s has either NaN or INF values." % pid)
        lm = reconstruction.points[pid]
        lm.coordinates = x
        lm.reprojection_errors = dict(errors.get(i, {}))


def bundle_shot_poses(reconstruction, shot_ids: Set[str], camera_priors: Dict[str, Any],
                      rig_camera_priors: Dict[str, Any], config: Dict[str, Any]) -> Dict[str, Any]:
    """opensfm.reconstruction.bundle_shot_poses (reconstruction.py:89-104) = BAHelpers::BundleShotPoses: cameras,
    rig cameras and points fixed; instances holding a shot outside `shot_ids` fixed; 10 iterations."""
    t0 = time.perf_counter()
    shot_ids = set(shot_ids)
    ba = _bundle.BundleAdjuster()
    instance_ids = []
    for sid in shot_ids:
        iid = reconstruction.shots[sid].rig_instance_id
        if iid not in instance_ids:
            instance_ids.append(iid)
    rc_ids, cam_ids = [], []
    for iid in instance_ids:
        for shot_id, rc_id in _instance_shots(reconstruction.rig_instances[iid]).items():
            if rc_id not in rc_ids:
                rc_ids.append(rc_id)
            cid = reconstruction.shots[shot_id].camera.id
            if cid not in cam_ids:
                cam_ids.append(cid)
    for rc_id in rc_ids:
        ba.add_rig_camera(rc_id, reconstruction.rig_cameras[rc_id].pose, rig_camera_priors[rc_id].pose, True)
    for cid in cam_ids:
        ba.add_camera(cid, reconstruction.cameras[cid], camera_priors[cid], True)
    triples = []
    seen = {}
    for sid in shot_ids:
        for lm, obs in _shot_observations(reconstruction.shots[sid]):
            seen[lm.id] = lm
            triples.append((sid, lm.id, obs))
    ba.add_points_bulk(list(seen), np.array([lm.coordinates for lm in seen.values()], dtype=np.float64).reshape(-1, 3), True)
    for iid in instance_ids:
        _add_instance(ba, reconstruction, iid, reconstruction.rig_instances[iid], config,
                      lambda s: s not in shot_ids, lambda s: True, False)
    _add_observations(ba, triples)
    _configure(ba, config)
    ba.set_max_num_iterations(10)
    ba.set_linear_solver_type("DENSE_QR")
    t1 = time.perf_counter()
    ba.run()
    t2 = time.perf_counter()
    _, res = ba.results()
    for i, iid in enumerate(ba._order[1]):
        _write_pose(reconstruction.rig_instances[iid], "pose", res["inst"][i], "Rig Instance %s" % iid)
    t3 = time.perf_counter()
    return _report(ba, t0, t1, t2, t3)


def bundle_local(reconstruction, camera_priors: Dict[str, Any], rig_camera_priors: Dict[str, Any],
                 gcp: Optional[List[Any]], central_shot_id: str, config: Dict[str, Any]) -> Tuple[List[str], Dict[str, Any]]:
    """opensfm.reconstruction.bundle_local (reconstruction.py:107-126) = BAHelpers::BundleLocal: cameras and rig
    cameras fixed, interior instances free, instances with a boundary shot fixed, points of the interior free,
    10 iterations."""
    t0 = time.perf_counter()
    gcp = gcp if gcp is not None else []
    interior, boundary = shot_neighborhood_ids(reconstruction, central_shot_id, config["local_bundle_radius"],
                                               config["local_bundle_min_common_points"], config["local_bundle_max_shots"])
    ba = _bundle.BundleAdjuster()
    for cam_id, cam in _items(reconstruction.cameras):
        ba.add_camera(cam_id, cam, camera_priors[cam_id], True)
    both = list(interior) + [s for s in boundary if s not in interior]
    rc_ids, inst_ids = [], []
    for sid in both:
        shot = reconstruction.shots[sid]
        if shot.rig_camera_id not in rc_ids:
            rc_ids.append(shot.rig_camera_id)
        if shot.rig_instance_id not in inst_ids:
            inst_ids.append(shot.rig_instance_id)
    for rc_id in rc_ids:
        ba.add_rig_camera(rc_id, reconstruction.rig_cameras[rc_id].pose, rig_camera_priors[rc_id].pose, True)
    for iid in inst_ids:
        _add_instance(ba, reconstruction, iid, reconstruction.rig_instances[iid], config,
                      lambda s: s in boundary, lambda s: s not in boundary, False)
    points: Dict[str, Any] = {}
    triples = []
    for sid in interior:
        for lm, obs in _shot_observations(reconstruction.shots[sid]):
            points.setdefault(lm.id, lm)
            triples.append((sid, lm.id, obs))
    for sid in boundary:
        for lm, obs in _shot_observations(reconstruction.shots[sid]):
            if lm.id in points:
                triples.append((sid, lm.id, obs))
    pt_ids = list(points)
    ba.add_points_bulk(pt_ids, np.array([lm.coordinates for lm in points.values()], dtype=np.float64).reshape(-1, 3), False)
    added = _add_observations(ba, triples)
    if config["bundle_use_gcp"] and gcp:
        add_gcp_to_bundle(ba, reconstruction, gcp, config, len(inst_ids) + added)
    _configure(ba, config)
    ba.set_max_num_iterations(10)
    ba.set_linear_solver_type("DENSE_SCHUR")
    t1 = time.perf_counter()
    ba.run()
    t2 = time.perf_counter()
    _, res = ba.results()
    for i, iid in enumerate(ba._order[1]):
        _write_pose(reconstruction.rig_instances[iid], "pose", res["inst"][i], "Rig Instance %s" % iid)
    _points_to_map(ba, reconstruction, pt_ids, False)
    t3 = time.perf_counter()
    report = _report(ba, t0, t1, t2, t3)
    report["num_images"] = len(interior)
    report["num_interior_images"] = len(interior)
    report["num_boundary_images"] = len(boundary)
    report["num_other_images"] = len(reconstruction.shots) - len(interior) - len(boundary)
    report["num_points"] = len(pt_ids)
    report["num_reprojections"] = added
    return pt_ids, report


# ---------------------------------------------------------------------------------------------------------------
# outlier removal (reconstruction.py:1227-1289)
# ---------------------------------------------------------------------------------------------------------------
def get_actual_threshold(config: Dict[str, Any], points) -> float:
    filter_type = config["bundle_outlier_filtering_type"]
    if filter_type == "FIXED":
        return config["bundle_outlier_fixed_threshold"]
    if filter_type == "AUTO":
        all_errors = [e for lm in points.values() for e in lm.reprojection_errors.values()]
        robust_mean = np.median(all_errors, axis=0)
        robust_std = 1.486 * np.median(np.linalg.norm(np.array(all_errors) - robust_mean, axis=1))
        return config["bundle_outlier_auto_ratio"] * float(np.linalg.norm(robust_mean + robust_std))
    return 1.0


def remove_outliers(reconstruction, config: Dict[str, Any], points=None) -> int:
    """Remove observations whose reprojection error exceeds the threshold, then landmarks left with < 2
    observations.  The errors are the ones the last bundle wrote (`Landmark.reprojection_errors`)."""
    if points is None:
        points = reconstruction.points
    threshold_sqr = get_actual_threshold(config, reconstruction.points) ** 2
    outliers = []
    for point_id in points:
        for shot_id, error in reconstruction.points[point_id].reprojection_errors.items():
            if error[0] ** 2 + error[1] ** 2 > threshold_sqr:
                outliers.append((point_id, shot_id))
    track_ids = set()
    for track, shot_id in outliers:
        reconstruction.map.remove_observation(shot_id, track)
        track_ids.add(track)
    for track in track_ids:
        if track in reconstruction.points:
            lm = reconstruction.points[track]
            if lm.number_of_observations() < 2:
                reconstruction.map.remove_landmark(lm)
    logger.info("Removed outliers: {}".format(len(outliers)))
    return len(outliers)


# ---------------------------------------------------------------------------------------------------------------
# image pairs for the bootstrap (reconstruction.py:193-244, 377-412, 1668-1709)
# ---------------------------------------------------------------------------------------------------------------
def pairwise_reconstructability(common_tracks: int, rotation_inliers: int) -> float:
    """Likeliness of an image pair giving a good initial reconstruction: the outliers of the rotation-only model if
    they are at least 30 % of the common tracks, else 0."""
    outliers = common_tracks - rotation_inliers
    outlier_ratio = float(outliers) / common_tracks
    if outlier_ratio >= 0.3:
        return outliers
    return 0


def two_view_reconstruction_rotation_only(p1: np.ndarray, p2: np.ndarray, camera1, camera2,
                                          threshold: float) -> Tuple[np.ndarray, np.ndarray]:
    """(angle-axis of R^T, chord inlier rows) of the rotation-only RANSAC of one pair, R b2 ~ b1."""
    import cv2

    b1 = camera1.pixel_bearing_many(p1)
    b2 = camera2.pixel_bearing_many(p2)
    res = _rr.ransac_pairs_lists([b1], [b2], threshold)
    R = res.rotations()[0]
    return cv2.Rodrigues(R.T)[0].ravel(), res.inliers(0)


def _ranked_by_argsort(keys: List[Tuple[Any, Any]], scores: List[int]) -> List[Tuple[Any, Any]]:
    """compute_image_pairs' order: non-zero scores, np.argsort(-score) (numpy's default, unstable sort)."""
    pairs = [k for k, r in zip(keys, scores) if r > 0]
    score = [r for r in scores if r > 0]
    order = np.argsort(-np.array(score))
    return [pairs[o] for o in order]


def compute_image_pairs(track_dict: Dict[Tuple[str, str], Any], data) -> List[Tuple[str, str]]:
    """All matched image pairs sorted by reconstructability.  track_dict: {(im1, im2): (tracks, p1, p2)} as
    tracking.all_common_tracks_with_features returns; bearings from the cameras' own pixel_bearing_many."""
    cameras = data.load_camera_models()
    threshold = 4 * data.config["five_point_algo_threshold"]
    keys, b1s, b2s = [], [], []
    for (im1, im2), (_, p1, p2) in track_dict.items():
        camera1 = cameras[data.load_exif(im1)["camera"]]
        camera2 = cameras[data.load_exif(im2)["camera"]]
        keys.append((im1, im2))
        b1s.append(camera1.pixel_bearing_many(p1))
        b2s.append(camera2.pixel_bearing_many(p2))
    if not keys:
        return []
    res = _rr.ransac_pairs_lists(b1s, b2s, threshold)
    return _ranked_by_argsort(keys, res.scores())


def _get_common_feature_arrays(tracks_manager, im1: Any, im2: Any) -> Tuple[np.ndarray, np.ndarray]:
    """Points of im1 and im2 in their common tracks: from the arrays of this engine's TracksManager, else from
    get_all_common_observations."""
    if hasattr(tracks_manager, "_pair_rows"):
        r1, r2 = tracks_manager._pair_rows(im1, im2)
        xy = tracks_manager._points()[0]
        return xy[r1], xy[r2]
    obs = tracks_manager.get_all_common_observations(im1, im2)
    return np.array([o1.point for _, o1, _ in obs]), np.array([o2.point for _, _, o2 in obs])


def compute_image_pairs_sequential(data, tracks_manager, min_common: int = 50) -> List[Tuple[str, str]]:
    """Image pairs with at least min_common common tracks sorted by reconstructability, in the reference's
    connectivity order and with its stable sort; all pairs go to the device in one batch."""
    cameras = data.load_camera_models()
    threshold = 4 * data.config["five_point_algo_threshold"]
    keys, b1s, b2s = [], [], []
    for (im1, im2), size in tracks_manager.get_all_pairs_connectivity().items():
        if size < min_common:
            continue
        features1, features2 = _get_common_feature_arrays(tracks_manager, im1, im2)
        keys.append((im1, im2))
        b1s.append(cameras[data.load_exif(im1)["camera"]].pixel_bearing_many(features1))
        b2s.append(cameras[data.load_exif(im2)["camera"]].pixel_bearing_many(features2))
    if not keys:
        return []
    res = _rr.ransac_pairs_lists(b1s, b2s, threshold)
    results = [(im1, im2, r) for (im1, im2), r in zip(keys, res.scores()) if r > 0]
    results.sort(key=lambda x: x[2], reverse=True)
    return [(im1, im2) for im1, im2, _ in results]


def compute_image_pairs_from_tracks(tracks_manager, cameras_by_image: Dict[Any, Any], config: Dict[str, Any],
                                    min_common: int = 50) -> List[Tuple[Any, Any]]:
    """compute_image_pairs(tracking.all_common_tracks_with_features(tracks_manager, min_common), data) for this
    engine's TracksManager, without the per-pair lists: pixel_bearing_many runs once per image over that image's
    observations, and the rows come from the device's common-track lists.  cameras_by_image: {image: camera}."""
    pa, pb, ps, ca, cb = tracks_manager._common_arrays()
    kept = np.nonzero(np.diff(ps) >= min_common)[0]
    if not len(kept):
        return []
    lens = np.diff(ps)[kept]
    pair_start = np.zeros(len(kept) + 1, dtype=np.int64)
    np.cumsum(lens, out=pair_start[1:])
    src = np.repeat(ps[kept] - pair_start[:-1], lens) + np.arange(pair_start[-1], dtype=np.int64)
    row_a, row_b = ca[src], cb[src]

    order, start = tracks_manager._shot_order()
    xy = tracks_manager._points()[0]
    bearings = np.zeros((len(xy), 3), dtype=np.float64)
    images = tracks_manager.images
    for i in np.union1d(pa[kept], pb[kept]).tolist():
        rows = order[start[i]:start[i + 1]]
        bearings[rows] = cameras_by_image[images[i]].pixel_bearing_many(xy[rows])
    res = _rr.ransac_pairs(bearings, pair_start, row_a, row_b, 4 * config["five_point_algo_threshold"])
    keys = [(images[a], images[b]) for a, b in zip(pa[kept].tolist(), pb[kept].tolist())]
    return _ranked_by_argsort(keys, res.scores())


# ---------------------------------------------------------------------------------------------------------------
# resection (reconstruction.py:247-285, 677-762; reconstruction_helpers.py:129-185; rig.py:39-52)
# ---------------------------------------------------------------------------------------------------------------
MAXIMUM_ALTITUDE = 1e4   # opensfm.exif.maximum_altitude
RESECTION_MIN_ROWS = 5   # resect rejects a candidate with fewer common points before RANSAC

_last_resect_times: Dict[str, float] = {}


def rig_assignments_per_image(rig_assignments: Dict[str, List[Tuple[str, str]]]) -> Dict[str, Tuple[str, str, List[str]]]:
    """{image: (instance id, rig camera id, the instance's images)} of {instance id: [(image, rig camera id)]}."""
    out = {}
    for instance_id, instance in rig_assignments.items():
        instance_shots = [s[0] for s in instance]
        for shot_id, rig_camera_id in instance:
            out[shot_id] = (f"{instance_id}", rig_camera_id, instance_shots)
    return out


def exif_to_metadata(exif: Dict[str, Any], use_altitude: bool, reference) -> ShotMeasurements:
    """Shot metadata from the EXIF dict: GPS position (topocentric, through `reference.to_topocentric`) and accuracy,
    OPK angles and accuracy, orientation, gravity down, compass angle and accuracy, capture time, sequence key."""
    metadata = ShotMeasurements()
    gps = exif.get("gps")
    if gps and "latitude" in gps and "longitude" in gps:
        lat, lon = gps["latitude"], gps["longitude"]
        alt = min([MAXIMUM_ALTITUDE, gps.get("altitude", 2.0)]) if use_altitude else 2.0
        x, y, z = reference.to_topocentric(lat, lon, alt)
        metadata.gps_position.value = np.array([x, y, z])
        metadata.gps_accuracy.value = gps.get("dop", 15.0)
        if metadata.gps_accuracy.value == 0.0:
            metadata.gps_accuracy.value = 15.0
    opk = exif.get("opk")
    if opk and "omega" in opk and "phi" in opk and "kappa" in opk:
        metadata.opk_angles.value = np.array([opk["omega"], opk["phi"], opk["kappa"]])
        metadata.opk_accuracy.value = opk.get("accuracy", 1.0)
    metadata.orientation.value = exif.get("orientation", 1)
    if "accelerometer" in exif:
        logger.warning("'accelerometer' EXIF tag is deprecated in favor of 'gravity_down', which expresses the gravity "
                       "down direction in the image coordinate frame.")
    if "gravity_down" in exif:
        metadata.gravity_down.value = exif["gravity_down"]
    if "compass" in exif:
        metadata.compass_angle.value = exif["compass"]["angle"]
        if exif["compass"].get("accuracy") is not None:
            metadata.compass_accuracy.value = exif["compass"]["accuracy"]
    if "capture_time" in exif:
        metadata.capture_time.value = exif["capture_time"]
    if "skey" in exif:
        metadata.sequence_key.value = exif["skey"]
    return metadata


def get_image_metadata(data, image: str) -> ShotMeasurements:
    return exif_to_metadata(data.load_exif(image), data.config["use_altitude_tag"], data.load_reference())


def add_shot(data, reconstruction, rig_assignments: Dict[str, Tuple[str, str, List[str]]], shot_id: str,
             pose: T.Pose) -> Set[str]:
    """Adds a shot with the given pose; a shot of a rig brings its whole rig instance, placed so that the shot has
    that pose.  Returns the ids of the shots added."""
    if shot_id not in rig_assignments:
        shot = reconstruction.create_shot(shot_id, data.load_exif(shot_id)["camera"], pose)
        shot.metadata = get_image_metadata(data, shot_id)
        return {shot_id}
    instance_id, _, instance_shots = rig_assignments[shot_id]
    rig_instance = reconstruction.add_rig_instance(RigInstance(instance_id))
    for shot in instance_shots:
        _, rig_camera_id, _ = rig_assignments[shot]
        created = reconstruction.create_shot(shot, data.load_exif(shot)["camera"], T.Pose(), rig_camera_id,
                                             instance_id)
        created.metadata = get_image_metadata(data, shot)
    rig_instance.update_instance_pose_with_shot(shot_id, pose)
    return set(instance_shots)


def _point_tracks(tracks_manager, reconstruction) -> Tuple[np.ndarray, np.ndarray]:
    """(per track: is a point of the reconstruction, its coordinates); a point's id is its track id."""
    T_ = tracks_manager.num_tracks()
    is_point = np.zeros(T_, dtype=bool)
    coords = np.zeros((T_, 3), dtype=np.float64)
    for point_id, lm in reconstruction.points.items():
        t = int(point_id) if isinstance(point_id, str) and point_id.isdigit() else -1
        if 0 <= t < T_ and str(t) == point_id:
            is_point[t] = True
            coords[t] = lm.coordinates
    return is_point, coords


def reconstructed_points_for_images(tracks_manager, reconstruction, images) -> List[Tuple[Any, int]]:
    """(image, reconstructed points it sees) of the images not in the reconstruction, by decreasing count; ties in
    the order of tracks_manager.images (the reference's follow a set's iteration order)."""
    images = set(images)
    is_point = _point_tracks(tracks_manager, reconstruction)[0]
    seen = is_point[tracks_manager.obs_track]
    counts = np.bincount(tracks_manager.obs_image[seen], minlength=len(tracks_manager.images))
    has_obs = np.diff(tracks_manager._shot_order()[1]) > 0
    keep = [i for i, im in enumerate(tracks_manager.images)
            if im in images and im not in reconstruction.shots and has_obs[i]]
    keep.sort(key=lambda i: -counts[i])
    return [(tracks_manager.images[i], int(counts[i])) for i in keep]


def resect_candidates(data, tracks_manager, reconstruction, candidates, threshold: float, min_inliers: int
                      ) -> Tuple[Optional[Any], Set[str], Optional[Dict[str, Any]], List[Dict[str, Any]]]:
    """Resects every candidate image (ids, or (id, count) pairs as reconstructed_points_for_images returns) in one
    launch and adds the first one, in candidate order, with at least min_inliers chord inliers, exactly as
    `resect` called on the candidates one after another would: a failed resection changes nothing.  Returns (that
    image or None, the shots added, its report, the report of every candidate)."""
    t0 = time.perf_counter()
    images = [c[0] if isinstance(c, tuple) else c for c in candidates]
    rig_assignments = rig_assignments_per_image(data.load_rig_assignments())
    is_point, coords = _point_tracks(tracks_manager, reconstruction)
    order, start = tracks_manager._shot_order()
    xy = tracks_manager._points()[0]
    index = {im: i for i, im in enumerate(tracks_manager.images)}
    rows_of, bearings_of = [], []
    for im in images:
        i = index[im]
        rows = order[start[i]:start[i + 1]]
        rows = rows[is_point[tracks_manager.obs_track[rows]]]
        camera = reconstruction.cameras[data.load_exif(im)["camera"]]
        rows_of.append(rows)
        bearings_of.append(camera.pixel_bearing_many(xy[rows]) if len(rows) else np.zeros((0, 3)))
    t1 = time.perf_counter()
    launched = [k for k, r in enumerate(rows_of) if len(r) >= RESECTION_MIN_ROWS]
    bs = [bearings_of[k] for k in launched]
    Xs = [coords[tracks_manager.obs_track[rows_of[k]]] for k in launched]
    packed = _rs.pack_lists(bs, Xs)
    t2 = time.perf_counter()
    res = _rs.ransac_shots(*packed, threshold) if launched else None
    t3 = time.perf_counter()

    reports: List[Dict[str, Any]] = [{"num_common_points": len(r)} for r in rows_of]
    chosen = None
    poses = res.poses() if res is not None else None
    for s, k in enumerate(launched):
        reports[k]["num_inliers"] = int(res.chord_inliers[s])
        if chosen is None and res.chord_inliers[s] >= min_inliers:
            chosen = (s, k)
    new_shots: Set[str] = set()
    if chosen is not None:
        s, k = chosen
        shot_id, rows = images[k], rows_of[k]
        Tp = poses[s]
        R = Tp[:, :3].T
        pose = T.Pose()
        pose.set_rotation_matrix(R)
        pose.translation = -R.dot(Tp[:, 3])
        assert shot_id not in reconstruction.shots
        new_shots = add_shot(data, reconstruction, rig_assignments, shot_id, pose)
        if shot_id in rig_assignments:
            triangulate_shot_features(tracks_manager, reconstruction, new_shots, data.config)
        ids = tracks_manager._track_ids()
        for r in rows[res.inliers(s)].tolist():
            reconstruction.add_observation(shot_id, ids[tracks_manager.obs_track[r]], tracks_manager._observation(r))
        reports[k]["shots"] = list(new_shots)
    t4 = time.perf_counter()
    _last_resect_times.clear()
    _last_resect_times.update(bearings=t1 - t0, packing=t2 - t1, device_call=t3 - t2, map_writes=t4 - t3,
                              device_ms=_rs.last_device_ms() if launched else 0.0)
    if chosen is None:
        return None, set(), None, reports
    return images[chosen[1]], new_shots, reports[chosen[1]], reports


def last_resect_times() -> Dict[str, float]:
    """Host seconds of the last resect_candidates / resect call, by part (bearings, packing, device_call,
    map_writes), and the kernel's device milliseconds (device_ms)."""
    return dict(_last_resect_times)


def resect(data, tracks_manager, reconstruction, shot_id: str, threshold: float, min_inliers: int
           ) -> Tuple[bool, Set[str], Dict[str, Any]]:
    """Tries resecting and adding one shot: (success, shots added, report), the reference's signature and report."""
    image, new_shots, _, reports = resect_candidates(data, tracks_manager, reconstruction, [shot_id], threshold,
                                                     min_inliers)
    return image is not None, new_shots, reports[0]
