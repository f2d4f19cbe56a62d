"""Drop-in triangulation of tracks: the `opensfm.reconstruction` names this engine replaces.

    triangulate_shot_features(tracks_manager, reconstruction, shot_ids, config)   opensfm/reconstruction.py:1143-1183
    retriangulate(tracks_manager, reconstruction, config)                         opensfm/reconstruction.py:1186-1226

Both hand every track they would loop over to `TracksManager.triangulate` (the bulk form: arrays in, (X[T, 3],
status[T]) out), which runs TrackTriangulator.triangulate (:1032-1073) for all of them in one launch of
opensfm_b200/csrc/triangulate.cu on the tracks handle that built `tracks_manager`; there is no CPU path.  The host
part is the bearings, computed with each shot's `camera.pixel_bearing_many` once per image over that image's
observations, and the writes into the map: `create_point(track_id, X)` and `add_observation(shot_id, track_id,
observation)` for each of the track's observations in a shot of the reconstruction, as TrackHandlerTrackManager does
(:861-892).  Point ids are track ids, so the result does not depend on the order the reference's set of track ids
iterates in.

`tracks_manager` is this engine's `tracking.TracksManager`; `reconstruction` is `opensfm_b200.map_types.Reconstruction`
or anything with its names (shots with `pose` and a `camera` that has `pixel_bearing_many`, `points`, `create_point`,
`add_observation`).  Only the "FULL" triangulation type (the reference's default) is built: "ROBUST" raises, any other
value triangulates nothing, as in the reference.
"""
from __future__ import annotations

import time
from typing import Any, Dict, Iterable, Tuple

import numpy as np

STATUS_NOT_SELECTED = 0
STATUS_TOO_FEW = 1                # fewer than 2 observations in shots of the reconstruction
STATUS_BAD_ANGLE = 2              # no pair of rays at an angle in [min_ray_angle, pi - min_ray_angle]
STATUS_BAD_REPROJECTION = 3       # the midpoint fails the reprojection or the depth test
STATUS_OK = 4


def _options(config: Dict[str, Any]) -> Tuple[float, float, float, int]:
    """(threshold, min_ray_angle in radians, min_depth, iterations) from the reference's config keys."""
    return (float(config["triangulation_threshold"]), float(np.radians(config["triangulation_min_ray_angle"])),
            float(config["triangulation_min_depth"]), int(config["triangulation_refinement_iterations"]))


def _full(config: Dict[str, Any]) -> bool:
    kind = config.get("triangulation_type", "FULL")
    if kind == "ROBUST":
        raise NotImplementedError(
            "triangulation_type ROBUST is not built: the reference draws its samples from the global np.random state "
            "in the iteration order of a set of string track ids, which string hashing makes differ from run to run")
    return kind == "FULL"


def shot_rays(tracks_manager, reconstruction) -> Dict[str, np.ndarray]:
    """The per-image and per-observation inputs of TracksManager.triangulate for the shots of `reconstruction`:
    image_rt, image_origin, image_in and bearings (pixel_bearing_many once per reconstructed image)."""
    images = tracks_manager.images
    I, N = len(images), len(tracks_manager.obs_track)
    rt = np.zeros((I, 3, 3))
    origin = np.zeros((I, 3))
    image_in = np.zeros(I, dtype=np.uint8)
    bearings = np.zeros((N, 3))
    order, start = tracks_manager._shot_order()
    xy = tracks_manager._points()[0]
    shots = reconstruction.shots
    for i, im in enumerate(images):
        rows = order[start[i]:start[i + 1]]
        if not len(rows) or im not in shots:
            continue
        shot = shots[im]
        image_in[i] = 1
        rt[i] = np.asarray(shot.pose.get_rotation_matrix(), dtype=np.float64).T
        origin[i] = shot.pose.get_origin()
        bearings[rows] = shot.camera.pixel_bearing_many(xy[rows])
    return dict(image_rt=rt, image_origin=origin, image_in=image_in, bearings=bearings)


def _triangulate_into(tracks_manager, reconstruction, selected: np.ndarray, config: Dict[str, Any]) -> Dict[str, float]:
    """Triangulates the selected tracks and writes the points and their observations into the map; returns the
    host clock of each part (s) and the kernel's device time (ms)."""
    t0 = time.perf_counter()
    rays = shot_rays(tracks_manager, reconstruction)
    t1 = time.perf_counter()
    X, status = tracks_manager.triangulate(rays["image_rt"], rays["image_origin"], rays["image_in"], rays["bearings"],
                                           selected, *_options(config))
    t2 = time.perf_counter()
    ok = np.nonzero(status == STATUS_OK)[0]
    if len(ok):
        obs_track, obs_image = tracks_manager.obs_track, tracks_manager.obs_image
        rows = np.nonzero(rays["image_in"][obs_image].astype(bool) & (status[obs_track] == STATUS_OK))[0]
        groups = np.split(rows, np.searchsorted(obs_track[rows], ok[1:]))
        ids = tracks_manager._track_ids()
        images = tracks_manager.images
        for t, track_rows in zip(ok.tolist(), groups):
            track_id = ids[t]
            reconstruction.create_point(track_id, X[t].tolist())
            for r in track_rows.tolist():
                reconstruction.add_observation(images[obs_image[r]], track_id, tracks_manager._observation(r))
    t3 = time.perf_counter()
    return {"bearings": t1 - t0, "device_call": t2 - t1, "write": t3 - t2,
            "device_ms": tracks_manager.triangulate_device_ms}


def _seen_in(tracks_manager, image_mask: np.ndarray) -> np.ndarray:
    """Per track: observed in an image of the mask."""
    selected = np.zeros(tracks_manager.num_tracks(), dtype=np.uint8)
    selected[tracks_manager.obs_track[image_mask[tracks_manager.obs_image]]] = 1
    return selected


def triangulate_shot_features(tracks_manager, reconstruction, shot_ids: Iterable[Any], config: Dict[str, Any]) -> None:
    """Reconstruct as many tracks seen in shot_ids as possible: every track observed in one of them that is not yet a
    point of the reconstruction (opensfm/reconstruction.py:1143-1183)."""
    if not _full(config):
        return
    index = {im: i for i, im in enumerate(tracks_manager.images)}
    mask = np.zeros(len(tracks_manager.images), dtype=bool)
    for s in shot_ids:
        if s in index:
            mask[index[s]] = True
    selected = _seen_in(tracks_manager, mask)
    T = tracks_manager.num_tracks()
    for point_id in reconstruction.points:
        t = int(point_id) if isinstance(point_id, str) and point_id.isdigit() else -1
        if 0 <= t < T and str(t) == point_id:
            selected[t] = 0
    if selected.any():
        _triangulate_into(tracks_manager, reconstruction, selected, config)


def retriangulate(tracks_manager, reconstruction, config: Dict[str, Any]) -> Dict[str, Any]:
    """Retriangulate all points: clear them and triangulate every track seen in a shot of the reconstruction
    (opensfm/reconstruction.py:1186-1226).  Returns the reference's report (num_points_before, num_points_after,
    wall_time) and this engine's split of the wall time (wall_times: bearings, device_call, write; device_ms)."""
    t0 = time.perf_counter()
    full = _full(config)
    report: Dict[str, Any] = {"num_points_before": len(reconstruction.points)}
    reconstruction.points = {}
    if full:
        mask = np.array([im in reconstruction.shots for im in tracks_manager.images], dtype=bool)
        times = _triangulate_into(tracks_manager, reconstruction, _seen_in(tracks_manager, mask), config)
        report["wall_times"] = {k: v for k, v in times.items() if k != "device_ms"}
        report["device_ms"] = times["device_ms"]
    report["num_points_after"] = len(reconstruction.points)
    report["wall_time"] = time.perf_counter() - t0
    return report
