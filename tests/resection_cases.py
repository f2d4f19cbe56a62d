"""Inputs for the resection tests: shots of synthetic cube scenes with injected outliers, and a small incremental
reconstruction (tracks manager, map, dataset and camera stand-ins) that resect and resect_candidates run on."""
import copy
from typing import List, Tuple

import numpy as np

from opensfm_b200 import map_types as M
from opensfm_b200 import synthetic as syn
from opensfm_b200 import tracking
from opensfm_b200 import types as T


def unit(v: np.ndarray) -> np.ndarray:
    return v / np.sqrt((v * v).sum(axis=1))[:, None]


def cube_shots(num_cameras: int, num_points: int, seed: int, sizes, outlier_ratios=(0.0, 0.1, 0.2, 0.3, 0.5, 0.65),
               count: int = 0, noise: float = 2e-4) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """(bearing list, point list) of shots of a cube scene: the rows of a camera's visible points subsampled to the
    shot's size, bearings from the true pose with `noise`, then a fraction of them replaced by random directions in
    front of the camera."""
    sc = syn.cube_scene(num_cameras, num_points, seed=seed, with_descriptors=False)
    rng = np.random.RandomState(seed + 1)
    count = count or max(len(sizes), len(outlier_ratios)) * num_cameras
    bs, Xs = [], []
    for k in range(count):
        s = k % num_cameras
        n = min(sizes[k % len(sizes)], num_points)
        X = sc.points[np.sort(rng.choice(num_points, n, replace=False))]
        b = unit(unit((X - sc.origins[s]) @ sc.R_wc[s].T) + noise * rng.randn(n, 3))
        bad = rng.rand(n) < outlier_ratios[k % len(outlier_ratios)]
        b[bad] = unit(np.column_stack([rng.uniform(-0.6, 0.6, (int(bad.sum()), 2)), np.ones(int(bad.sum()))]))
        bs.append(b)
        Xs.append(X)
    return bs, Xs


THRESHOLD = 0.004          # resection_threshold, OpenSfM's default


def batch_shots() -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """The GPU comparison batch: 204 shots of a cube scene with 0 .. 65 % outliers, of 5, 6, 12, 50, 200, 600, 1025
    and 3000 rows."""
    return cube_shots(36, 3000, 7, sizes=(5, 50, 600, 12, 200, 1025, 50, 6, 600, 200, 3000, 12), count=204)


def digest(bs, Xs) -> str:
    """sha256 of the batch's inputs, so that a fixture made from them is checked to belong to them."""
    import hashlib

    h = hashlib.sha256()
    for b, X in zip(bs, Xs):
        h.update(np.ascontiguousarray(b, dtype=np.float64).tobytes())
        h.update(np.ascontiguousarray(X, dtype=np.float64).tobytes())
    return h.hexdigest()


class PinholeCamera:
    id = "cam"

    def pixel_bearing_many(self, p) -> np.ndarray:
        p = np.asarray(p, dtype=np.float64).reshape(-1, 2)
        return unit(np.column_stack([p[:, 0], p[:, 1], np.ones(len(p))]))


class Reference:
    def to_topocentric(self, lat, lon, alt):
        return lat, lon, alt


class Dataset:
    def __init__(self, rigs=None):
        self.config = {"use_altitude_tag": True, "triangulation_type": "FULL", "triangulation_threshold": 0.006,
                       "triangulation_min_ray_angle": 1.0, "triangulation_min_depth": 0.001,
                       "triangulation_refinement_iterations": 10, "resection_threshold": 0.004,
                       "resection_min_inliers": 10}
        self.rigs = rigs or {}

    def load_exif(self, image):
        return {"camera": "cam"}

    def load_rig_assignments(self):
        return self.rigs

    def load_reference(self):
        return Reference()


def incremental_scene(num_cameras: int, num_points: int, seed: int, outliers: float = 0.2, max_obs: int = 10,
                      reconstructed=None):
    """(tracks manager, reconstruction, scene): a thinned cube scene whose features are pinhole coordinates of the
    true points, `outliers` of the observations of the shots not reconstructed moved to random positions, linked
    into tracks on the GPU from the true matches.  The shots in `reconstructed` (default: the first half) are in the
    map at their true poses; every track seen twice among them is a point at its true position, with its
    observations in them."""
    sc = syn.cube_scene(num_cameras, num_points, seed=seed, with_descriptors=False, max_obs_per_point=max_obs)
    rng = np.random.RandomState(seed)
    reconstructed = sorted(range(num_cameras // 2) if reconstructed is None else reconstructed)
    images = ["im%03d" % s for s in range(num_cameras)]
    feats, point_of = {}, {}
    for s in range(num_cameras):
        pts = np.sort(sc.obs_point[sc.obs_shot == s])
        pc = (sc.points[pts] - sc.origins[s]) @ sc.R_wc[s].T
        xy = pc[:, :2] / pc[:, 2:3]
        if s not in reconstructed:
            moved = rng.rand(len(xy)) < outliers
            xy[moved] = rng.uniform(-0.5, 0.5, (int(moved.sum()), 2))
        feats[images[s]] = np.column_stack([xy, np.full(len(xy), 0.004)])
        point_of[images[s]] = pts
    matches = {}
    for i in range(num_cameras):
        for j in range(i + 1, num_cameras):
            _, ki, kj = np.intersect1d(point_of[images[i]], point_of[images[j]], return_indices=True)
            if len(ki):
                matches[images[i], images[j]] = np.column_stack([ki, kj]).astype(np.int32)
    colors = {im: np.zeros((len(f), 3), dtype=np.int32) for im, f in feats.items()}
    tm = tracking.create_tracks_manager(feats, colors, {}, {}, matches, 2)
    rec = M.Reconstruction()
    rec.add_camera(PinholeCamera())
    for s in reconstructed:
        pose = T.Pose()
        pose.set_rotation_matrix(sc.R_wc[s])
        pose.set_origin(sc.origins[s])
        rec.create_shot(images[s], "cam", pose)
    ids = tm._track_ids()
    in_rec = np.isin(tm.obs_image, [tm.images.index(images[s]) for s in reconstructed])
    twice = np.bincount(tm.obs_track[in_rec], minlength=tm.num_tracks()) >= 2
    for r in np.nonzero(in_rec & twice[tm.obs_track])[0].tolist():
        t = int(tm.obs_track[r])
        im = tm.images[tm.obs_image[r]]
        if ids[t] not in rec.points:
            rec.create_point(ids[t], sc.points[point_of[im][tm.obs_feature[r]]])
        rec.add_observation(im, ids[t], tm._observation(r))
    return tm, rec, sc
def map_state(rec):
    """Everything resect writes, comparable with ==: shots with their exact poses, points, observations."""
    shots = {s: (tuple(sh.pose.rotation.tolist()), tuple(sh.pose.translation.tolist()), sh.rig_instance_id,
                 sh.rig_camera_id) for s, sh in rec.shots.items()}
    points = {p: tuple(lm.coordinates.tolist()) for p, lm in rec.points.items()}
    obs = {s: {p: tuple(o.point.tolist()) for p, o in d.items()} for s, d in rec._shot_obs.items() if d}
    return shots, points, obs


def clone(rec):
    return copy.deepcopy(rec)
