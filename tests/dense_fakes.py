"""In-memory stand-ins for the objects opensfm.dense.compute_depthmaps reads: shots with poses and perspective
cameras, a reconstruction, a pymap-like tracks manager and an UndistortedDataSet, over synthetic.textured_scene."""
import os

import numpy as np

from opensfm_b200 import synthetic as syn


class Camera:
    projection_type = "perspective"

    def __init__(self, width, height, focal):
        self.width, self.height, self.focal = width, height, focal

    def get_K_in_pixel_coordinates(self, width, height):
        f = self.focal * max(width, height)
        return np.array([[f, 0, (width - 1) / 2.0], [0, f, (height - 1) / 2.0], [0, 0, 1.0]])


class Pose:
    def __init__(self, R, t):
        self.R, self.translation = np.asarray(R, float), np.asarray(t, float)

    def get_rotation_matrix(self):
        return self.R

    def get_origin(self):
        return -self.R.T @ self.translation

    def transform(self, p):
        return self.R @ np.asarray(p, float) + self.translation


class Shot:
    def __init__(self, sid, camera, pose):
        self.id, self.camera, self.pose = sid, camera, pose


class Point:
    def __init__(self, X):
        self.coordinates = np.asarray(X, float)


class Reconstruction:
    def __init__(self, shots, points):
        self.shots, self.points = shots, points


class TracksManager:
    def __init__(self, obs):
        self.obs = obs                                   # {shot: [track ids]}

    def get_shot_ids(self):
        return list(self.obs)

    def get_shot_observations(self, shot_id):
        return {t: None for t in self.obs[shot_id]}


CONFIG = dict(depthmap_num_neighbors=10, depthmap_num_matching_views=6, depthmap_min_depth=0, depthmap_max_depth=0,
              depthmap_method="PATCH_MATCH_SAMPLE", depthmap_patch_size=7, depthmap_patchmatch_iterations=2,
              depthmap_min_patch_sd=1.0, depthmap_min_correlation_score=0.1, depthmap_same_depth_threshold=0.01,
              depthmap_min_consistent_views=2, depthmap_resolution=640, depthmap_save_debug_files=True)


class DataSet:
    def __init__(self, images, path, config=None):
        self.config = dict(CONFIG, **(config or {}))
        self.images, self.path = images, path
        self.raw, self.clean, self.pruned, self.clouds = {}, {}, {}, {}

    def load_undistorted_image(self, sid):
        return self.images[sid]

    def load_undistorted_combined_mask(self, sid):
        return None

    def undistorted_segmentation_exists(self, sid):
        return False

    def raw_depthmap_exists(self, sid):
        return sid in self.raw

    def clean_depthmap_exists(self, sid):
        return sid in self.clean

    def pruned_depthmap_exists(self, sid):
        return sid in self.pruned

    def save_raw_depthmap(self, sid, depth, plane, score, nghbr, nghbrs):
        self.raw[sid] = (np.array(depth, np.float32), np.array(plane), np.array(score), np.array(nghbr), list(nghbrs))

    def load_raw_depthmap(self, sid):
        return self.raw[sid]

    def save_clean_depthmap(self, sid, depth, plane, score):
        self.clean[sid] = (np.array(depth), np.array(plane), np.array(score))

    def load_clean_depthmap(self, sid):
        return self.clean[sid]

    def save_pruned_depthmap(self, sid, points, normals, colors, labels):
        self.pruned[sid] = tuple(np.array(a) for a in (points, normals, colors, labels))

    def load_pruned_depthmap(self, sid):
        return self.pruned[sid]

    def depthmap_file(self, sid, suffix):
        return os.path.join(self.path, "%s.%s" % (sid, suffix))

    def save_point_cloud(self, points, normals, colors, labels, filename):
        self.clouds.setdefault(filename, []).append(tuple(np.array(a) for a in (points, normals, colors, labels)))


def scene(num_cameras=5, width=96, height=72, seed=3):
    """Shots s0..s{n-1} of textured_scene sharing 400 tracks on the ground plane, and a lone shot that shares none."""
    sc = syn.textured_scene(num_cameras + 1, width, height, seed=seed, arc_degrees=48)
    rng = np.random.RandomState(seed)
    pts = np.column_stack([rng.uniform(-2, 2, 400), rng.uniform(-2, 2, 400), np.zeros(400)])
    points = {"t%d" % k: Point(p) for k, p in enumerate(pts)}
    shots, images, obs = {}, {}, {}
    for k in range(num_cameras + 1):
        sid = "s%d" % k
        shots[sid] = Shot(sid, Camera(width, height, 0.9), Pose(sc.R[k], sc.t[k]))
        images[sid] = sc.rgb[k]
        obs[sid] = list(points) if k < num_cameras else ["lone%d" % q for q in range(60)]
    return Reconstruction(shots, points), TracksManager(obs), images
