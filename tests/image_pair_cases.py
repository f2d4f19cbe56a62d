"""Inputs for the rotation-only RANSAC tests: the known-answer case of OpenSfM's test_robust (30 % outliers), image
pairs of synthetic cube scenes with injected outliers, and the small camera and dataset objects compute_image_pairs
reads."""
from typing import Dict, List, Tuple

import numpy as np

from opensfm_b200 import synthetic as syn


def unit(v: np.ndarray) -> np.ndarray:
    return v / np.sqrt((v * v).sum(axis=1))[:, None]


def robust_case(seed: int, n: int = 400):
    """(b1, b2, true model M with b2 ~ M b1, threshold) like test_outliers_relative_rotation_ransac: bearings in a
    camera's field of view, an arbitrary rotation, 1e-3 uniform noise on both sides and 30 % of the rows pushed by
    0.1 .. 1 per coordinate."""
    rng = np.random.RandomState(seed)
    f1 = unit(np.column_stack([rng.uniform(-0.6, 0.6, (n, 2)), np.ones(n)]))
    vx = rng.rand(3)
    vx /= np.linalg.norm(vx)
    vy = np.array([-vx[1], vx[0], 0.0])
    vy /= np.linalg.norm(vy)
    rotation = np.array([vx, vy, np.cross(vx, vy)])
    scale = 1e-3
    points = np.hstack([f1, f1 @ rotation.T]) + rng.rand(n, 6) * scale
    for i in rng.permutation(n)[:int(0.3 * n)]:
        points[i] += np.where(rng.randint(2, size=6) > 0, 1.0, -1.0) * rng.uniform(0.1, 1.0, 6)
    return unit(points[:, :3]), unit(points[:, 3:]), rotation, float(np.sqrt(3 * scale * scale))


class PinholeCamera:
    """pixel_bearing_many of a distortion-free perspective camera with normalised coordinates."""

    def __init__(self, focal: float = 1.0):
        self.focal = focal

    def pixel_bearing_many(self, p) -> np.ndarray:
        p = np.asarray(p, dtype=np.float64).reshape(-1, 2)
        return unit(np.column_stack([p[:, 0], p[:, 1], np.full(len(p), self.focal)]))


class Dataset:
    """The three things compute_image_pairs reads from a DataSet."""

    def __init__(self, threshold: float = 0.004, camera=None):
        self.config = {"five_point_algo_threshold": threshold, "processes": 1}
        self.camera = camera or PinholeCamera()

    def load_camera_models(self):
        return {"cam": self.camera}

    def load_exif(self, image):
        return {"camera": "cam"}


def cube_pairs(num_cameras: int, num_points: int, seed: int, sizes=(600,), outlier_ratios=(0.0, 0.1, 0.3, 0.5, 0.65),
               baselines=(0.0, 1e-3, 1e-2), translational_every: int = 0, noise: float = 2e-4
               ) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """(b1 list, b2 list) of image pairs over the points and cameras of a cube scene.  For shots i < j (every pair,
    then again with the next size / outlier ratio / baseline until the cycles are used): bearings of the points in
    shot i's frame from shot i's centre, and in shot j's frame from a centre moved from shot i's towards shot j's by
    a fraction of the distance between them (the baseline; every translational_every-th pair moves all the way), with
    `noise` on both; then a fraction of the second image's bearings replaced by random directions, and the rows
    subsampled to the pair's size."""
    sc = syn.cube_scene(num_cameras, num_points, seed=seed)
    rng = np.random.RandomState(seed + 1)
    shots = [(i, j) for i in range(sc.num_shots) for j in range(i + 1, sc.num_shots)]
    count = max(len(sizes), len(outlier_ratios), len(baselines)) * len(shots)
    b1s, b2s = [], []
    for k in range(count):
        i, j = shots[k % len(shots)]
        n = min(sizes[k % len(sizes)], len(sc.points))
        X = sc.points[np.sort(rng.choice(len(sc.points), n, replace=False))]
        f = 1.0 if translational_every and k % translational_every == translational_every - 1 else baselines[k % len(baselines)]
        c1, c2 = sc.origins[i], sc.origins[i] + f * (sc.origins[j] - sc.origins[i])
        b1 = unit(unit((X - c1) @ sc.R_wc[i].T) + noise * rng.randn(n, 3))
        b2 = unit(unit((X - c2) @ sc.R_wc[j].T) + noise * rng.randn(n, 3))
        bad = rng.rand(n) < outlier_ratios[k % len(outlier_ratios)]
        b2[bad] = unit(rng.randn(int(bad.sum()), 3))
        b1s.append(b1)
        b2s.append(b2)
    return b1s, b2s


def subsample(b1: np.ndarray, b2: np.ndarray, n: int, seed: int):
    keep = np.sort(np.random.RandomState(seed).choice(len(b1), n, replace=False))
    return b1[keep], b2[keep]


def rotation_about(axis, angle: float) -> np.ndarray:
    return syn.angle_axis_to_rotation(np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis) * angle)
