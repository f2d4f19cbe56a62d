"""Inputs for the relative-pose tests: image pairs of synthetic cube scenes (some with every point on one plane) with
injected outliers."""
import hashlib
from typing import List, Tuple

import numpy as np

from opensfm_b200 import synthetic as syn

THRESHOLD = 0.004          # five_point_algo_threshold, OpenSfM's default
SIZES = (5, 50, 600, 12, 200, 1025, 50, 6, 600, 200, 3000, 12, 7, 100)
OUTLIERS = (0.0, 0.1, 0.2, 0.3, 0.5, 0.65)


def unit(v: np.ndarray) -> np.ndarray:
    return v / np.sqrt((v * v).sum(axis=1))[:, None]


def cube_pairs(num_cameras: int, num_points: int, seed: int, count: int, sizes=SIZES, outlier_ratios=OUTLIERS,
               noise: float = 2e-4, planar_every: int = 7) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """(first bearings, second bearings) of pairs of cameras of a cube scene: pair k joins cameras k and k + 1 + k % 3
    (mod num_cameras), its rows are `sizes[k % len(sizes)]` points of the scene (every `planar_every`-th pair: of
    the plane z = 0), bearings from the true poses with `noise`, then a fraction of the second bearings replaced by
    random directions in front of the camera."""
    sc = syn.cube_scene(num_cameras, num_points, seed=seed, with_descriptors=False)
    rng = np.random.RandomState(seed + 1)
    b1s, b2s = [], []
    for k in range(count):
        s, o = k % num_cameras, (k + 1 + k % 3) % num_cameras
        n = min(sizes[k % len(sizes)], num_points)
        X = sc.points[np.sort(rng.choice(num_points, n, replace=False))]
        if planar_every and k % planar_every == planar_every - 1:
            X = X * [1.0, 1.0, 0.0]
        b1 = unit(unit((X - sc.origins[s]) @ sc.R_wc[s].T) + noise * rng.randn(n, 3))
        b2 = unit(unit((X - sc.origins[o]) @ sc.R_wc[o].T) + noise * rng.randn(n, 3))
        bad = rng.rand(n) < outlier_ratios[k % len(outlier_ratios)]
        b2[bad] = unit(np.column_stack([rng.uniform(-0.6, 0.6, (int(bad.sum()), 2)), np.ones(int(bad.sum()))]))
        b1s.append(b1)
        b2s.append(b2)
    return b1s, b2s


def batch_pairs() -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """The GPU comparison batch: 196 pairs of 5 to 3000 rows with 0 .. 65 % outliers, every seventh planar."""
    return cube_pairs(24, 3000, 5, count=196)


def digest(b1s, b2s) -> str:
    """sha256 of the batch's inputs, so that a fixture made from them is checked to belong to them."""
    h = hashlib.sha256()
    for a, b in zip(b1s, b2s):
        h.update(np.ascontiguousarray(a, dtype=np.float64).tobytes())
        h.update(np.ascontiguousarray(b, dtype=np.float64).tobytes())
    return h.hexdigest()
