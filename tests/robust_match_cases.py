"""Inputs for the geometric verification tests and measurement: a camera for the cube scenes' distorted projection,
and the per-image descriptors and points of a cube scene."""
from typing import Dict, Tuple

import numpy as np

from opensfm_b200 import synthetic as syn

CONFIG = {"lowes_ratio": 0.8, "symmetric_matching": True, "robust_matching_min_match": 20,
          "robust_matching_threshold": 0.004, "robust_matching_calib_threshold": 0.004,
          "five_point_refine_match_iterations": 10}


class RadialCamera:
    """pixel_bearing_many of the cube scenes' camera: the inverse of synthetic.project_perspective (focal, then
    x_d = x_u (1 + k1 r^2 + k2 r^4)), by fixed-point iteration on the undistorted radius."""

    projection_type = "perspective"

    def __init__(self, k1: float, k2: float, focal: float):
        self.k1, self.k2, self.focal = k1, k2, focal

    def pixel_bearing_many(self, p) -> np.ndarray:
        d = np.asarray(p, dtype=np.float64).reshape(-1, 2) / self.focal
        u = d.copy()
        for _ in range(50):
            r2 = (u * u).sum(axis=1)
            u = d / (1.0 + r2 * (self.k1 + self.k2 * r2))[:, None]
        b = np.column_stack([u, np.ones(len(u))])
        return b / np.linalg.norm(b, axis=1)[:, None]


def cube_images(sc: syn.SyntheticScene) -> Tuple[Dict[str, np.ndarray], Dict[str, np.ndarray], Dict[str, np.ndarray],
                                                  RadialCamera]:
    """(descriptors, points, point ids) per image "im%02d" of a cube scene, and the scene's camera."""
    desc, points, ids = {}, {}, {}
    for s in range(sc.num_shots):
        sel = np.nonzero(sc.obs_shot == s)[0]
        im = "im%02d" % s
        desc[im] = sc.track_descriptors[sc.obs_point[sel]]
        points[im] = np.column_stack([sc.obs_xy[sel], sc.obs_sigma[sel]])
        ids[im] = sc.obs_point[sel]
    k1, k2, focal = (float(v) for v in sc.cam_params[0])
    return desc, points, ids, RadialCamera(k1, k2, focal)
