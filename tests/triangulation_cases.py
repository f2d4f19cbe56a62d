"""Cameras, maps and tracks for the triangulation tests: the reference's known answers (tests/golden/
triangulation_known_answers.json) and synthetic scenes whose tracks reach every status of the triangulation."""
import json
import os
from typing import Any, Dict, List, Tuple

import numpy as np

from opensfm_b200 import map_types, synthetic
from opensfm_b200 import types as T

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIG = {"triangulation_threshold": 0.006, "triangulation_min_ray_angle": 1.0, "triangulation_min_depth": 0.001,
          "triangulation_type": "FULL", "triangulation_refinement_iterations": 10}


def known_answers() -> Dict[str, Any]:
    with open(os.path.join(HERE, "golden", "triangulation_known_answers.json")) as f:
        return json.load(f)


class SphericalCamera:
    """pixel_bearing of the spherical projection (geometry/camera_projections_functions.h SphericalProjection)."""

    def __init__(self, camera_id: str = "theta"):
        self.id = camera_id

    def pixel_bearing_many(self, p) -> np.ndarray:
        p = np.asarray(p, dtype=np.float64).reshape(-1, 2)
        lon, lat = p[:, 0] * 2 * np.pi, -p[:, 1] * 2 * np.pi
        return np.column_stack([np.cos(lat) * np.sin(lon), -np.sin(lat), np.cos(lat) * np.cos(lon)])

    def pixel_bearing(self, p) -> np.ndarray:
        return self.pixel_bearing_many(p)[0]


class PinholeCamera:
    """pixel_bearing of a distortion-free perspective camera with normalised image coordinates."""

    def __init__(self, focal: float = 0.9, camera_id: str = "pinhole"):
        self.focal, self.id = focal, camera_id

    def project(self, pc: np.ndarray) -> np.ndarray:
        return self.focal * pc[:, :2] / pc[:, 2:3]

    def pixel_bearing_many(self, p) -> np.ndarray:
        p = np.asarray(p, dtype=np.float64).reshape(-1, 2)
        b = np.column_stack([p / self.focal, np.ones(len(p))])
        return b / np.linalg.norm(b, axis=1)[:, None]

    def pixel_bearing(self, p) -> np.ndarray:
        return self.pixel_bearing_many(p)[0]


class DictTracksManager:
    """The part of pymap.TracksManager the reference's triangulation loop reads, over dictionaries."""

    def __init__(self):
        self.tracks: Dict[str, Dict[str, map_types.Observation]] = {}

    def add_observation(self, shot_id: str, track_id: str, obs: map_types.Observation) -> None:
        self.tracks.setdefault(track_id, {})[shot_id] = obs

    def get_track_observations(self, track_id: str) -> Dict[str, map_types.Observation]:
        return dict(sorted(self.tracks[track_id].items()))

    def get_observation(self, shot_id: str, track_id: str) -> map_types.Observation:
        return self.tracks[track_id][shot_id]

    def get_shot_ids(self) -> List[str]:
        return sorted({s for t in self.tracks.values() for s in t})

    def get_shot_observations(self, shot_id: str) -> Dict[str, map_types.Observation]:
        return {t: o[shot_id] for t, o in self.tracks.items() if shot_id in o}


def reconstruction_from_json(case: Dict[str, Any], camera) -> map_types.Reconstruction:
    rec = map_types.Reconstruction()
    rec.add_camera(camera)
    for shot_id, pose in case["shots"].items():
        rec.create_shot(shot_id, camera.id, T.Pose(pose["rotation"], pose["translation"]))
    return rec


def known_answer_inputs(case: Dict[str, Any]):
    """(features {shot: 1 x 3}, colors, matches) of the case's one track, for create_tracks_manager."""
    obs = case["observations"]
    features = {s: np.array([[xy[0], xy[1], 1.0]]) for s, xy in obs.items()}
    colors = {s: np.zeros((1, 3), dtype=np.uint8) for s in obs}
    shots = sorted(obs)
    return features, colors, {(shots[0], shots[1]): [(0, 0)]}


# ---------------------------------------------------------------------------------------------------------------
# synthetic scenes
# ---------------------------------------------------------------------------------------------------------------
class Scene:
    """Shots (id -> world-to-camera rotation, origin), the observations of every point ({shot: xy} per point) and
    the tracks-manager inputs made of them: one feature per observation, each point's observations chained by
    matches."""

    def __init__(self):
        self.R: Dict[str, np.ndarray] = {}
        self.origin: Dict[str, np.ndarray] = {}
        self.points: List[Dict[str, np.ndarray]] = []

    def add_shot(self, shot_id: str, R: np.ndarray, origin: np.ndarray) -> None:
        self.R[shot_id], self.origin[shot_id] = np.asarray(R, dtype=np.float64), np.asarray(origin, dtype=np.float64)

    def observe(self, camera: PinholeCamera, X: np.ndarray, shots: List[str], rng, noise: float) -> None:
        obs = {}
        for s in shots:
            pc = (self.R[s] @ (X - self.origin[s]))[None, :]
            obs[s] = camera.project(pc)[0] + rng.normal(0.0, noise, 2)
        self.points.append(obs)

    def tracks_inputs(self):
        feats: Dict[str, List[np.ndarray]] = {s: [] for s in self.R}
        matches: Dict[Tuple[str, str], List[Tuple[int, int]]] = {}
        for obs in self.points:
            chain = []
            for s in sorted(obs):
                chain.append((s, len(feats[s])))
                feats[s].append(np.array([obs[s][0], obs[s][1], 0.004]))
            for (a, fa), (b, fb) in zip(chain[:-1], chain[1:]):
                matches.setdefault((a, b), []).append((fa, fb))
        features = {s: np.array(f).reshape(-1, 3) for s, f in feats.items() if len(f)}
        colors = {s: np.zeros((len(f), 3), dtype=np.uint8) for s, f in features.items()}
        return features, colors, matches

    def reconstruction(self, camera, shots, rng, rotation_noise: float = 0.0, position_noise: float = 0.0):
        """The map of the given shots, their poses perturbed."""
        rec = map_types.Reconstruction()
        rec.add_camera(camera)
        for s in shots:
            R = synthetic.angle_axis_to_rotation(rng.normal(0.0, rotation_noise, 3)) @ self.R[s]
            o = self.origin[s] + rng.normal(0.0, position_noise, 3)
            pose = T.Pose()
            pose.set_rotation_matrix(R)
            pose.set_origin(o)
            rec.create_shot(s, camera.id, pose)
        return rec


def cube_case(seed: int = 3, num_cameras: int = 16, num_points: int = 700):
    """Scene of synthetic.cube_scene's cameras and points, with noisy pinhole observations, plus tracks made to fail:
    outlier observations (reprojection test), cameras placed right at a point (depth test), pairs of cameras a
    fraction of a degree apart that alone see a point (angle test); some shots stay out of the reconstruction, so
    that some tracks have fewer than 2 observations in it.  Returns (scene, camera, shots of the reconstruction)."""
    rng = np.random.RandomState(seed)
    cube = synthetic.cube_scene(num_cameras, num_points, 0.0, seed=seed, with_descriptors=False)
    camera = PinholeCamera()
    sc = Scene()
    shots = ["s%02d" % i for i in range(num_cameras)]
    for i, s in enumerate(shots):
        sc.add_shot(s, cube.R_wc[i], cube.origins[i])
    seen: Dict[int, List[str]] = {}
    for s, p in zip(cube.obs_shot.tolist(), cube.obs_point.tolist()):
        seen.setdefault(p, []).append(shots[s])
    for p in sorted(seen):
        sc.observe(camera, cube.points[p], seen[p], rng, 1.0 / 800)
    # outliers: a random point in place of one observation of every 15th track
    for obs in sc.points[::15]:
        s = sorted(obs)[rng.randint(len(obs))]
        obs[s] = rng.uniform(-0.4, 0.4, 2)
    # a camera 1e-4 in front of a point, on the ray of a camera that sees it, with that camera's rotation
    for k, p in enumerate(sorted(seen)[1:200:20]):
        X, s = cube.points[p], seen[p][0]
        d = (X - sc.origin[s]) / np.linalg.norm(X - sc.origin[s])
        sid = "z%02d" % k
        sc.add_shot(sid, sc.R[s], X - 1e-4 * d)
        sc.points[sorted(seen).index(p)][sid] = camera.project((sc.R[s] @ (1e-4 * d))[None, :])[0]
        shots.append(sid)
    # near-parallel rays: two cameras 0.02 apart, 2.0 from a point only they see (0.57 degrees)
    for k in range(6):
        X = rng.uniform(-0.5, 0.5, 3)
        o = X + 2.0 * synthetic._normalized(rng.normal(size=3))
        R, _ = synthetic.camera_pose(o, X, [0.0, 0.0, 1.0])
        a, b = "p%02da" % k, "p%02db" % k
        sc.add_shot(a, R, o)
        sc.add_shot(b, R, o + 0.02 * R[0])
        sc.observe(camera, X, [a, b], rng, 1.0 / 800)
        shots += [a, b]
    # a few cube shots stay out of the reconstruction, and some points are seen by one of them and one other shot
    out = ("s01", "s05", "s09")
    for p in [p for p in sorted(seen) if "s01" in seen[p] and "s02" in seen[p]][:8]:
        sc.observe(camera, cube.points[p] + 0.01, ["s01", "s02"], rng, 1.0 / 800)
    in_rec = [s for s in shots if s not in out]
    return sc, camera, in_rec


def ring_case(lengths=(200, 40, 33), seed: int = 5):
    """Long tracks: max(lengths) cameras on a ring of radius 3 around the origin, looking at it; point k near the
    origin is seen by the first lengths[k] of them."""
    rng = np.random.RandomState(seed)
    camera = PinholeCamera()
    sc = Scene()
    n = max(lengths)
    shots = ["r%03d" % i for i in range(n)]
    for i, s in enumerate(shots):
        a = 2 * np.pi * i / n
        o = np.array([3 * np.cos(a), 3 * np.sin(a), 0.3 * np.sin(3 * a)])
        R, _ = synthetic.camera_pose(o, [0.0, 0.0, 0.0], [0.0, 0.0, 1.0])
        sc.add_shot(s, R, o)
    for L in lengths:
        sc.observe(camera, rng.uniform(-0.1, 0.1, 3), shots[:L], rng, 1.0 / 800)
    return sc, camera, shots
