"""In-memory stand-ins for the parts of `opensfm.types.Reconstruction` / `pymap.Map` that bundle adjustment reads
and writes (opensfm/types.py, opensfm/src/map/pymap.pyi: Map, Shot, Landmark, RigInstance, RigCamera, Observation,
ShotMeasurements).  `pymap` is a compiled extension that cannot be built in this image (Eigen missing), so the
drop-in functions of `opensfm_b200.reconstruction` are duck-typed: they accept the real `types.Reconstruction` as
well as this one.  This one additionally keeps the observations as growing arrays so that the whole map exports to
the engine's SoA form without a Python loop per observation (`export_observations`, SURVEY.md §8f.2).

Attribute names and meanings are the reference's; nothing here is on the GPU path.
"""
from __future__ import annotations

from typing import Any, Dict, Iterable, List, Optional, Tuple

import numpy as np

from . import types as T


class Measurement:
    """pymap.ShotMeasurementDouble / Vec3d: an optional value (has_value / value / reset)."""

    def __init__(self):
        self._v = None

    @property
    def has_value(self) -> bool:
        return self._v is not None

    @property
    def value(self):
        return self._v

    @value.setter
    def value(self, v) -> None:
        self._v = np.asarray(v, dtype=np.float64).copy() if np.ndim(v) else float(v)

    def reset(self) -> None:
        self._v = None


class ShotMeasurements:
    def __init__(self):
        self.gps_position = Measurement()
        self.gps_accuracy = Measurement()
        self.compass_angle = Measurement()
        self.compass_accuracy = Measurement()
        self.gravity_down = Measurement()
        self.capture_time = Measurement()


class Depth:
    """pymap.Depth: a depth prior carried by an observation (value, its standard deviation, radial or along z)."""

    def __init__(self, value: float, std_deviation: float, is_radial: bool = True):
        self.value = float(value)
        self.std_deviation = float(std_deviation)
        self.is_radial = bool(is_radial)


class Observation:
    """pymap.Observation: normalised image point, scale (its std-deviation in the bundle), optional depth prior."""

    def __init__(self, x: float, y: float, s: float, r: int = 0, g: int = 0, b: int = 0, feature: int = -1,
                 segmentation: int = -1, instance: int = -1):
        self.point = np.array([x, y], dtype=np.float64)
        self.scale = float(s)
        self.color = np.array([r, g, b], dtype=np.int32)
        self.id = int(feature)
        self.segmentation = segmentation
        self.instance = instance
        self.depth_prior = None


class RigCamera:
    def __init__(self, pose: Optional[T.Pose] = None, rig_camera_id: str = ""):
        self.pose = pose if pose is not None else T.Pose()
        self.id = rig_camera_id


class RigInstance:
    def __init__(self, instance_id: str):
        self.id = instance_id
        self.pose = T.Pose()
        self.shots: Dict[str, "Shot"] = {}
        self.rig_cameras: Dict[str, RigCamera] = {}

    @property
    def rig_camera_ids(self) -> Dict[str, str]:
        return {s: rc.id for s, rc in self.rig_cameras.items()}

    @property
    def camera_ids(self) -> Dict[str, str]:
        return {s: sh.camera.id for s, sh in self.shots.items()}

    def keys(self):
        return set(self.shots)

    def add_shot(self, rig_camera: RigCamera, shot: "Shot") -> None:
        self.shots[shot.id] = shot
        self.rig_cameras[shot.id] = rig_camera
        shot.rig_instance = self
        shot.rig_camera = rig_camera


class _ShotPose:
    """`shot.pose`: rig camera pose o rig instance pose (map/shot.h); setters move the instance
    (RigInstance::UpdateInstancePoseWithShot) so that `shot.pose.set_origin(...)` works as in the reference."""

    def __init__(self, shot: "Shot"):
        self._s = shot

    def _compose(self) -> T.Pose:
        ri, rc = self._s.rig_instance.pose, self._s.rig_camera.pose
        R = rc.get_rotation_matrix() @ ri.get_rotation_matrix()
        p = T.Pose()
        p.set_rotation_matrix(R)
        p.translation = rc.get_rotation_matrix() @ ri.translation + rc.translation
        return p

    def _assign(self, shot_pose: T.Pose) -> None:
        rc = self._s.rig_camera.pose
        Rc = rc.get_rotation_matrix()
        ri = T.Pose()
        ri.set_rotation_matrix(Rc.T @ shot_pose.get_rotation_matrix())
        ri.translation = Rc.T @ (shot_pose.translation - rc.translation)
        self._s.rig_instance.pose = ri

    rotation = property(lambda self: self._compose().rotation)
    translation = property(lambda self: self._compose().translation)

    def get_origin(self):
        return self._compose().get_origin()

    def get_rotation_matrix(self):
        return self._compose().get_rotation_matrix()

    def set_origin(self, origin) -> None:
        p = self._compose()
        p.set_origin(origin)
        self._assign(p)

    def set_rotation_matrix(self, R) -> None:
        p = self._compose()
        o = p.get_origin()
        p.set_rotation_matrix(R)
        p.set_origin(o)
        self._assign(p)

    def transform(self, point):
        p = self._compose()
        return p.get_rotation_matrix() @ np.asarray(point, dtype=np.float64) + p.translation


class Shot:
    def __init__(self, shot_id: str, camera, rig_instance: RigInstance, rig_camera: RigCamera, owner: "Reconstruction"):
        self.id = shot_id
        self.camera = camera
        self.metadata = ShotMeasurements()
        self.rig_instance = rig_instance
        self.rig_camera = rig_camera
        self._map = owner

    @property
    def rig_instance_id(self) -> str:
        return self.rig_instance.id

    @property
    def rig_camera_id(self) -> str:
        return self.rig_camera.id

    @property
    def pose(self) -> _ShotPose:
        return _ShotPose(self)

    def get_valid_landmarks(self) -> List["Landmark"]:
        return [self._map.points[p] for p in self._map._shot_obs.get(self.id, {})]

    def get_landmark_observation(self, lm: "Landmark") -> Observation:
        return self._map._shot_obs[self.id][lm.id]


class Landmark:
    def __init__(self, lm_id: str, coordinates, owner: "Reconstruction"):
        self.id = lm_id
        self.coordinates = np.asarray(coordinates, dtype=np.float64).copy()
        self.reprojection_errors: Dict[str, np.ndarray] = {}
        self.color = np.zeros(3, dtype=np.int32)
        self._map = owner

    def get_observations(self) -> Dict[Shot, int]:
        return {self._map.shots[s]: o.id for s, o in self._map._pt_obs.get(self.id, {}).items()}

    def number_of_observations(self) -> int:
        return len(self._map._pt_obs.get(self.id, {}))


class GroundControlPointObservation:
    def __init__(self, shot_id: str = "", projection=(0.0, 0.0)):
        self.shot_id = shot_id
        self.projection = np.asarray(projection, dtype=np.float64)


class GroundControlPoint:
    """pymap.GroundControlPoint: id, optional lla (dict latitude / longitude / altitude), has_altitude, image
    observations."""

    def __init__(self):
        self.id = ""
        self.lla: Dict[str, float] = {}
        self.has_altitude = False
        self.observations: List[GroundControlPointObservation] = []

    def add_observation(self, obs: GroundControlPointObservation) -> None:
        self.observations.append(obs)


class Reconstruction:
    """The containers `reconstruction.bundle*` touch: cameras, biases, rig cameras, rig instances, shots, points
    (dicts keyed by id, insertion ordered) and the observation graph."""

    def __init__(self):
        self.cameras: Dict[str, Any] = {}
        self.biases: Dict[str, np.ndarray] = {}     # camera id -> [rotation(3) | translation(3) | scale]
        self.rig_cameras: Dict[str, RigCamera] = {}
        self.rig_instances: Dict[str, RigInstance] = {}
        self.shots: Dict[str, Shot] = {}
        self._points: Dict[str, Landmark] = {}
        self._shot_obs: Dict[str, Dict[str, Observation]] = {}
        self._pt_obs: Dict[str, Dict[str, Observation]] = {}
        self.reference = None   # object with to_topocentric(lat, lon, alt) (opensfm.geo.TopocentricConverter)

    @property
    def points(self) -> Dict[str, Landmark]:
        return self._points

    @points.setter
    def points(self, value: Dict[str, Landmark]) -> None:
        """Replaces every point, dropping all observations, as types.Reconstruction.set_points does."""
        self._shot_obs.clear()
        self._pt_obs.clear()
        self._points = {}
        for lm in list(value.values()):
            self.create_point(lm.id, lm.coordinates)

    @property
    def map(self) -> "Reconstruction":
        return self

    # -- construction (types.Reconstruction: add_camera / create_shot / create_point / add_observation) --------
    def add_camera(self, camera) -> None:
        self.cameras[camera.id] = camera
        self.biases[camera.id] = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])

    def add_rig_camera(self, rig_camera: RigCamera) -> RigCamera:
        self.rig_cameras[rig_camera.id] = rig_camera
        return rig_camera

    def add_rig_instance(self, instance: RigInstance) -> RigInstance:
        self.rig_instances[instance.id] = instance
        return instance

    def create_shot(self, shot_id: str, camera_id: str, pose: Optional[T.Pose] = None,
                    rig_camera_id: Optional[str] = None, rig_instance_id: Optional[str] = None) -> Shot:
        """A shot without an explicit rig gets an identity rig camera named after its camera and an instance named
        after the shot (opensfm/types.py:188-192)."""
        rc_id = camera_id if rig_camera_id is None else rig_camera_id
        ri_id = shot_id if rig_instance_id is None else rig_instance_id
        if rc_id not in self.rig_cameras:
            self.add_rig_camera(RigCamera(T.Pose(), rc_id))
        if ri_id not in self.rig_instances:
            self.add_rig_instance(RigInstance(ri_id))
        shot = Shot(shot_id, self.cameras[camera_id], self.rig_instances[ri_id], self.rig_cameras[rc_id], self)
        self.rig_instances[ri_id].add_shot(self.rig_cameras[rc_id], shot)
        self.shots[shot_id] = shot
        if pose is not None:
            shot.pose._assign(pose)
        return shot

    def create_point(self, point_id: str, coordinates) -> Landmark:
        lm = Landmark(point_id, coordinates, self)
        self.points[point_id] = lm
        return lm

    def add_observation(self, shot_id: str, point_id: str, obs: Observation) -> None:
        self._shot_obs.setdefault(shot_id, {})[point_id] = obs
        self._pt_obs.setdefault(point_id, {})[shot_id] = obs

    def remove_observation(self, shot_id: str, point_id: str) -> None:
        self._shot_obs.get(shot_id, {}).pop(point_id, None)
        self._pt_obs.get(point_id, {}).pop(shot_id, None)

    def remove_landmark(self, lm: Landmark) -> None:
        for s in list(self._pt_obs.get(lm.id, {})):
            self._shot_obs[s].pop(lm.id, None)
        self._pt_obs.pop(lm.id, None)
        self.points.pop(lm.id, None)

    def number_of_shots(self) -> int:
        return len(self.shots)

    # -- bulk export (SURVEY.md §8f.2) -------------------------------------------------------------------------
    def export_observations(self, shot_ids: Optional[Iterable[str]] = None, point_ids: Optional[Iterable[str]] = None
                            ) -> Tuple[List[str], List[str], np.ndarray, np.ndarray]:
        """Observations of the given shots (all when None), restricted to the given points: parallel lists / arrays
        (shot id, point id, xy[n,2], scale[n])."""
        shots = self.shots if shot_ids is None else shot_ids
        keep = None if point_ids is None else set(point_ids)
        so, po, xy, sc = [], [], [], []
        for s in shots:
            for p, o in self._shot_obs.get(s, {}).items():
                if keep is not None and p not in keep:
                    continue
                so.append(s); po.append(p); xy.append(o.point); sc.append(o.scale)
        return so, po, np.asarray(xy, dtype=np.float64).reshape(-1, 2), np.asarray(sc, dtype=np.float64)
