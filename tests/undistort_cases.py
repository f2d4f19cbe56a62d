"""Cameras, shots and in-memory datasets for the undistortion tests: every undistortable model with mild and strong
distortion, the perspective target cameras the reference builds for them (opensfm/undistort.py:253-307), panorama
faces as perspective_views_of_a_panorama poses them (:310-357), and stand-ins for DataSet / UndistortedDataSet."""
import numpy as np
from scipy.spatial.transform import Rotation

from opensfm_b200.types import Camera

MODELS = ("perspective", "brown", "fisheye", "fisheye_opencv", "fisheye62")


def camera(model: str, strength: str) -> Camera:
    s = 1.0 if strength == "mild" else 6.0
    if model == "perspective":
        return Camera.create_perspective(0.9, -0.05 * s, 0.01 * s)
    if model == "fisheye":
        return Camera.create_fisheye(0.45, -0.02 * s, 0.005 * s)
    if model == "brown":
        return Camera.create_brown(0.85, 1.02, [0.01, -0.02],
                                   [-0.05 * s, 0.02 * s, -0.002 * s, 0.001 * s, -0.0005 * s])
    if model == "fisheye_opencv":
        return Camera.create_fisheye_opencv(0.5, 0.98, [0.02, 0.01], [0.02 * s, -0.01 * s, 0.002 * s, -0.0005 * s])
    return Camera.create_fisheye62(0.5, 1.01, [-0.01, 0.015], [0.02 * s, -0.01 * s, 0.002 * s, -0.0005 * s,
                                                               0.0001 * s, 0.00002 * s, 0.001 * s, -0.0008 * s])


def undistorted_camera(cam: Camera) -> Camera:
    """perspective_camera_from_perspective / _brown / _fisheye / _fisheye_opencv / _fisheye62."""
    f = cam.focal if cam.projection_type in ("perspective", "fisheye") else cam.focal * (1 + cam.aspect_ratio) / 2.0
    out = Camera.create_perspective(f, 0.0, 0.0)
    out.id, out.width, out.height = cam.id, cam.width, cam.height
    return out


class Pose:
    def __init__(self, R):
        self.R = np.asarray(R, dtype=np.float64)

    def get_rotation_matrix(self):
        return self.R


class Shot:
    def __init__(self, sid, camera, R=np.eye(3)):
        self.id, self.camera, self.pose = sid, camera, Pose(R)


def rotation_matrix(angle, axis):
    """The rotation part of transformations.rotation_matrix(angle, axis)."""
    axis = np.asarray(axis, dtype=np.float64)
    return Rotation.from_rotvec(angle * axis / np.linalg.norm(axis)).as_matrix()


FACE_NAMES = ["front", "left", "back", "right", "top", "bottom"]
FACE_ROTATIONS = [rotation_matrix(-k * np.pi / 2, [0, 1, 0]) for k in range(4)] + [
    rotation_matrix(-np.pi / 2, [1, 0, 0]), rotation_matrix(np.pi / 2, [1, 0, 0])]


def shot_pair(model: str, strength: str, width: int, height: int, sid: str = "im"):
    """A distorted shot of `model` and its one undistorted shot."""
    cam = camera(model, strength)
    cam.id, cam.width, cam.height = model, width, height
    shot = Shot(sid, cam, Rotation.from_rotvec([0.1, -0.2, 0.3]).as_matrix())
    return shot, [Shot(sid + ".jpg", undistorted_camera(cam), shot.pose.R)]


def panorama(face_size: int, sid: str = "pano"):
    """A spherical shot with a pose and its six face shots (rig camera rotation times the shot's)."""
    cam = Camera.create_spherical()
    cam.id, cam.width, cam.height = "sph", 2 * face_size * 2, face_size * 2
    R = Rotation.from_rotvec([0.05, 0.4, -0.1]).as_matrix()
    shot = Shot(sid, cam, R)
    face = Camera.create_perspective(0.5, 0.0, 0.0)
    face.id, face.width, face.height = "perspective_panorama_camera", face_size, face_size
    return shot, [Shot("%s_perspective_view_%s.jpg" % (sid, n), face, Rf @ R)
                  for n, Rf in zip(FACE_NAMES, FACE_ROTATIONS)]


class DataSet:
    """load_image / load_mask / load_segmentation over dicts, and the config undistortion reads."""

    def __init__(self, images, masks, segmentations, max_size=100000, read_processes=3):
        self.images, self.masks, self.segmentations = images, masks, segmentations
        self.config = {"undistorted_image_max_size": max_size, "read_processes": read_processes}

    def load_image(self, sid, unchanged=False, anydepth=False):
        assert unchanged and anydepth
        return self.images[sid]

    def load_mask(self, sid):
        return self.masks.get(sid)

    def load_segmentation(self, sid):
        return self.segmentations.get(sid)


class UndistortedDataSet:
    def __init__(self):
        self.saved = {}

    def save_undistorted_image(self, key, image):
        self.saved[("image", key)] = np.array(image)

    def save_undistorted_mask(self, key, image):
        self.saved[("mask", key)] = np.array(image)

    def save_undistorted_segmentation(self, key, image):
        self.saved[("segmentation", key)] = np.array(image)
