"""OpenSfM's image undistortion on the GPU: `opensfm.undistort.undistort_image` and its batched form.

The reference (opensfm/undistort.py:90-232,360-403) rebuilds every image's camera mapping on the host
(`pygeometry.compute_camera_mapping`, one Bearing and one Project per pixel) and remaps with `cv2.remap`; spherical
shots render six perspective faces through numpy.  Here the `osfm_undistort` handle computes each output pixel's
source coordinate in fp64 on the device, rounds it to f32 as the reference stores its maps, and samples with
`cv2.remap`'s fixed-point rules, fused with `scale_image`'s nearest resize.  Wherever the f32 coordinates agree, the
result equals the reference's bit for bit (oracle/undistort_oracle.py restates every rule).

Deliberate differences: CUDA's fp64 atan2 / sqrt and the face rotation's summation order may move an f32
coordinate by an ulp, which rarely moves the fixed-point coordinate rint(32 x); only `uint8` and `uint16` images
with 1, 3 or 4 channels are accepted (NotImplementedError otherwise).

Cameras are duck-typed through `types.camera_type_id` / `camera_values` (pygeometry.Camera or types.Camera); shots
need `.id`, `.camera` and `.pose.get_rotation_matrix()`.
"""
from __future__ import annotations

import ctypes
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .types import camera_type_id, camera_values

# cv2's flag values
INTER_NEAREST, INTER_LINEAR, INTER_AREA = 0, 1, 3
BORDER_CONSTANT, BORDER_WRAP = 0, 3
JOB_INTS, PARAMS = 12, 16
CAMERA, FACE = 0, 1
UNDISTORTABLE = ("perspective", "brown", "fisheye", "fisheye_opencv", "fisheye62")
PANORAMAS = ("spherical", "equirectangular")


def _projection_name(camera) -> str:
    pt = camera.projection_type
    return pt if isinstance(pt, str) else str(pt).split(".")[-1].lower()


def scaled_size(width: int, height: int, max_size: int) -> Tuple[int, int]:
    """The (width, height) scale_image resizes a width x height image to (undistort.py:224-232)."""
    factor = max_size / float(max(height, width))
    if factor >= 1:
        return width, height
    return int(round(width * factor)), int(round(height * factor))


def face_rotation(panoshot, perspectiveshot) -> np.ndarray:
    """R_pano R_face^T, as render_perspective_view_of_a_panorama computes it."""
    return np.dot(panoshot.pose.get_rotation_matrix(), perspectiveshot.pose.get_rotation_matrix().T)


def _sampling(interpolation: int) -> int:
    if interpolation == INTER_NEAREST:
        return INTER_NEAREST
    if interpolation in (INTER_LINEAR, INTER_AREA):
        return INTER_LINEAR
    raise NotImplementedError("interpolation %r: INTER_NEAREST, INTER_LINEAR and INTER_AREA are supported"
                              % (interpolation,))


def _border(border: int) -> int:
    if border not in (BORDER_CONSTANT, BORDER_WRAP):
        raise NotImplementedError("border mode %r: BORDER_CONSTANT and BORDER_WRAP are supported" % (border,))
    return border


def _layout(image: np.ndarray) -> Tuple[np.ndarray, int, int]:
    """(C-contiguous image, channels, bytes per sample); NotImplementedError for anything but uint8 / uint16 images
    with 1, 3 or 4 channels."""
    if image.dtype not in (np.uint8, np.uint16):
        raise NotImplementedError("undistort: image dtype %s; uint8 and uint16 are supported" % image.dtype)
    if image.ndim == 2:
        ch = 1
    elif image.ndim == 3 and image.shape[2] in (1, 3, 4):
        ch = image.shape[2]
    else:
        raise NotImplementedError("undistort: image of shape %s; 1, 3 or 4 channels are supported" % (image.shape,))
    return np.ascontiguousarray(image), ch, image.dtype.itemsize


def _out_shape(image: np.ndarray, width: int, height: int) -> Tuple[int, ...]:
    # cv2 returns single-channel images without a channel axis
    return (height, width) if image.ndim == 2 or image.shape[2] == 1 else (height, width, image.shape[2])


def _camera_params(from_camera, to_camera) -> Tuple[int, np.ndarray]:
    """(projection type, OSFM_UNDISTORT_PARAMS doubles) of a camera mapping; NotImplementedError unless `from` is
    undistortable and `to` perspective with k1 = k2 = 0."""
    name = _projection_name(from_camera)
    if name not in UNDISTORTABLE:
        raise NotImplementedError("Undistort not implemented for projection type: {}".format(name))
    tv = camera_values(to_camera)
    if _projection_name(to_camera) != "perspective" or tv[0] != 0.0 or tv[1] != 0.0:
        raise NotImplementedError("undistort: the target camera must be perspective with k1 = k2 = 0")
    p = np.zeros(PARAMS)
    v = camera_values(from_camera)
    p[:len(v)] = v
    p[12] = tv[2]
    return camera_type_id(from_camera), p


class _Job:
    """One output image: where its pixels come from and what it is called."""

    def __init__(self, key, image, kind, ptype, params, grid, interpolation, border, out_size):
        self.key, self.image = key, image
        self.src, ch, nbytes = _layout(image)
        h, w = self.src.shape[:2]
        self.ints = [w, h, ch, nbytes, _sampling(interpolation), _border(border), kind, ptype, grid[0], grid[1],
                     out_size[0], out_size[1]]
        self.params = params
        self.out = np.empty(_out_shape(image, out_size[0], out_size[1]), dtype=image.dtype)


def _run(jobs: List[_Job], device: int = 0) -> None:
    if not jobs:
        return
    ints = np.array([j.ints for j in jobs], dtype=np.int32)
    params = np.array([j.params for j in jobs], dtype=np.float64)
    src = (ctypes.c_void_p * len(jobs))(*[j.src.ctypes.data for j in jobs])
    dst = (ctypes.c_void_p * len(jobs))(*[j.out.ctypes.data for j in jobs])
    with _lib.pooled("undistort", device) as h:
        _lib.check(h.L.osfm_undistort_run(h.h, len(jobs), _lib.ptr(ints), _lib.ptr(params), src, dst))


def _jobs_of_shot(shot, undistorted_shots, original: np.ndarray, interpolation: int, max_size: int) -> List[_Job]:
    """The jobs of undistort_image(shot, undistorted_shots, original, interpolation, max_size)."""
    name = _projection_name(shot.camera)
    if name in UNDISTORTABLE:
        [ushot] = undistorted_shots
        height, width = original.shape[:2]
        ptype, params = _camera_params(shot.camera, ushot.camera)
        return [_Job(ushot.id, original, CAMERA, ptype, params, (width, height), interpolation, BORDER_CONSTANT,
                     scaled_size(width, height, max_size))]
    if name in PANORAMAS:
        import cv2

        _layout(original)
        s = int(undistorted_shots[0].camera.width)
        image = cv2.resize(original, (4 * s, 2 * s), interpolation=interpolation)
        mint = INTER_LINEAR if interpolation == INTER_AREA else interpolation
        jobs = []
        for ushot in undistorted_shots:
            p = np.zeros(PARAMS)
            p[:9] = face_rotation(shot, ushot).ravel()
            size = (int(ushot.camera.width), int(ushot.camera.height))
            jobs.append(_Job(ushot.id, image, FACE, 0, p, size, mint, BORDER_WRAP, scaled_size(*size, max_size)))
        return jobs
    raise NotImplementedError("Undistort not implemented for projection type: {}".format(shot.camera.projection_type))


def undistort_image(shot, undistorted_shots, original: Optional[np.ndarray], interpolation: int,
                    max_size: int) -> Dict[str, np.ndarray]:
    """opensfm.undistort.undistort_image on the GPU: {undistorted shot id: image}, {} for a missing image."""
    if original is None:
        return {}
    jobs = _jobs_of_shot(shot, undistorted_shots, original, interpolation, max_size)
    _run(jobs)
    return {j.key: j.out for j in jobs}


def compute_camera_mapping(from_camera, to_camera, width: int, height: int,
                           device: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """pygeometry.compute_camera_mapping: the f32 maps (height, width) from `to_camera`'s pixels to `from_camera`'s.
    `to_camera` must be perspective with k1 = k2 = 0."""
    ptype, params = _camera_params(from_camera, to_camera)
    mx = np.empty((height, width), np.float32)
    my = np.empty((height, width), np.float32)
    with _lib.pooled("undistort", device) as h:
        _lib.check(h.L.osfm_undistort_camera_maps(h.h, ptype, _lib.ptr(params), int(width), int(height),
                                                  _lib.ptr(mx), _lib.ptr(my)))
    return mx, my


def panorama_face_mapping(panoshot, perspectiveshot, pano_width: int, pano_height: int,
                          device: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """The f32 maps render_perspective_view_of_a_panorama samples a pano_width x pano_height panorama with."""
    s = int(perspectiveshot.camera.width)
    if int(perspectiveshot.camera.height) != s:
        raise NotImplementedError("undistort: panorama faces are square")
    rot = np.ascontiguousarray(face_rotation(panoshot, perspectiveshot), dtype=np.float64)
    mx = np.empty((s, s), np.float32)
    my = np.empty((s, s), np.float32)
    with _lib.pooled("undistort", device) as h:
        _lib.check(h.L.osfm_undistort_face_maps(h.h, s, _lib.ptr(rot), int(pano_width), int(pano_height),
                                                _lib.ptr(mx), _lib.ptr(my)))
    return mx, my


def remap(image: np.ndarray, map_x: np.ndarray, map_y: np.ndarray, interpolation: int,
          border: int = BORDER_CONSTANT, device: int = 0) -> np.ndarray:
    """cv2.remap(image, map_x, map_y, interpolation, borderMode=border) with f32 maps (border value 0)."""
    src, ch, nbytes = _layout(image)
    mx = np.ascontiguousarray(map_x, dtype=np.float32)
    my = np.ascontiguousarray(map_y, dtype=np.float32)
    if mx.ndim != 2 or mx.shape != my.shape:
        raise ValueError("remap: the maps must be two arrays of one 2-d shape")
    interp, border = _sampling(interpolation), _border(border)
    out = np.empty(_out_shape(image, mx.shape[1], mx.shape[0]), dtype=image.dtype)
    with _lib.pooled("undistort", device) as h:
        _lib.check(h.L.osfm_undistort_remap(h.h, _lib.ptr(src), src.shape[1], src.shape[0], ch, nbytes, _lib.ptr(mx),
                                            _lib.ptr(my), mx.shape[1], mx.shape[0], interp, border, _lib.ptr(out)))
    return out


def render_perspective_view_of_a_panorama(image: np.ndarray, panoshot, perspectiveshot,
                                          interpolation: int = INTER_LINEAR,
                                          borderMode: int = BORDER_WRAP) -> np.ndarray:
    """opensfm.undistort.render_perspective_view_of_a_panorama on the GPU."""
    s = (int(perspectiveshot.camera.width), int(perspectiveshot.camera.height))
    if s[0] != s[1]:
        raise NotImplementedError("undistort: panorama faces are square")
    p = np.zeros(PARAMS)
    p[:9] = face_rotation(panoshot, perspectiveshot).ravel()
    job = _Job(perspectiveshot.id, image, FACE, 0, p, s, interpolation, borderMode, s)
    _run([job])
    return job.out


# ---- the batched driver -------------------------------------------------------------------------------------------

def _load(data, shot):
    return (data.load_image(shot.id, unchanged=True, anydepth=True), data.load_mask(shot.id),
            data.load_segmentation(shot.id))


def undistort_images(data, udata, undistorted_shots, device: int = 0, batch_size: Optional[int] = None) -> None:
    """The image half of opensfm.undistort.undistort_reconstruction_with_images on the GPU: for every
    {shot: [undistorted shots]} entry (or (shot, [undistorted shots]) pair), the undistorted image (INTER_AREA), mask
    and segmentation (INTER_NEAREST), saved through udata.save_undistorted_image / _mask / _segmentation under the
    undistorted shots' ids.

    Images are decoded on `read_processes` host threads, `batch_size` shots at a time (default: twice the thread
    count), while the previous batch is undistorted and saved; every batch is one submission to the device."""
    max_size = data.config["undistorted_image_max_size"]
    threads = max(1, int(data.config.get("read_processes", 1)))
    batch = max(1, int(batch_size or 2 * threads))
    items = list(undistorted_shots.items() if hasattr(undistorted_shots, "items") else undistorted_shots)
    savers = (udata.save_undistorted_image, udata.save_undistorted_mask, udata.save_undistorted_segmentation)
    interps = (INTER_AREA, INTER_NEAREST, INTER_NEAREST)
    with ThreadPoolExecutor(max_workers=threads) as pool:
        def submit(k):
            return [pool.submit(_load, data, shot) for shot, _ in items[k:k + batch]]

        pending = submit(0)
        for k in range(0, len(items), batch):
            loaded = [f.result() for f in pending]
            pending = submit(k + batch) if k + batch < len(items) else []
            jobs, saves = [], []
            for (shot, subshots), arrays in zip(items[k:k + batch], loaded):
                for image, save, interp in zip(arrays, savers, interps):
                    if image is None:
                        continue
                    js = _jobs_of_shot(shot, subshots, image, interp, max_size)
                    jobs += js
                    saves += [(save, j) for j in js]
            _run(jobs, device)
            for f in [pool.submit(save, j.key, j.out) for save, j in saves]:
                f.result()
