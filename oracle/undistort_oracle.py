"""fp64 numpy restatement of OpenSfM's image undistortion, for tests only.

* `camera_mapping`: `ComputeCameraMapping` (opensfm/src/geometry/src/camera.cc:319-342) for the five undistortable
  models, through the target camera's `Bearing` (UniformScale, Disto24 and perspective backward,
  camera_instances.h:153-159, camera_projections_functions.h:111-116) and the source camera's `Project`
  (camera_projections_functions.h, camera_distortions_functions.h, transformations_functions.h).
* `face_mapping`: the coordinates `render_perspective_view_of_a_panorama` (opensfm/undistort.py:360-403) hands to
  cv2.remap, with `normalized_image_coordinates` / `denormalized_image_coordinates` (opensfm/features.py:324-341)
  and the spherical projection (camera_projections_functions.h:216-223), in the reference's numpy expressions.
* `remap`: the subset of `cv2.remap` the reference uses (float maps; INTER_NEAREST, INTER_LINEAR and INTER_AREA;
  BORDER_CONSTANT 0 and BORDER_WRAP; uint8 and uint16), as fixed-point rules.
* `resize_nearest`: `cv2.resize(..., INTER_NEAREST)`, the reference's `scale_image` (undistort.py:224-232).

Shares no code with opensfm_b200.  tests/test_undistort_oracle.py pins every rule to live cv2 and the forward models
to oracle/ba_functors.hpp.
"""
from __future__ import annotations

import math

import numpy as np

PERSPECTIVE, BROWN, FISHEYE, FISHEYE_OPENCV, FISHEYE62, SPHERICAL = 0, 1, 2, 3, 4, 6
INTER_NEAREST, INTER_LINEAR, INTER_AREA = 0, 1, 3
BORDER_CONSTANT, BORDER_WRAP = 0, 3
INT_MIN = -(2 ** 31)


# ---- forward models ---------------------------------------------------------------------------------------------

def _perspective(x, y, z):
    return x / z, y / z


def _fisheye(x, y, z):
    r = np.sqrt(x * x + y * y)
    small = r < 1e-8
    rs = np.where(small, 1.0, r)
    theta = np.arctan2(r, z)
    px = np.where(small, x / z, theta / rs * x)
    py = np.where(small, y / z, theta / rs * y)
    return px, py


def _radial(r2, ks):
    """1 + r2 (k1 + r2 (k2 + ...)), innermost last coefficient first."""
    acc = ks[-1]
    for k in ks[-2::-1]:
        acc = k + r2 * acc
    return 1.0 + r2 * acc


def _tangential(r2, x, y, p1, p2):
    return 2.0 * p1 * x * y + p2 * (r2 + 2.0 * x * x), 2.0 * p2 * x * y + p1 * (r2 + 2.0 * y * y)


def project(ptype: int, v, x, y, z):
    """Camera::Project of the camera (type, values in the reference's order) at camera-frame points (x, y, z)."""
    v = [float(a) for a in v]
    x, y, z = (np.asarray(a, dtype=np.float64) for a in (x, y, z))
    if ptype == SPHERICAL:
        lon = np.arctan2(x, z)
        lat = np.arctan2(-y, np.sqrt(x * x + z * z))
        inv = 1.0 / (2.0 * math.pi)
        return lon * inv, -lat * inv
    if ptype in (PERSPECTIVE, FISHEYE):  # Disto24, UniformScale: [k1, k2, focal]
        px, py = (_perspective if ptype == PERSPECTIVE else _fisheye)(x, y, z)
        r2 = px * px + py * py
        d = 1.0 + r2 * (v[0] + v[1] * r2)
        return v[2] * (px * d), v[2] * (py * d)
    if ptype == BROWN:  # [k1 k2 k3 p1 p2 | focal ar cx cy]
        px, py = _perspective(x, y, z)
        r2 = px * px + py * py
        rad = _radial(r2, v[0:3])
        tx, ty = _tangential(r2, px, py, v[3], v[4])
        dx, dy = px * rad + tx, py * rad + ty
        a = v[5:9]
    elif ptype == FISHEYE_OPENCV:  # [k1..k4 | focal ar cx cy]
        px, py = _fisheye(x, y, z)
        r2 = px * px + py * py
        rad = _radial(r2, v[0:4])
        dx, dy = px * rad, py * rad
        a = v[4:8]
    elif ptype == FISHEYE62:  # [k1..k6 p1 p2 | focal ar cx cy]
        px, py = _fisheye(x, y, z)
        r2 = px * px + py * py
        rad = _radial(r2, v[0:6])
        tx, ty = _tangential(r2, px, py, v[6], v[7])
        dx, dy = px * rad + tx, py * rad + ty
        a = v[8:12]
    else:
        raise NotImplementedError("projection type %d" % ptype)
    return a[0] * dx + a[2], a[0] * a[1] * dy + a[3]


def perspective_bearing(px, py, focal):
    """Bearing of a perspective camera with k1 = k2 = 0: UniformScale, Disto24 (the identity at k = 0), then the
    normalised (x, y, 1)."""
    a, b = px / focal, py / focal
    inv = 1.0 / np.sqrt((a * a + b * b) + 1.0)
    return a * inv, b * inv, inv


# ---- mappings ---------------------------------------------------------------------------------------------------

def camera_mapping(ptype: int, values, to_focal: float, width: int, height: int):
    """ComputeCameraMapping(from, to, width, height) as f32 maps (height, width)."""
    n = max(width, height)
    inv = 1.0 / n
    hw, hh = width * 0.5, height * 0.5
    v, u = np.indices((height, width), dtype=np.float64)
    bx, by, bz = perspective_bearing(inv * (u - hw), inv * (v - hh), to_focal)
    px, py = project(ptype, values, bx, by, bz)
    return (n * px + hw).astype(np.float32), (n * py + hh).astype(np.float32)


def face_mapping(face_size: int, rotation, pano_width: int, pano_height: int):
    """The maps render_perspective_view_of_a_panorama samples a face of face_size^2 pixels with, where rotation is
    R_pano R_face^T and the panorama image is pano_width x pano_height."""
    dst_y, dst_x = np.indices((face_size, face_size)).astype(np.float32)
    pix = np.column_stack([dst_x.ravel(), dst_y.ravel()])
    p = np.empty((len(pix), 2))
    p[:, 0] = (pix[:, 0] + 0.5 - face_size / 2.0) / face_size
    p[:, 1] = (pix[:, 1] + 0.5 - face_size / 2.0) / face_size
    b = np.column_stack(perspective_bearing(p[:, 0], p[:, 1], 0.5))
    rb = np.dot(b, np.asarray(rotation, dtype=np.float64).T)
    sx, sy = project(SPHERICAL, [0.0], rb[:, 0], rb[:, 1], rb[:, 2])
    size = max(pano_width, pano_height)
    x = sx * size - 0.5 + pano_width / 2.0
    y = sy * size - 0.5 + pano_height / 2.0
    return x.reshape(face_size, face_size).astype(np.float32), y.reshape(face_size, face_size).astype(np.float32)


# ---- cv2.remap and cv2.resize(INTER_NEAREST) ----------------------------------------------------------------------

def cv_round(v):
    """cvRound of float32 values on x86: round half to even; NaN and results outside int32 give INT_MIN."""
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.rint(np.asarray(v, dtype=np.float32).astype(np.float64))
        ok = (r >= -2.0 ** 31) & (r < 2.0 ** 31)
        return np.where(ok, r, INT_MIN).astype(np.int64)


def _sat16(a):
    return np.clip(a, -32768, 32767)


def _taps(img, xs, ys, border):
    """Pixel values (..., C) at integer coordinates under the border rule, and nothing else."""
    h, w = img.shape[:2]
    if border == BORDER_WRAP:
        return img[np.mod(ys, h), np.mod(xs, w)].astype(np.int64), None
    ok = (xs >= 0) & (xs < w) & (ys >= 0) & (ys < h)
    vals = img[np.where(ok, ys, 0), np.where(ok, xs, 0)].astype(np.int64)
    vals[~ok] = 0
    return vals, ok


def remap(img, map_x, map_y, interpolation: int, border: int = BORDER_CONSTANT):
    """cv2.remap(img, map_x, map_y, interpolation, borderMode=border) with f32 maps, border value 0."""
    img = np.asarray(img)
    if img.dtype not in (np.uint8, np.uint16):
        raise NotImplementedError(str(img.dtype))
    if border not in (BORDER_CONSTANT, BORDER_WRAP):
        raise NotImplementedError("border %d" % border)
    squeeze = img.ndim == 2
    im = img[..., None] if squeeze else img
    mx = np.asarray(map_x, dtype=np.float32)
    my = np.asarray(map_y, dtype=np.float32)
    if interpolation == INTER_NEAREST:
        X, Y = _sat16(cv_round(mx)), _sat16(cv_round(my))
        out, _ = _taps(im, X, Y, border)
    elif interpolation in (INTER_LINEAR, INTER_AREA):
        with np.errstate(over="ignore", invalid="ignore"):
            X = cv_round(mx * np.float32(32))
            Y = cv_round(my * np.float32(32))
        fx, fy = X & 31, Y & 31
        sx, sy = _sat16(X >> 5), _sat16(Y >> 5)
        v00, _ = _taps(im, sx, sy, border)
        v01, _ = _taps(im, sx + 1, sy, border)
        v10, _ = _taps(im, sx, sy + 1, border)
        v11, _ = _taps(im, sx + 1, sy + 1, border)
        if im.dtype == np.uint8:
            w = [((32 - fx) * (32 - fy) * 32), (fx * (32 - fy) * 32), ((32 - fx) * fy * 32), (fx * fy * 32)]
            acc = sum(v * wk[..., None] for v, wk in zip((v00, v01, v10, v11), w))
            out = np.clip((acc + (1 << 14)) >> 15, 0, 255)
        else:
            f32 = np.float32
            tx = [f32(1) - fx.astype(f32) / f32(32), fx.astype(f32) / f32(32)]
            ty = [f32(1) - fy.astype(f32) / f32(32), fy.astype(f32) / f32(32)]
            w = [ty[0] * tx[0], ty[0] * tx[1], ty[1] * tx[0], ty[1] * tx[1]]
            p = [v.astype(f32) * wk[..., None] for v, wk in zip((v00, v01, v10, v11), w)]
            acc = ((p[0] + p[1]) + p[2]) + p[3]
            out = np.clip(np.rint(acc.astype(np.float64)), 0, 65535)
    else:
        raise NotImplementedError("interpolation %d" % interpolation)
    out = out.astype(img.dtype)
    return out[..., 0] if squeeze else out


def resize_nearest(img, width: int, height: int):
    """cv2.resize(img, (width, height), interpolation=cv2.INTER_NEAREST)."""
    h, w = img.shape[:2]
    ifx, ify = 1.0 / (width / w), 1.0 / (height / h)
    xs = np.minimum(np.floor(np.arange(width) * ifx).astype(np.int64), w - 1)
    ys = np.minimum(np.floor(np.arange(height) * ify).astype(np.int64), h - 1)
    return img[ys[:, None], xs[None, :]]
