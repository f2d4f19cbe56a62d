"""The undistortion oracle against live cv2 and the pinned camera models, without a GPU: its remap equals cv2.remap
bit for bit on adversarial maps in every dtype, channel count, interpolation and border; its nearest resize equals
cv2.resize; its forward models equal oracle/ba_functors.hpp (pinned to the reference's golden pixels by
tests/test_oracle_ba.py); its maps follow closed forms; and the host-side helpers of opensfm_b200.undistort follow
the reference's expressions."""
import math

import cv2
import numpy as np
import pytest

import undistort_cases as uc
from opensfm_b200 import undistort as GU
from opensfm_b200.types import camera_type_id, camera_values
from oracle import ba_lm
from oracle import undistort_oracle as uo

W, H = 41, 29
LAYOUTS = [(np.uint8, 1), (np.uint8, 3), (np.uint8, 4), (np.uint16, 1), (np.uint16, 3)]


def adversarial_maps(w, h, seed=0):
    """Maps (rows of 64) with every fractional position of 1/32 on random taps, exact k/64 ties, the coordinates
    -1, -1/32, size-1, size-1+1/32 and size, and NaN, +-inf, +-1e30 and large finite values."""
    rng = np.random.RandomState(seed)
    fx, fy = np.meshgrid(np.arange(32), np.arange(32))
    n = fx.size
    xs = [rng.randint(-2, w + 2, n) + fx.ravel() / 32.0, rng.randint(-4 * 64, (w + 4) * 64, 4096) / 64.0]
    ys = [rng.randint(-2, h + 2, n) + fy.ravel() / 32.0, rng.randint(-4 * 64, (h + 4) * 64, 4096) / 64.0]
    ex = np.array([-1, -1 / 32, w - 1, w - 1 + 1 / 32, w, 0.5, 1e30, -1e30, np.nan, np.inf, -np.inf, 5e7, -5e7, 1e9])
    ey = np.array([-1, -1 / 32, h - 1, h - 1 + 1 / 32, h, 0.5, 1e30, -1e30, np.nan, np.inf, -np.inf, 5e7, -5e7, 1e9])
    gx, gy = np.meshgrid(ex, ey)
    xs.append(gx.ravel())
    ys.append(gy.ravel())
    mx = np.concatenate(xs).astype(np.float32)
    my = np.concatenate(ys).astype(np.float32)
    pad = (-len(mx)) % 64
    mx = np.concatenate([mx, np.full(pad, 0.25, np.float32)]).reshape(-1, 64)
    my = np.concatenate([my, np.full(pad, 0.75, np.float32)]).reshape(-1, 64)
    return mx, my


def random_image(dtype, ch, w=W, h=H, seed=1):
    rng = np.random.RandomState(seed)
    top = 256 if dtype == np.uint8 else 65536
    return rng.randint(0, top, (h, w) if ch == 1 else (h, w, ch)).astype(dtype)


@pytest.mark.parametrize("dtype,ch", LAYOUTS)
@pytest.mark.parametrize("interp", [cv2.INTER_LINEAR, cv2.INTER_AREA, cv2.INTER_NEAREST])
@pytest.mark.parametrize("border", [cv2.BORDER_CONSTANT, cv2.BORDER_WRAP])
def test_oracle_remap_equals_cv2(dtype, ch, interp, border):
    img = random_image(dtype, ch)
    mx, my = adversarial_maps(W, H)
    want = cv2.remap(img, mx, my, interp, borderMode=border)
    got = uo.remap(img, mx, my, interp, border)
    assert got.shape == want.shape and got.dtype == want.dtype
    assert np.array_equal(got, want), int((got != want).sum())


def test_oracle_remap_equals_cv2_at_one_pixel_images():
    for w, h in [(1, 1), (2, 1), (1, 2)]:
        mx, my = adversarial_maps(w, h, seed=w + 3 * h)
        for dtype, ch in LAYOUTS:
            img = random_image(dtype, ch, w, h)
            for interp in (cv2.INTER_LINEAR, cv2.INTER_NEAREST):
                for border in (cv2.BORDER_CONSTANT, cv2.BORDER_WRAP):
                    assert np.array_equal(uo.remap(img, mx, my, interp, border),
                                          cv2.remap(img, mx, my, interp, borderMode=border)), (w, h, dtype, ch)


def test_oracle_linear_u8_covers_every_fractional_position_with_cv2s_weights():
    """All 1024 (fx, fy) at one interior tap with values that expose any weight off by one."""
    img = np.array([[255, 1], [254, 3]], np.uint8)
    img = np.pad(img, 2)
    fx, fy = np.meshgrid(np.arange(32), np.arange(32))
    mx = (2 + fx / 32.0).astype(np.float32)
    my = (2 + fy / 32.0).astype(np.float32)
    for vals in ([[255, 1], [254, 3]], [[0, 255], [255, 0]], [[128, 129], [127, 130]], [[255, 255], [255, 255]]):
        img[2:4, 2:4] = vals
        assert np.array_equal(uo.remap(img, mx, my, cv2.INTER_LINEAR), cv2.remap(img, mx, my, cv2.INTER_LINEAR))


def test_oracle_nearest_resize_equals_cv2():
    rng = np.random.RandomState(5)
    for _ in range(300):
        sw, sh, dw, dh = (int(a) for a in rng.randint(1, 700, 4))
        img = rng.randint(0, 256, (sh, sw, 3)).astype(np.uint8)
        assert np.array_equal(uo.resize_nearest(img, dw, dh),
                              cv2.resize(img, (dw, dh), interpolation=cv2.INTER_NEAREST)), (sw, sh, dw, dh)


@pytest.mark.parametrize("model", uc.MODELS)
@pytest.mark.parametrize("strength", ["mild", "strong"])
def test_oracle_forward_models_equal_the_pinned_functors(model, strength):
    cam = uc.camera(model, strength)
    t, v = camera_type_id(cam), camera_values(cam)
    rng = np.random.RandomState(7)
    pts = np.column_stack([rng.uniform(-0.8, 0.8, (200, 2)), rng.uniform(0.3, 2.0, 200)])
    pts = np.vstack([pts, [[0, 0, 1.0], [1e-9, -1e-9, 1.0], [0.3, 0.0, 1.0]]])
    got = np.column_stack(uo.project(t, v, pts[:, 0], pts[:, 1], pts[:, 2]))
    want = np.array([ba_lm.project(t, v, p) for p in pts])
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


def test_oracle_spherical_projection_closed_form():
    rng = np.random.RandomState(8)
    b = rng.randn(500, 3)
    b /= np.linalg.norm(b, axis=1)[:, None]
    x, y = uo.project(uo.SPHERICAL, [0.0], b[:, 0], b[:, 1], b[:, 2])
    lon, lat = 2 * np.pi * x, -2 * np.pi * y
    back = np.column_stack([np.cos(lat) * np.sin(lon), -np.sin(lat), np.cos(lat) * np.cos(lon)])
    assert np.abs(back - b).max() < 1e-14


def test_oracle_camera_maps_follow_closed_forms():
    w, h = 64, 48
    n = max(w, h)
    v, u = np.indices((h, w), dtype=np.float64)
    # perspective with no distortion, focal f onto focal g: x = (f / g) (u - w/2) + w/2
    mx, my = uo.camera_mapping(uo.PERSPECTIVE, [0, 0, 0.8], 0.5, w, h)
    assert np.abs(mx - (0.8 / 0.5 * (u - w / 2) + w / 2)).max() < 1e-4
    assert np.abs(my - (0.8 / 0.5 * (v - h / 2) + h / 2)).max() < 1e-4
    # brown with no distortion: focal, aspect ratio and principal point
    mx, my = uo.camera_mapping(uo.BROWN, [0, 0, 0, 0, 0, 0.7, 1.1, 0.02, -0.03], 0.7, w, h)
    assert np.abs(mx - ((u - w / 2) + 0.02 * n + w / 2)).max() < 1e-4
    assert np.abs(my - (1.1 * (v - h / 2) - 0.03 * n + h / 2)).max() < 1e-4
    # fisheye with no distortion: the angle atan(rho) of the target ray, scaled by the focal
    a, b = (u - w / 2) / n / 0.6, (v - h / 2) / n / 0.6
    rho = np.hypot(a, b)
    s = np.where(rho > 0, np.arctan(rho) / np.where(rho > 0, rho, 1), 1.0)
    mx, my = uo.camera_mapping(uo.FISHEYE, [0, 0, 0.6], 0.6, w, h)
    assert np.abs(mx - (n * 0.6 * s * a + w / 2)).max() < 1e-4
    assert np.abs(my - (n * 0.6 * s * b + h / 2)).max() < 1e-4


def test_oracle_face_maps_follow_closed_forms():
    s, pw, ph = 32, 128, 64
    # the front face of an unrotated panorama: its centre looks along +z, the panorama's centre column and row
    mx, my = uo.face_mapping(s, np.eye(3), pw, ph)
    c = (s - 1) / 2.0
    x = (np.arange(s) + 0.5 - s / 2) / s / 0.5
    assert np.abs(mx[int(c), :] - (np.arctan2(x, np.sqrt(1 + 0 * x)) / (2 * np.pi) * pw - 0.5 + pw / 2)).max() < 1e-2
    # a yaw by R turns every longitude by the same angle
    yaw = uc.rotation_matrix(np.pi / 2, [0, 1, 0])
    mx2, _ = uo.face_mapping(s, yaw, pw, ph)
    d = np.mod(mx2 - mx, pw)
    assert np.abs(d - pw / 4).max() < 1e-3


def test_scaled_size_is_scale_images_size():
    rng = np.random.RandomState(9)
    for _ in range(200):
        w, h, m = (int(a) for a in rng.randint(1, 5000, 3))
        factor = m / float(max(h, w))
        want = (w, h) if factor >= 1 else (int(round(w * factor)), int(round(h * factor)))
        assert GU.scaled_size(w, h, m) == want
    assert GU.scaled_size(4000, 3000, 2000) == (2000, 1500)
    assert GU.scaled_size(10, 3, 3) == (3, 1)
    assert GU.scaled_size(7, 7, 7) == (7, 7)


def test_face_rotations_are_the_references():
    shot, faces = uc.panorama(16)
    for face, Rf in zip(faces, uc.FACE_ROTATIONS):
        want = np.dot(shot.pose.get_rotation_matrix(), face.pose.get_rotation_matrix().T)
        got = GU.face_rotation(shot, face)
        assert np.array_equal(got, want)
        # the face shot is the rig camera's rotation composed with the panorama's
        assert np.abs(got - Rf.T).max() < 1e-15
    # front, left, back, right turn about y by 0, 90, 180 and 270 degrees
    assert np.abs(uc.FACE_ROTATIONS[2] - np.diag([-1.0, 1.0, -1.0])).max() < 1e-15


def test_unsupported_inputs_are_refused_before_the_device():
    shot, subs = uc.shot_pair("brown", "mild", 8, 6)
    for bad in (np.zeros((6, 8), np.float32), np.zeros((6, 8, 2), np.uint8), np.zeros((6, 8, 5), np.uint16)):
        with pytest.raises(NotImplementedError):
            GU.undistort_image(shot, subs, bad, cv2.INTER_AREA, 100)
    with pytest.raises(NotImplementedError, match="Undistort not implemented for projection type: dual"):
        dual = uc.Shot("d", uc.Camera.create_dual(0.5, 0.5, 0.0, 0.0))
        GU.undistort_image(dual, subs, np.zeros((6, 8), np.uint8), cv2.INTER_AREA, 100)
    assert GU.undistort_image(shot, subs, None, cv2.INTER_AREA, 100) == {}
    with pytest.raises(NotImplementedError):
        GU.compute_camera_mapping(shot.camera, uc.Camera.create_perspective(0.5, 0.1, 0.0), 8, 6)
    with pytest.raises(NotImplementedError):
        GU.undistort_image(shot, subs, np.zeros((6, 8), np.uint8), cv2.INTER_CUBIC, 100)
    assert math.isclose(uc.undistorted_camera(uc.camera("brown", "mild")).focal, 0.85 * 2.02 / 2)
