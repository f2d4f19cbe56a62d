"""The dense oracle (oracle/dense_oracle.cpp) on the CPU: the reference's depthmap_test.cc cases restated on it, its
median against cv2, its generator's exp / log, and its three estimators' accuracy on textured_scene."""
import math

import cv2
import numpy as np
import pytest

from opensfm_b200 import dense as D
from opensfm_b200 import synthetic as syn
from oracle import dense_oracle as do

K = np.array([[600.0, 0, 320], [0, 600, 240], [0, 0, 1]])


def _rot(ax, ang):
    return syn.angle_axis_to_rotation(np.asarray(ax, float) * ang)


def test_plane_induced_homography():
    """depthmap_test.cc TEST(PlaneInducedHomography, RandomPoint) on the oracle's baked homography (the one its score
    uses, rounded to f32), applied as ApplyHomography applies it: 1e-4."""
    K1 = np.array([[600.0, 0, 300], [0, 400, 200], [0, 0, 1]])
    K2 = np.array([[400.0, 0, 200], [0, 300, 150], [0, 0, 1]])
    R1, t1 = cv2.Rodrigues(np.array([0.1, 0.1, 0.1]))[0], np.array([0.1, 0.2, 0.3])
    R2, t2 = cv2.Rodrigues(np.array([0.1, 0.2, 0.3]))[0], np.array([-0.3, -0.1, 0.2])
    v = np.array([0.5, 0.7, -1.0])
    pc = np.array([-1 - v[2], -1 - v[2], 1.0])
    assert abs(v @ pc + 1) < 1e-6
    p = R1.T @ (pc - t1)
    p1, p2 = K1 @ (R1 @ p + t1), K2 @ (R2 @ p + t2)
    x1, y1 = np.float32(p1[0] / p1[2]), np.float32(p1[1] / p1[2])
    Kinv, Q, a = D.view_terms([K1, K2], [R1, R2], [t1, t2])
    H = do.homography(Kinv[0], Q[1], a[1], K2, v.astype(np.float32))
    w = H[2, 0] * x1 + H[2, 1] * y1 + H[2, 2]
    x2 = (H[0, 0] * x1 + H[0, 1] * y1 + H[0, 2]) / w
    y2 = (H[1, 0] * x1 + H[1, 1] * y1 + H[1, 2]) / w
    assert abs(x2 - p2[0] / p2[2]) < 1e-4 and abs(y2 - p2[1] / p2[2]) < 1e-4


def test_depth_plane_loop():
    """depthmap_test.cc TEST(DepthOfPlaneBackprojection, DepthNormalPlaneLoop): 1e-6, over random normals."""
    Kinv = np.linalg.inv(np.array([[600.0, 0, 300], [0, 400, 200], [0, 0, 1]]))
    rng = np.random.RandomState(0)
    for _ in range(100):
        normal = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), -1.0], np.float32)
        pl = do.plane_from_depth_normal(20, 30, Kinv, 3.0, normal)
        assert abs(do.depth_of_plane(20, 30, Kinv, pl) - 3.0) < 1e-6


def test_backproject_project():
    """depthmap_test.cc TEST(Backproject, Reprojection): 1e-6."""
    K1 = np.array([[600.0, 0, 300], [0, 400, 200], [0, 0, 1]])
    R, t = cv2.Rodrigues(np.array([0.1, 0.1, 0.1]))[0], np.array([0.1, 0.2, 0.3])
    X = do.backproject(10.0, 20.0, 13.0, np.linalg.inv(K1), R, t)
    p = do.project(X, K1, R, t)
    assert abs(p[2] - 13) < 1e-6 and abs(p[0] / p[2] - 10) < 1e-6 and abs(p[1] / p[2] - 20) < 1e-6


def test_ncc_of_a_line_is_one():
    x = np.arange(10, dtype=np.float32)
    assert abs(do.ncc(x, 2 * x + 3, np.ones(10)) - 1.0) < 1e-6
    assert abs(do.ncc(x, -x, np.ones(10)) + 1.0) < 1e-6
    assert do.ncc(x, np.ones(10), np.ones(10)) == -1.0       # variance below 0.1
    assert do.ncc(x, x, np.zeros(10)) == -1.0                # no weight


def test_median_equals_cv2():
    rng = np.random.RandomState(0)
    for h, w in [(5, 5), (17, 31), (64, 48)]:
        d = rng.uniform(1, 10, (h, w)).astype(np.float32)
        d[rng.rand(h, w) < 0.4] = 0
        assert np.array_equal(do.median5(d), cv2.medianBlur(d, 5))


def test_generator_exp_log():
    for x in [1e-300, 1e-8, 0.02, 0.5, 1.0, 1.5, 2.0, 1e3, 1e300]:
        assert abs(do.log(x) - math.log(x)) <= 4e-16 * max(1.0, abs(math.log(x)))
    for x in [-700.0, -20.0, -1.0, -1e-3, 0.0, 1e-3, 0.3, 1.0, 20.0, 700.0]:
        assert abs(do.exp(x) - math.exp(x)) <= (4e-15 if abs(x) < 30 else 1e-13) * math.exp(x)
    z = np.array([do.normal(p, 1, 3, 7, 11) for p in range(20000)])
    assert abs(z.mean()) < 0.03 and abs(z.std() - 1.0) < 0.03
    # Philox4x32-10 known answer (Random123 kat_vectors: ctr = key = 0)
    assert do.philox([0, 0, 0, 0], [0, 0]).tolist() == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]


def test_bilateral_weights_table():
    w = D.bilateral_weights()
    for dc, dx, dy in [(0, 0, 0), (10, 1, 2), (255, 7, 7), (37, 3, 0)]:
        arg = np.float32(-dc) * np.float32(dc) * np.float32(1 / 5000.0) - np.float32(dx * dx + dy * dy) * np.float32(0.02)
        assert abs(w[dc, dx * dx + dy * dy] - math.exp(float(arg))) <= 1e-7


# Floors measured on this scene with the oracle on the CPU (0.25, 0.54, 0.535 at the time of writing)
FLOORS = {"BRUTE_FORCE": 0.22, "PATCH_MATCH": 0.48, "PATCH_MATCH_SAMPLE": 0.48}


@pytest.mark.parametrize("method", sorted(FLOORS))
def test_oracle_accuracy_on_textured_scene(method):
    sc = syn.textured_scene(4, 160, 120)
    mask = np.ones((120, 160), np.uint8)
    mask[:20, :40] = 0
    depth, plane, score, nghbr = do.estimate(sc.K, sc.R, sc.t, list(sc.gray), mask, method, 7, 100, 3, 5.0, 3.0, 30.0)
    true = sc.depth[0]
    inner = np.zeros_like(mask, bool)
    inner[3:-3, 3:-3] = True
    sel = inner & (mask > 0) & ~sc.flat[0] & (true > 0) & (true < 30)
    frac = (np.abs(depth - true) < 0.01 * true)[sel].mean()
    assert frac >= FLOORS[method], frac
    if method != "BRUTE_FORCE":
        assert (depth[mask == 0] == 0).all()
        flat = cv2.erode(sc.flat[0].astype(np.uint8), np.ones((7, 7), np.uint8)) > 0
        assert flat.any() and (depth[flat] == 0).all()
