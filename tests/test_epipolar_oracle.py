"""Pins the numpy restatement of the guided-matching epipolar mask (`oracle/match_oracle.py:epipolar_mask`):
the reference's own known-answer test for geometry::EpipolarAngleTwoBearingsMany, Eigen's zero-norm semantics,
and an element-by-element restatement of triangulation.cc:195-219."""
import math

import numpy as np

from oracle import match_oracle as mo


def two_cams_many_points():
    """TwoCamsManyPointsFixture (opensfm/src/geometry/test/triangulation_test.cc:157-178): two points seen by two
    cameras, rotation_1_2 = AngleAxis(0.1, Y), translation_1_2 = (-1, 2, 0.2)."""
    pts = np.array([[0.0, 0.0, 1.0], [1.0, 2.0, 3.0]])
    c, s = math.cos(0.1), math.sin(0.1)
    R = np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
    t = np.array([-1.0, 2.0, 0.2])
    b1 = pts / np.linalg.norm(pts, axis=1, keepdims=True)
    b2 = (pts - t) @ R             # rows of R^T (p - t)
    b2 /= np.linalg.norm(b2, axis=1, keepdims=True)
    return b1, b2, R, t


def _normalized(v):
    z = v[0] * v[0] + v[1] * v[1] + v[2] * v[2]
    return [x / math.sqrt(z) for x in v] if z > 0.0 else list(v)


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def angles_elementwise(b1, b2, R, t):
    """triangulation.cc:195-219 one element at a time, with Eigen's `normalized()` (Dot.h: `if (z > 0) return
    n / sqrt(z); else return n;`), on the float32 bearings matching.py:860-861 passes."""
    b1 = np.asarray(b1, np.float32).astype(np.float64).tolist()
    b2 = np.asarray(b2, np.float32).astype(np.float64).tolist()
    R = np.asarray(R, np.float64).reshape(3, 3).tolist()
    tn = _normalized([float(x) for x in np.asarray(t, np.float64).reshape(3)])
    b2w = [[_dot(R[r], b) for r in range(3)] for b in b2]
    e1 = [_normalized(_cross(tn, b)) for b in b1]
    e2 = [_normalized(_cross(tn, b)) for b in b2w]
    out = np.empty((len(b1), len(b2)))
    for i in range(len(b1)):
        for j in range(len(b2)):
            sym = (abs(_dot(e1[i], b2w[j])) + abs(_dot(b1[i], e2[j]))) / 2.0
            out[i, j] = math.pi / 2.0 - math.acos(sym) if sym <= 1.0 else math.nan
    return out


def test_reference_known_answer_two_cams_many_points():
    """triangulation_test.cc:327-341: angles(i, i) < 1e-6, every other angle > 1e-6 -- so the mask at threshold
    1e-6 is the identity."""
    b1, b2, R, t = two_cams_many_points()
    ang = mo.epipolar_angles(b1, b2, R, t)
    assert ang.shape == (2, 2)
    assert np.all(np.diag(ang) < 1e-6)
    assert np.all(ang[~np.eye(2, dtype=bool)] > 1e-6)
    assert np.array_equal(mo.epipolar_mask(b1, b2, R, t, 1e-6), np.eye(2, dtype=bool))


def test_zero_translation_keeps_every_pair_like_eigen():
    """t = 0: Eigen's normalized() returns the zero vector, so every epipolar vector is 0, symmetric_epi = 0 and the
    angle is 0 everywhere: the mask is all true for any positive threshold (unguided matching), all false at 0."""
    rng = np.random.RandomState(1)
    b1 = rng.normal(size=(40, 3)); b1 /= np.linalg.norm(b1, axis=1, keepdims=True)
    b2 = rng.normal(size=(30, 3)); b2 /= np.linalg.norm(b2, axis=1, keepdims=True)
    R = np.eye(3)
    ang = mo.epipolar_angles(b1, b2, R, np.zeros(3))
    assert np.array_equal(ang, np.zeros((40, 30)))
    for thr in (1e-9, 0.006, 2.0):
        assert mo.epipolar_mask(b1, b2, R, np.zeros(3), thr).all()
    assert not mo.epipolar_mask(b1, b2, R, np.zeros(3), 0.0).any()


def test_bearing_parallel_to_translation_gives_a_zero_epipolar_vector():
    """A bearing exactly along +-t: t^ x b = 0 stays 0, so its row (column) of symmetric_epi keeps only the other
    term, |b1_i . e2_j| / 2 (|e1_i . R b2_j| / 2).  e2_j is perpendicular to t, so that term is 0 too: the angle is
    0 -- finite, not NaN -- and any positive threshold keeps the bearing against every other."""
    rng = np.random.RandomState(2)
    b1 = rng.normal(size=(12, 3)); b1 /= np.linalg.norm(b1, axis=1, keepdims=True)
    b2 = rng.normal(size=(9, 3)); b2 /= np.linalg.norm(b2, axis=1, keepdims=True)
    t = np.array([0.0, 0.0, 2.5])
    b1[3] = [0.0, 0.0, 1.0]
    b1[7] = [0.0, 0.0, -1.0]
    b2[4] = [0.0, 0.0, 1.0]          # R = I: R b2 is parallel to t as well
    sym = mo.epipolar_sym(b1, b2, np.eye(3), t)
    assert np.isfinite(sym).all()
    e2 = np.cross([0.0, 0.0, 1.0], b2.astype(np.float32).astype(np.float64))
    e2 = e2 / np.where(np.linalg.norm(e2, axis=1, keepdims=True) > 0, np.linalg.norm(e2, axis=1, keepdims=True), 1)
    want_row = np.abs(b1[3].astype(np.float32).astype(np.float64) @ e2.T) / 2.0
    assert np.allclose(sym[3], want_row, rtol=0, atol=1e-15)
    assert np.array_equal(sym[[3, 7]], np.zeros((2, 9))) and np.array_equal(sym[:, 4], np.zeros(12))
    assert mo.epipolar_mask(b1, b2, np.eye(3), t, 1e-9)[[3, 7]].all()
    # rows parallel to t and the column parallel to t meet at an element where both terms vanish
    assert sym[3, 4] == 0.0 and sym[7, 4] == 0.0
    assert np.allclose(mo.epipolar_angles(b1, b2, np.eye(3), t), angles_elementwise(b1, b2, np.eye(3), t),
                       rtol=0, atol=1e-15)


def test_vectorised_restatement_equals_the_elementwise_one():
    """Random poses and bearings over the whole sphere, thresholds on both sides of pi/2: the numpy mask equals the
    element-by-element restatement wherever the fp64 angle is not within 1e-12 of the threshold (the two sum in
    different orders)."""
    rng = np.random.RandomState(3)
    for trial in range(4):
        b1 = rng.normal(size=(60, 3)); b1 /= np.linalg.norm(b1, axis=1, keepdims=True)
        b2 = rng.normal(size=(50, 3)); b2 /= np.linalg.norm(b2, axis=1, keepdims=True)
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        t = rng.normal(size=3) * 3.0
        ref = angles_elementwise(b1, b2, q, t)
        got = mo.epipolar_angles(b1, b2, q, t)
        fin = np.isfinite(ref)
        assert np.array_equal(fin, np.isfinite(got))
        assert np.allclose(got[fin], ref[fin], rtol=0, atol=1e-12)
        for thr in (1e-6, 0.006, 0.5, np.pi / 2 - 1e-9, np.pi / 2, 2.0, -0.01):
            with np.errstate(invalid="ignore"):
                want = ref < thr
            keep = ~(np.abs(ref - thr) < 1e-12)
            assert np.array_equal(mo.epipolar_mask(b1, b2, q, t, thr)[keep], want[keep])


def test_threshold_beyond_half_pi_keeps_every_finite_angle():
    """The angle is at most pi/2, so past pi/2 the reference keeps every element whose symmetric_epi is <= 1."""
    rng = np.random.RandomState(4)
    b1 = rng.normal(size=(300, 3)); b1 /= np.linalg.norm(b1, axis=1, keepdims=True)
    b2 = rng.normal(size=(300, 3)); b2 /= np.linalg.norm(b2, axis=1, keepdims=True)
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    t = np.array([0.3, -1.0, 0.4])
    sym = mo.epipolar_sym(b1, b2, q, t)
    assert np.array_equal(mo.epipolar_mask(b1, b2, q, t, 2.0), sym <= 1.0)
    # sin(2.0) < 1: a test in sine space against sin(threshold) would drop every element above it
    assert ((sym > math.sin(2.0)) & (sym <= 1.0)).sum() > 1000
