"""oracle/two_view_oracle.py and the host side of the two-view stage (opensfm_b200.relative_pose.plane_motions /
plane_motion): glibc's rand() and the picked rows, RelativePoseCost's Jacobian, the refinement's fixed point on
noise-free pairs, the shared TinySolver loop, the plane decomposition against the reference's first motion (kept in
tests/golden/plane_motion_reference.npz) and the decision rules.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest

import relative_pose_cases as C
from opensfm_b200 import relative_pose as rp
from opensfm_b200 import synthetic as syn
from oracle import triangulation_oracle as tro
from oracle import two_view_oracle as tv

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "plane_motion_reference.npz")


def test_glibc_rand_restatement():
    libc = ctypes.CDLL("libc.so.6")
    libc.srand(42)
    want = [libc.rand() for _ in range(1000)]
    assert tv.glibc_rand(42, 1000) == want
    assert max(want[:100]) == 2145078185


@pytest.mark.parametrize("count", [6, 7, 100, 101, 999, 3000, 16777215])
def test_picked_positions(count):
    fr = np.array(tv.glibc_rand(42, 100), dtype=np.float32) / np.float32(2147483647)
    want = [int(np.float32(f) * np.float32(count)) for f in fr]
    got = tv.picked_positions(count)
    assert got.tolist() == want and got.max() < count and got.min() >= 0


def _pair(seed, n=60, rot=0.2, noise=0.0):
    rng = np.random.RandomState(seed)
    X = rng.uniform(-1, 1, (n, 3)) + [0, 0, 5]
    R = syn.angle_axis_to_rotation(rng.randn(3) * rot)
    t = rng.randn(3)
    t /= np.linalg.norm(t)
    # B = [R | t] maps the second camera to the first: the second camera is at t, its bearings R^T (X - t)
    x = C.unit(X + noise * rng.randn(n, 3))
    y = C.unit((X - t) @ R + noise * rng.randn(n, 3))
    return x, y, np.column_stack([R, t])


@pytest.mark.parametrize("small", [False, True])
def test_cost_jacobian_against_central_differences(small):
    """Both AngleAxisRotatePoint branches: |aa|^2 above and below DBL_EPSILON."""
    x, y, B = _pair(1, 40)
    p = tv.refine_parameters(B)
    if small:
        p[:3] = [3e-9, -5e-9, 4e-9]
        assert p[:3] @ p[:3] <= tv.DBL_EPSILON
    f = tv.relative_pose_cost(p, x, y)
    assert f.v.shape == (41,) and f.d.shape == (41, 6)
    h = 1e-7 if not small else 1e-9
    for k in range(6):
        e = np.zeros(6)
        e[k] = h
        if small and k < 3:
            # stay on the first-order branch: the difference quotient of that branch
            num = (tv.relative_pose_cost(p + e, x, y).v - tv.relative_pose_cost(p - e, x, y).v) / (2 * h)
        else:
            num = (tv.relative_pose_cost(p + e, x, y).v - tv.relative_pose_cost(p - e, x, y).v) / (2 * h)
        assert np.abs(num - f.d[:, k]).max() < 1e-6 * max(1.0, np.abs(f.d[:, k]).max()), k


def test_failed_midpoint_has_unit_residual_and_no_derivative():
    x, y, B = _pair(2, 10)
    y = x.copy()
    B = np.column_stack([np.eye(3), [1.0, 0.0, 0.0]])
    x[3] = [1.0, 0.0, 0.0]
    y[3] = [1.0, 0.0, 0.0]
    f = tv.relative_pose_cost(tv.refine_parameters(B), x, y)
    assert f.v[3] == 1.0 and not f.d[3].any()


@pytest.mark.parametrize("seed", [3, 4, 5, 6])
def test_refinement_on_noise_free_pairs(seed):
    """The reference's test_relative_pose_refinement on noise-free rows.  The true pose is a fixed point to 1e-9.
    From a perturbed pose the cost falls by more than 4 orders and the pose lands within the reference's 0.18 and
    closer than it started; not to 1e-9, because the residuals 1 - cos are quadratic in the angular error, so the
    cost (their squares) is quartic and TinySolver's cost and gradient stops end about 1e-3 from the truth."""
    x, y, B = _pair(seed, 80)
    assert tv.bearing_inliers(B, x, y, 0.004).all()
    assert np.abs(tv.refine(B, x, y, np.arange(len(x)), 1000) - B).max() < 1e-9
    rng = np.random.RandomState(seed + 100)
    P = B.copy()
    P[:, :3] = syn.angle_axis_to_rotation(rng.randn(3) * 0.01) @ B[:, :3]
    P[:, 3] = B[:, 3] + 0.01 * rng.randn(3)
    got = tv.refine(P, x, y, np.arange(len(x)), 1000)
    rows = np.arange(len(x))[tv.picked_positions(len(x))]

    def cost(M):
        f = tv.relative_pose_cost(tv.refine_parameters(M), x[rows], y[rows]).v
        return f @ f

    assert cost(got) < 1e-4 * cost(P)
    assert np.linalg.norm(got - B) < min(0.18, np.linalg.norm(P - B))


def test_refinement_parametrisation_round_trip():
    for seed in range(5):
        _, _, B = _pair(seed, 5, rot=1.0 + seed)
        assert np.abs(tv.refine_pose(tv.refine_parameters(B)) - B).max() < 1e-13
    R = np.diag([1.0, -1.0, -1.0])   # trace -1: the non-trace quaternion branch, angle pi
    assert np.allclose(tv.rotation_to_angle_axis(R), [np.pi, 0, 0])
    assert np.allclose(tv.angle_axis_to_rotation(np.array([1e-9, 0, 0])), np.eye(3) + [[0, 0, 0], [0, 0, -1e-9],
                                                                                          [0, 1e-9, 0]])


def test_tiny_solver_is_triangulation_refine():
    """The generic loop returns triangulation_oracle.refine's points bit for bit on the bearing cost."""
    rng = np.random.RandomState(7)
    for _ in range(10):
        X = rng.randn(3) * 3
        c = rng.randn(4, 3)
        b = C.unit(X - c + 0.01 * rng.randn(4, 3))
        x0 = X + 0.1 * rng.randn(3)

        def res(p, jac):
            return tro.bearing_cost(p, c, b, jacobian=True) if jac else (tro.bearing_cost(p, c, b), None)

        assert np.array_equal(tv.tiny_solver(res, x0, 10), tro.refine(c, b, x0, 10))


def test_bearing_inliers_match_reference_formula():
    x, y, B = _pair(8, 100, noise=1e-3)
    y[:30] = C.unit(np.random.RandomState(0).randn(30, 3))
    R, t = B[:, :3], B[:, 3]
    # compute_inliers_bearings, written out with an explicit 2 x 2 solve
    want = np.zeros(len(x), bool)
    for i in range(len(x)):
        by = R @ y[i]
        A = np.array([[x[i] @ x[i], -(x[i] @ by)], [x[i] @ by, -(by @ by)]])
        lam = np.linalg.solve(A, [t @ x[i], t @ by])
        X = 0.5 * (lam[0] * x[i] + t + lam[1] * by)
        b2 = R.T @ (X - t)
        want[i] = (np.linalg.norm(X / np.linalg.norm(X) - x[i]) < 0.004 and
                   np.linalg.norm(b2 / np.linalg.norm(b2) - y[i]) < 0.004)
    got = tv.bearing_inliers(B, x, y, 0.004)
    assert np.array_equal(got, want) and 50 < got.sum() < 71


# ---------------------------------------------------------------------------------------------------------------
# the plane motion
# ---------------------------------------------------------------------------------------------------------------
def test_plane_motions_satisfy_the_decomposition():
    g = np.load(GOLDEN)
    for H in g["H"]:
        ms = rp.plane_motions(H)
        if ms is None:
            continue
        assert len(ms) == 8
        for R, t, n, d in ms:
            assert np.abs(R @ R.T - np.eye(3)).max() < 1e-12 and abs(np.linalg.det(R) - 1) < 1e-12
            assert np.abs(d * R + np.outer(t, n) - H).max() < 1e-12 * np.abs(H).max()


def test_plane_motion_zero_equals_reference():
    g = np.load(GOLDEN)
    none = 0
    for H, R, t in zip(g["H"], g["R"], g["t"]):
        ms = rp.plane_motions(H)
        if np.isnan(t).any():
            assert ms is None
            none += 1
            continue
        assert np.abs(ms[0][0] - R).max() < 1e-12 and np.abs(ms[0][1] - t).max() < 1e-12 * max(1, np.abs(t).max())
    assert none == 2 and len(g["H"]) >= 50
    assert rp.plane_motions(None) is None


def test_plane_result_is_motion_zero_even_when_another_has_more_inliers():
    """The reference's argmax over a map object is 0: motion 0 is kept whatever the inlier counts.  Among planar
    pairs of random motions, those where another motion has more inliers still get motion 0."""
    import cv2

    found = 0
    for seed in range(12):
        rng = np.random.RandomState(seed)
        X = np.column_stack([rng.uniform(-1, 1, (200, 2)), np.zeros(200)]) + [0, 0, 4]
        R = syn.angle_axis_to_rotation(rng.randn(3) * 0.2)
        t = rng.randn(3) * 0.5
        b1 = C.unit(X)
        b2 = C.unit((X - t) @ R)
        H, _ = cv2.findHomography(b1[:, :2] / b1[:, 2:], b2[:, :2] / b2[:, 2:], cv2.RANSAC, 0.004)
        ms = rp.plane_motions(H)
        if ms is None:
            continue
        counts = [tv.bearing_inliers(np.column_stack([Rm.T, -(Rm.T @ tm)]), b1, b2, 0.004).sum()
                  for Rm, tm, _, _ in ms]
        if max(counts) > counts[0]:
            found += 1
            assert np.array_equal(rp.plane_motion(b1, b2, 0.004), np.column_stack([ms[0][0], ms[0][1]]))
    assert found >= 2


def test_plane_motion_without_homography():
    b = C.unit(np.random.RandomState(1).randn(3, 3) + [0, 0, 3])
    assert np.isnan(rp.plane_motion(np.vstack([b, b]), np.vstack([b, b]), 0.004)).all()


# ---------------------------------------------------------------------------------------------------------------
# decisions
# ---------------------------------------------------------------------------------------------------------------
def test_necker_rule():
    assert tv.necker([100, 97], 0.95) == -1            # un-decidable: 0.97 > 0.95
    assert tv.necker([100, 90], 0.95) == 0
    assert tv.necker([90, 100], 0.95) == 1
    assert tv.necker([50, 50], 1.0) == 1               # a tie reaches the rule only at ratio >= 1: transposed wins
    assert tv.necker([50, 50], 0.95) == -1
    assert tv.necker([5, 50], 0.95) == 1               # at most 5 inliers: dropped
    assert tv.necker([6], 1.0) == 0 and tv.necker([5], 1.0) == -1
    assert tv.necker([5, 5], 1.0) == -1


def test_method_rule():
    assert tv.decide(40, 40) == "plane_based"          # equal counts: the plane wins
    assert tv.decide(41, 40) == "5_point"
    assert tv.decide(41, None) == "5_point"
    assert tv.decide(None, 0) == "plane_based"
    assert tv.decide(None, None) is None


def test_two_view_oracle_on_a_planar_pair():
    """H is None for three distinct rows repeated; the plane result is then absent and a degenerate pose gives no
    5-point result."""
    x, y, B = _pair(9, 80, noise=1e-4)
    lo = np.column_stack([B[:, :3].T, -(B[:, :3].T @ B[:, 3])])
    r = tv.two_view(x, y, lo, np.full((3, 4), np.nan), 0.004, 1000)
    assert r.method == "5_point" and r.chosen == 0 and r.counts[2] == 0 and r.counts[0] == 80
    assert np.abs(r.pose[0] - B).max() < 1e-3
    r = tv.two_view(x, y, lo, np.full((3, 4), np.nan), 0.004, 1000, check_reversal=True, reversal_ratio=1.0)
    assert r.chosen == 0 and r.counts[1] < r.counts[0]
    r = tv.two_view(x[:5], y[:5], lo, np.full((3, 4), np.nan), 0.004, 1000)
    assert r.method is None and r.chosen == -1 and not r.mask_5pt.any()
