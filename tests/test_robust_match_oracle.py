"""oracle/robust_match_oracle.py on known answers, and the host side of matching.robust_match: the small-input rule
of robust_match_calibrated, the dispatch between the fundamental and the calibrated branch, and the fundamental
branch against cv2 itself.  No GPU."""
import cv2
import numpy as np
import pytest

import relative_pose_cases as C
from opensfm_b200 import matching
from opensfm_b200 import synthetic as syn
from oracle import robust_match_oracle as rmo

THRESHOLD = 0.004            # robust_matching_calib_threshold, OpenSfM's default
CONFIG = {"robust_matching_calib_threshold": THRESHOLD, "robust_matching_threshold": 0.004,
          "five_point_refine_match_iterations": 10}


def true_pose(sc, s: int, o: int) -> np.ndarray:
    """lo_model [R | t] (x2 = R x1 + t, |t| = 1) of cameras s and o of a cube scene."""
    R = sc.R_wc[o] @ sc.R_wc[s].T
    t = sc.R_wc[o] @ (sc.origins[s] - sc.origins[o])
    return np.column_stack([R, t / np.linalg.norm(t)])


def test_outliers_are_removed_and_true_rows_kept():
    """Cube-scene pairs, 2e-4 bearing noise, 30 % of the rows replaced by random directions: the final inliers hold
    at least 97 % of the true rows and at most 2 outlier rows (a random direction can fall within the threshold of
    its epipolar line)."""
    sc = syn.cube_scene(6, 400, seed=21, with_descriptors=False)
    rng = np.random.RandomState(22)
    for s, o in ((0, 1), (2, 4), (3, 5)):
        X = sc.points[np.sort(rng.choice(400, 150, replace=False))]
        b1 = C.unit(C.unit((X - sc.origins[s]) @ sc.R_wc[s].T) + 2e-4 * rng.randn(150, 3))
        b2 = C.unit(C.unit((X - sc.origins[o]) @ sc.R_wc[o].T) + 2e-4 * rng.randn(150, 3))
        bad = rng.rand(150) < 0.3
        b2[bad] = C.unit(np.column_stack([rng.uniform(-0.6, 0.6, (int(bad.sum()), 2)), np.ones(int(bad.sum()))]))
        r = rmo.robust_match_calibrated(b1, b2, THRESHOLD)
        assert r.empty_round is None and r.counts[-1] == r.mask.sum()
        kept_true = int((r.mask & ~bad).sum())
        assert kept_true >= 0.97 * int((~bad).sum()), (s, o, kept_true, int((~bad).sum()))
        assert int((r.mask & bad).sum()) <= 2, (s, o)


def test_pair_emptied_by_the_2x_round():
    """Ten rows displaced by 0.024 rad in the second image and thirty random ones: the 4x round (chord 0.016) keeps
    8 or more rows, the 2x round after its refinement fewer, so the pair ends empty there, with no pose and no
    inliers, whatever the 1x round would have kept."""
    sc = syn.cube_scene(4, 400, seed=3, with_descriptors=False)
    rng = np.random.RandomState(3)
    X = sc.points[:40]
    b1 = C.unit((X - sc.origins[0]) @ sc.R_wc[0].T)
    b2 = C.unit((X - sc.origins[1]) @ sc.R_wc[1].T)
    b2[:10] = C.unit(b2[:10] + 0.024 * C.unit(np.cross(b2[:10], rng.randn(10, 3))))
    b2[10:] = C.unit(np.column_stack([rng.uniform(-0.6, 0.6, (30, 2)), np.ones(30)]))
    r = rmo.robust_match(b1, b2, true_pose(sc, 0, 1), THRESHOLD)
    assert r.counts[0] >= 8 and 0 <= r.counts[1] < 8 and r.counts[2:] == [-1, -1], r.counts
    assert r.empty_round == 1 and np.isnan(r.pose).all() and not r.mask.any()
    assert r.margins.chord > 1e-6


def test_fewer_than_8_matches_return_an_empty_array():
    p = np.random.RandomState(0).rand(20, 3)
    m = np.column_stack([np.arange(7), np.arange(7)])
    got = matching.robust_match_calibrated(p, p, None, None, m, CONFIG)
    assert isinstance(got, np.ndarray) and got.shape == (0,)
    with pytest.raises(ValueError, match="at least 8 rows"):
        rmo.robust_match_calibrated(p[:7], p[:7], THRESHOLD)


class FakeCamera:
    def __init__(self, projection_type: str, k1: float = 0.0, k2: float = 0.0):
        self.projection_type, self.k1, self.k2 = projection_type, k1, k2


@pytest.mark.parametrize("cam1,cam2,fundamental", [
    (FakeCamera("perspective"), FakeCamera("perspective"), True),
    (FakeCamera("brown"), FakeCamera("perspective"), True),
    (FakeCamera("brown"), FakeCamera("brown"), True),
    (FakeCamera("perspective", k1=-0.1), FakeCamera("perspective"), False),
    (FakeCamera("perspective"), FakeCamera("brown", k2=0.01), False),
    (FakeCamera("brown", k1=1e-9), FakeCamera("brown"), False),
    (FakeCamera("fisheye"), FakeCamera("perspective"), False),
    (FakeCamera("perspective"), FakeCamera("spherical"), False),
    (FakeCamera("fisheye_opencv"), FakeCamera("fisheye_opencv"), False),
])
def test_dispatch(monkeypatch, cam1, cam2, fundamental):
    calls = []
    monkeypatch.setattr(matching, "robust_match_fundamental",
                        lambda p1, p2, m, config: calls.append("fundamental") or (None, m[:1]))
    monkeypatch.setattr(matching, "robust_match_calibrated",
                        lambda p1, p2, c1, c2, m, config: calls.append("calibrated") or m[:2])
    m = np.column_stack([np.arange(30), np.arange(30)])
    got = matching.robust_match(None, None, cam1, cam2, m, CONFIG)
    assert calls == ["fundamental" if fundamental else "calibrated"]
    assert len(got) == (1 if fundamental else 2)


def test_fundamental_branch_is_cv2():
    """robust_match_fundamental keeps exactly the matches cv2.findFundamentalMat(FM_RANSAC, 0.004, 0.9999) marks."""
    sc = syn.cube_scene(3, 300, seed=4, with_descriptors=False)
    rng = np.random.RandomState(5)
    proj = [syn.project_perspective((sc.points - sc.origins[s]) @ sc.R_wc[s].T, 0.0, 0.0, 0.9) for s in (0, 1)]
    p1 = np.column_stack([proj[0], np.ones(300)])
    p2 = np.column_stack([proj[1] + rng.normal(0, 5e-4, (300, 2)), np.ones(300)])
    m = np.column_stack([rng.permutation(300), np.arange(300)])
    m[:200, 0] = np.arange(200)                      # 200 true matches, 100 wrong ones
    F, got = matching.robust_match_fundamental(p1, p2, m, CONFIG)
    _, mask = cv2.findFundamentalMat(p1[m[:, 0], :2].copy(), p2[m[:, 1], :2].copy(), cv2.FM_RANSAC, 0.004, 0.9999)
    assert np.array_equal(got, m[mask.ravel().astype(bool)])
    assert F.shape == (3, 3) and len(got) >= 190
    assert np.array_equal(matching.robust_match(p1, p2, FakeCamera("perspective"), FakeCamera("brown"), m, CONFIG),
                          got)
    F, got = matching.robust_match_fundamental(p1, p2, m[:7], CONFIG)
    assert len(got) == 0


def test_radial_camera_inverts_the_cube_projection():
    """The GPU tests' camera for the cube scenes: its bearings reproject onto synthetic.project_perspective."""
    import robust_match_cases as RC

    rng = np.random.RandomState(6)
    pc = np.column_stack([rng.uniform(-0.3, 0.3, (500, 2)), np.ones(500)]) * rng.uniform(1.0, 4.0, (500, 1))
    p = syn.project_perspective(pc, -0.1, 0.01, 0.9)
    b = RC.RadialCamera(-0.1, 0.01, 0.9).pixel_bearing_many(p)
    assert np.abs(b - pc / np.linalg.norm(pc, axis=1)[:, None]).max() < 1e-12
