"""oracle/absolute_pose_oracle.py and the resection drop-ins on the CPU: OpenSfM's known answers for the P3P solver,
Lu's iteration and the absolute-pose RANSAC (opensfm/test/test_robust.py, test_multiview.py, with their tolerances),
the quartic against numpy.roots, the product's host-compiled solvers (opensfm_b200/csrc/absolute_pose.cuh through
tests/cpu_harness/absolute_pose_host.cpp) against the oracle, and the map-side parts of resection:
reconstructed_points_for_images, add_shot and exif_to_metadata."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from opensfm_b200 import map_types as M
from opensfm_b200 import reconstruction as rec
from opensfm_b200 import synthetic as syn
from opensfm_b200 import tracking
from opensfm_b200 import types as T
from oracle import absolute_pose_oracle as ap

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpu_harness", "absolute_pose_host.cpp")
HDR = os.path.join(HERE, "..", "opensfm_b200", "csrc", "absolute_pose.cuh")
LIB = os.path.join(HERE, "cpu_harness", "_build", "libabsolute_pose_host.so")


@pytest.fixture(scope="module")
def hd():
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-o", LIB, SRC])
    return ctypes.CDLL(LIB)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def shot_rows(sc, s):
    """(unit bearings, world points) of shot s of a synthetic scene, from the true pose."""
    X = sc.points[sc.obs_point[sc.obs_shot == s]]
    b = (X - sc.origins[s]) @ sc.R_wc[s].T
    return b / np.linalg.norm(b, axis=1)[:, None], X


def true_pose(sc, s):
    return np.column_stack([sc.R_wc[s], -sc.R_wc[s] @ sc.origins[s]])


@pytest.fixture(scope="module")
def scene():
    return syn.cube_scene(20, 600, projection_noise=0.0, seed=5)


def test_absolute_pose_three_points(scene):
    """test_multiview.py's test_absolute_pose_three_points: some root within 1e-6 of the pose for all but 2 shots."""
    failed = 0
    for s in range(scene.num_shots):
        b, X = shot_rows(scene, s)
        models = ap.p3p(b[:3], X[:3])
        if not any(np.linalg.norm(m - true_pose(scene, s)) < 1e-6 for m in models):
            failed += 1
    assert failed <= 2


def test_absolute_pose_n_points(scene):
    for s in range(scene.num_shots):
        b, X = shot_rows(scene, s)
        assert np.linalg.norm(ap.lu_pose(b, X) - true_pose(scene, s)) < 1e-5, s


def test_outliers_absolute_pose_ransac():
    """test_robust.py's test_outliers_absolute_pose_ransac: 30 % outliers, inliers within 5 % of 70 %, lo_model within
    8e-2 of the pose."""
    sc = syn.cube_scene(4, 400, projection_noise=0.0, seed=11)
    rng = np.random.RandomState(3)
    for s in range(sc.num_shots):
        b, X = shot_rows(sc, s)
        n = len(b)
        bad = rng.permutation(n)[:int(0.3 * n)]
        b = b.copy()
        b[bad] = ap.normalize_rows(rng.randn(len(bad), 3))
        r = ap.ransac_absolute_pose(b, X, 0.01)
        assert np.isclose(r.ransac_inliers, 0.7 * n, rtol=0.05), (s, r.ransac_inliers, n)
        assert np.linalg.norm(r.lo_model - true_pose(sc, s)) < 8e-2


def test_quartic_against_numpy_roots(hd):
    rng = np.random.RandomState(0)
    for _ in range(200):
        roots = np.sort(rng.uniform(-1, 1, 4))
        coef = np.poly(roots)[::-1] * rng.uniform(0.5, 2.0)   # coef[k] of x^k
        got = np.sort(ap.solve_quartic(coef))
        got = np.sort([ap.refine_root(coef, x) for x in got])
        want = np.sort(np.roots(coef[::-1]).real)
        assert np.abs(got - want).max() < 1e-9, (got, want)
        out = np.zeros(4)
        assert hd.hd_solve_quartic(_p(np.ascontiguousarray(coef)), _p(out)) == 4
        assert np.abs(np.sort(out) - want).max() < 1e-9


def test_host_solvers_equal_oracle(hd, scene):
    """The header's P3P and Lu's iteration, compiled by g++, against the oracle on random samples of perturbed rows:
    to 1e-12 for at least 98 % of the models and within 1e-10 for all.  The rest differ by round-off (the oracle's
    numpy sums its 9 polar entries in another order) amplified by ill-conditioned samples."""
    rng = np.random.RandomState(1)
    diffs = []
    for s in range(scene.num_shots):
        b, X = shot_rows(scene, s)
        b = ap.normalize_rows(b + 1e-3 * rng.randn(*b.shape))
        for _ in range(10):
            idx = rng.choice(len(b), 3, replace=False)
            want = ap.p3p(b[idx], X[idx])
            out = np.zeros((4, 3, 4))
            nm = hd.hd_p3p(_p(np.ascontiguousarray(b[idx])), _p(np.ascontiguousarray(X[idx])), _p(out))
            assert nm == len(want)
            for m in range(nm):
                if np.isnan(want[m]).any():
                    assert np.isnan(out[m]).any()
                    continue
                diffs.append(np.abs(out[m] - want[m]).max() / max(1.0, np.abs(want[m]).max()))
            for k in (3, 5, 12):
                idx = rng.choice(len(b), k, replace=False)
                want = ap.lu_pose(b[idx], X[idx])
                out = np.zeros((3, 4))
                hd.hd_lu(k, _p(np.ascontiguousarray(b[idx])), _p(np.ascontiguousarray(X[idx])), _p(out))
                diffs.append(np.abs(out - want).max() / max(1.0, np.abs(want).max()))
    diffs = np.array(diffs)
    assert len(diffs) >= 500
    assert (diffs < 1e-12).mean() >= 0.98 and diffs.max() < 1e-10, (np.sort(diffs)[-10:])


# ---------------------------------------------------------------------------------------------------------------
# the map side
# ---------------------------------------------------------------------------------------------------------------
class Reference:
    def to_topocentric(self, lat, lon, alt):
        return 100.0 * lat, 100.0 * lon, alt


class Data:
    """The DataSet calls of resect: exif, rig assignments, reference, config."""

    def __init__(self, rigs=None, exif=None):
        self.config = {"use_altitude_tag": True, "triangulation_type": "FULL", "triangulation_threshold": 0.006,
                       "triangulation_min_ray_angle": 1.0, "triangulation_min_depth": 0.001,
                       "triangulation_refinement_iterations": 10}
        self._rigs = rigs or {}
        self._exif = exif or {}

    def load_exif(self, image):
        return dict(self._exif.get(image, {}), camera="cam")

    def load_rig_assignments(self):
        return self._rigs

    def load_reference(self):
        return Reference()


def test_exif_to_metadata_fills_the_reference_fields():
    exif = {"gps": {"latitude": 1.0, "longitude": 2.0, "altitude": 3e4, "dop": 0.0},
            "opk": {"omega": 0.1, "phi": 0.2, "kappa": 0.3}, "orientation": 6, "gravity_down": [0.0, 0.0, 1.0],
            "compass": {"angle": 30.0, "accuracy": 5.0}, "capture_time": 12.5, "skey": "seq"}
    m = rec.exif_to_metadata(exif, True, Reference())
    assert np.array_equal(m.gps_position.value, [100.0, 200.0, 1e4])
    assert m.gps_accuracy.value == 15.0
    assert np.array_equal(m.opk_angles.value, [0.1, 0.2, 0.3]) and m.opk_accuracy.value == 1.0
    assert m.orientation.value == 6 and isinstance(m.orientation.value, int)
    assert np.array_equal(m.gravity_down.value, [0.0, 0.0, 1.0])
    assert (m.compass_angle.value, m.compass_accuracy.value, m.capture_time.value) == (30.0, 5.0, 12.5)
    assert m.sequence_key.value == "seq"
    m = rec.exif_to_metadata({"gps": {"latitude": 1.0, "longitude": 2.0, "altitude": 7.0}}, False, Reference())
    assert np.array_equal(m.gps_position.value, [100.0, 200.0, 2.0]) and m.gps_accuracy.value == 15.0
    assert m.orientation.value == 1
    assert not (m.opk_angles.has_value or m.compass_angle.has_value or m.sequence_key.has_value)


class Camera:
    id = "cam"


def _pose(R, t):
    p = T.Pose()
    p.set_rotation_matrix(R)
    p.translation = np.asarray(t, dtype=np.float64)
    return p


def test_add_shot_without_and_with_rig():
    R = syn.angle_axis_to_rotation(np.array([0.1, -0.3, 0.2]))
    t = np.array([0.5, -1.0, 2.0])
    rigs = {"inst": [("a", "left"), ("b", "right")]}
    assignments = rec.rig_assignments_per_image(rigs)
    assert assignments["b"] == ("inst", "right", ["a", "b"])

    r = M.Reconstruction()
    r.add_camera(Camera())
    assert rec.add_shot(Data(rigs), r, assignments, "single", _pose(R, t)) == {"single"}
    shot = r.shots["single"]
    assert np.abs(shot.pose.get_rotation_matrix() - R).max() < 1e-12
    assert np.abs(shot.pose.translation - t).max() < 1e-12
    assert shot.metadata.orientation.value == 1

    r.add_rig_camera(M.RigCamera(_pose(syn.angle_axis_to_rotation(np.array([0.0, 0.2, 0.0])), [0.3, 0, 0]), "right"))
    r.add_rig_camera(M.RigCamera(T.Pose(), "left"))
    assert rec.add_shot(Data(rigs), r, assignments, "b", _pose(R, t)) == {"a", "b"}
    assert set(r.rig_instances["inst"].shots) == {"a", "b"}
    assert np.abs(r.shots["b"].pose.get_rotation_matrix() - R).max() < 1e-12
    assert np.abs(r.shots["b"].pose.translation - t).max() < 1e-12
    assert r.shots["a"].rig_camera_id == "left"


def cube_tracks_manager(sc):
    """A TracksManager of a synthetic scene's true tracks (one per point seen twice or more), made on the host."""
    order = np.lexsort((sc.obs_shot, sc.obs_point))
    pts, shots = sc.obs_point[order], sc.obs_shot[order]
    keep = np.isin(pts, np.nonzero(np.bincount(pts) >= 2)[0])
    pts, shots, order = pts[keep], shots[keep], order[keep]
    images = ["im%d" % s for s in range(sc.num_shots)]
    first = np.array([np.nonzero(sc.obs_shot == s)[0][0] for s in range(sc.num_shots)])
    feats = {images[s]: np.column_stack([sc.obs_xy[sc.obs_shot == s], sc.obs_sigma[sc.obs_shot == s]])
             for s in range(sc.num_shots)}
    colors = {im: np.zeros((len(f), 3), dtype=np.int32) for im, f in feats.items()}
    track = np.searchsorted(np.unique(pts), pts).astype(np.int32)
    track_start = np.searchsorted(track, np.arange(track.max() + 2)).astype(np.int64)
    return tracking.TracksManager(None, images, track, shots.astype(np.int32), (order - first[shots]).astype(np.int32),
                                  track_start, feats, colors, {}, {}, None, True, 1.0, 0.0)


def test_reconstructed_points_for_images():
    sc = syn.cube_scene(8, 300, seed=4, max_obs_per_point=4)
    tm = cube_tracks_manager(sc)
    r = M.Reconstruction()
    r.add_camera(Camera())
    r.create_shot("im0", "cam", T.Pose())
    rng = np.random.RandomState(0)
    for t in rng.choice(tm.num_tracks(), tm.num_tracks() // 3, replace=False):
        r.create_point(str(t), np.zeros(3))
    got = rec.reconstructed_points_for_images(tm, r, set(tm.images))
    want = []
    for pos, im in enumerate(tm.images):
        if im in r.shots:
            continue
        want.append((im, sum(1 for t in tm.get_shot_observations(im) if t in r.points), pos))
    want.sort(key=lambda x: (-x[1], x[2]))
    assert got == [(im, n) for im, n, _ in want]
    assert len(got) == 7 and len(set(n for _, n in got)) > 1
