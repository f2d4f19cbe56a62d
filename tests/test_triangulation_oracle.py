"""The triangulation oracle (oracle/triangulation_oracle.py) on the CPU: the reference's known answers
(opensfm/test/test_triangulation.py:7-102, 138-173), its refined point against an independent least-squares solve,
and the statuses of the synthetic scenes the GPU tests use."""
import numpy as np
import pytest
from scipy.optimize import least_squares

import triangulation_cases as tc
from opensfm_b200 import triangulation
from oracle import triangulation_oracle as to


def _unit(x):
    return np.array(x, dtype=np.float64) / np.linalg.norm(x)


@pytest.mark.parametrize("case", tc.known_answers()["tracks"], ids=lambda c: c["name"])
def test_track_triangulator_known_answers(case):
    camera = tc.SphericalCamera()
    rec = tc.reconstruction_from_json(case, camera)
    tm = tc.DictTracksManager()
    for s, xy in case["observations"].items():
        tm.add_observation(s, "1", tc.map_types.Observation(xy[0], xy[1], 1.0, 0, 0, 0, 0 if s == "im1" else 1))
    o = case["options"]
    to.triangulate_track(tm, rec, "1", o["reproj_threshold"], o["min_ray_angle_degrees"], o["min_depth"],
                         o["iterations"])
    if case["expected_point"] is None:
        assert not rec.points
    else:
        assert "1" in rec.points
        assert np.allclose(rec.points["1"].coordinates, case["expected_point"])
        assert len(rec.points["1"].get_observations()) == case["expected_observations"]


@pytest.mark.parametrize("case", tc.known_answers()["bearings_midpoint"], ids=lambda c: c["name"])
def test_triangulate_bearings_midpoint_known_answers(case):
    bearings = np.array([_unit(b) for b in case["bearings"]])
    status, X, _ = to.triangulate_bearings_midpoint(np.array(case["centers"]), bearings,
                                                     2 * [case["max_reprojection"]],
                                                     np.radians(case["min_ray_angle_degrees"]), case["min_depth"])
    if case["expected"] is None:
        assert status != to.OK
    else:
        assert status == to.OK
        assert np.allclose(X, case["expected"])


def _rays(seed, n, noise):
    rng = np.random.RandomState(seed)
    X = rng.uniform(-1, 1, 3)
    centers = X + 3.0 * rng.normal(size=(n, 3))
    b = X - centers + noise * rng.normal(size=(n, 3))
    return centers, b / np.linalg.norm(b, axis=1)[:, None]


@pytest.mark.parametrize("seed,n", [(0, 2), (1, 3), (2, 10), (3, 40)])
def test_refined_point_is_the_minimiser_of_the_bearing_cost(seed, n):
    centers, bearings = _rays(seed, n, 0.002)
    status, X, _ = to.triangulate_bearings_midpoint(centers, bearings, [0.1] * n, np.radians(1.0), 1e-3)
    assert status == to.OK
    refined = to.refine(centers, bearings, X, 10)
    f, J = to.bearing_cost(refined, centers, bearings, jacobian=True)
    f0, J0 = to.bearing_cost(X, centers, bearings, jacobian=True)
    # the gradient J^T f five orders of magnitude below its size at the midpoint
    g, g0 = np.abs(J.T @ f).max(), np.abs(J0.T @ f0).max()
    assert g <= 1e-5 * g0, (g, g0)
    ref = least_squares(lambda x: to.bearing_cost(x, centers, bearings), X, method="lm", xtol=1e-15, ftol=1e-15,
                        gtol=1e-15).x
    # relative to the point's distance to its cameras; TinySolver stops once its Jacobi-scaled gradient is below
    # 1e-10, which leaves the point up to a few 1e-10 of that distance from the minimiser
    assert np.abs(refined - ref).max() <= 1e-9 * np.linalg.norm(ref - centers, axis=1).mean()


def test_angle_between_vectors_edges():
    assert to.angle_between_vectors(np.array([1.0, 0, 0]), np.array([2.0, 0, 0])) == 0.0
    assert to.angle_between_vectors(np.array([1.0, 0, 0]), np.array([-1.0, 0, 0])) == 0.0   # |cos| >= 1
    assert np.isnan(to.angle_between_vectors(np.zeros(3), np.array([1.0, 0, 0])))
    assert to.angle_between_vectors(np.array([1.0, 0, 0]), np.array([0, 1.0, 0])) == pytest.approx(np.pi / 2)


def test_synthetic_scenes_reach_every_status():
    """The cube case of the GPU tests, on the oracle: every status occurs, and the triangulated points are close to
    the scene's points."""
    sc, camera, in_rec = tc.cube_case()
    rng = np.random.RandomState(0)
    rec = sc.reconstruction(camera, in_rec, rng, 1e-4, 1e-3)
    statuses = []
    for obs in sc.points:
        kept = [s for s in sorted(obs) if s in rec.shots]
        c = np.array([rec.shots[s].pose.get_origin() for s in kept]).reshape(-1, 3)
        b = np.array([rec.shots[s].pose.get_rotation_matrix().T @ camera.pixel_bearing(obs[s]) for s in kept])
        status, _, _ = to.triangulate_rays(c, b.reshape(-1, 3), 0.006, np.radians(1.0), 0.001, 10)
        statuses.append(status)
    counts = np.bincount(statuses, minlength=5)
    assert all(counts[1:] > 0), counts


def test_robust_triangulation_is_refused_and_other_types_do_nothing():
    """No device work is reached: ROBUST raises before anything changes, any other type triangulates nothing
    (retriangulate still clears the points, as the reference does)."""
    rec = tc.map_types.Reconstruction()
    rec.create_point("1", [0.0, 0.0, 1.0])
    with pytest.raises(NotImplementedError, match="ROBUST"):
        triangulation.triangulate_shot_features(None, rec, ["im1"], dict(tc.CONFIG, triangulation_type="ROBUST"))
    with pytest.raises(NotImplementedError, match="ROBUST"):
        triangulation.retriangulate(None, rec, dict(tc.CONFIG, triangulation_type="ROBUST"))
    assert list(rec.points) == ["1"]
    triangulation.triangulate_shot_features(None, rec, ["im1"], dict(tc.CONFIG, triangulation_type="DLT"))
    report = triangulation.retriangulate(None, rec, dict(tc.CONFIG, triangulation_type="DLT"))
    assert report["num_points_before"] == 1 and report["num_points_after"] == 0 and not rec.points
