"""Track triangulation on the GPU (csrc/triangulate.cu through TracksManager.triangulate and
opensfm_b200.triangulation) against the oracle (oracle/triangulation_oracle.py): statuses exactly, points within
1e-9 of their distance to the cameras, the reference's known answers, long tracks, and the drop-ins' writes."""
import numpy as np
import pytest

import triangulation_cases as tc
from oracle import triangulation_oracle as to
from opensfm_b200 import tracking, triangulation

pytestmark = pytest.mark.gpu

# a track whose deciding quantity lies this close to its threshold may differ by summation order
BORDERLINE = 1e-12


def _manager(sc):
    features, colors, matches = sc.tracks_inputs()
    return tracking.create_tracks_manager(features, colors, {}, {}, matches, 2)


def _run_both(tm, rec, selected, config=tc.CONFIG):
    rays = triangulation.shot_rays(tm, rec)
    opts = triangulation._options(config)
    X, status = tm.triangulate(rays["image_rt"], rays["image_origin"], rays["image_in"], rays["bearings"], selected,
                               *opts)
    ost, oX, margin = to.triangulate_tracks(tm.track_start, tm.obs_image, rays["image_rt"], rays["image_origin"],
                                            rays["image_in"], rays["bearings"], selected, *opts)
    return rays, X, status, oX, ost, margin


def _compare(tm, rays, X, status, oX, ost, margin):
    """Exact status parity outside the borderline tracks, which are counted and reported; the points of the
    triangulated tracks within 1e-9 of their mean distance to the track's cameras."""
    borderline = margin <= BORDERLINE
    differ = np.nonzero((status != ost) & ~borderline)[0]
    assert not len(differ), (differ[:10], status[differ[:10]], ost[differ[:10]])
    print("borderline tracks set aside: %d of %d" % (int(borderline.sum()), len(status)))
    both = np.nonzero((status == to.OK) & (ost == to.OK))[0]
    for t in both.tolist():
        rows = np.arange(tm.track_start[t], tm.track_start[t + 1])
        im = tm.obs_image[rows][rays["image_in"][tm.obs_image[rows]].astype(bool)]
        dist = np.linalg.norm(oX[t] - rays["image_origin"][im], axis=1).mean()
        assert np.abs(X[t] - oX[t]).max() <= 1e-9 * dist, (t, X[t], oX[t], dist)
    assert np.isnan(X[status != to.OK]).all()
    return np.bincount(status, minlength=5)


@pytest.fixture(scope="module")
def cube():
    sc, camera, in_rec = tc.cube_case()
    return sc, camera, in_rec, _manager(sc)


def test_statuses_and_points_equal_the_oracle(cube):
    sc, camera, in_rec, tm = cube
    rec = sc.reconstruction(camera, in_rec, np.random.RandomState(0), 1e-4, 1e-3)
    selected = np.ones(tm.num_tracks(), dtype=np.uint8)
    selected[::7] = 0
    counts = _compare(tm, *_run_both(tm, rec, selected))
    assert all(counts > 0), counts   # every status, not selected included
    assert tm.triangulate_device_ms > 0


def test_permuting_the_shots_of_the_reconstruction_changes_no_status(cube):
    sc, camera, in_rec, tm = cube
    selected = np.ones(tm.num_tracks(), dtype=np.uint8)
    rec = sc.reconstruction(camera, in_rec, np.random.RandomState(1), 1e-4, 1e-3)
    perm = sc.reconstruction(camera, [in_rec[i] for i in np.random.RandomState(2).permutation(len(in_rec))],
                             np.random.RandomState(1), 0.0, 0.0)
    for s in perm.shots:   # the same poses, inserted in another order
        perm.shots[s].pose.set_rotation_matrix(rec.shots[s].pose.get_rotation_matrix())
        perm.shots[s].pose.set_origin(rec.shots[s].pose.get_origin())
    _, X, status, _, _, _ = _run_both(tm, rec, selected)
    _, Xp, status_p, _, _, _ = _run_both(tm, perm, selected)
    assert np.array_equal(status, status_p)
    ok = status == to.OK
    assert np.abs(X[ok] - Xp[ok]).max() <= 1e-9


def test_long_tracks():
    sc, camera, shots = tc.ring_case((200, 40, 33))
    tm = _manager(sc)
    assert sorted(np.diff(tm.track_start).tolist()) == [33, 40, 200]
    rec = sc.reconstruction(camera, shots, np.random.RandomState(3), 1e-4, 1e-3)
    counts = _compare(tm, *_run_both(tm, rec, np.ones(tm.num_tracks(), dtype=np.uint8)))
    assert counts[to.OK] == 3, counts


def test_empty_selection(cube):
    sc, camera, in_rec, tm = cube
    rec = sc.reconstruction(camera, in_rec, np.random.RandomState(0))
    rays, X, status, _, _, _ = _run_both(tm, rec, np.zeros(tm.num_tracks(), dtype=np.uint8))
    assert (status == to.NOT_SELECTED).all() and np.isnan(X).all()
    triangulation.triangulate_shot_features(tm, rec, [], tc.CONFIG)
    assert not rec.points


def _observation_sets(rec):
    return {p: sorted(s.id for s in lm.get_observations()) for p, lm in rec.points.items()}


def test_retriangulate_equals_the_reference_loop(cube):
    sc, camera, in_rec, tm = cube
    rec = sc.reconstruction(camera, in_rec, np.random.RandomState(4), 1e-4, 1e-3)
    ref = sc.reconstruction(camera, in_rec, np.random.RandomState(4), 1e-4, 1e-3)
    rec.create_point("stale", [0.0, 0.0, 0.0])
    rec.add_observation(in_rec[0], "stale", tc.map_types.Observation(0, 0, 1))
    report = triangulation.retriangulate(tm, rec, tc.CONFIG)
    want = to.retriangulate(tm, ref, tc.CONFIG)
    assert report["num_points_before"] == 1 and report["num_points_after"] == want["num_points_after"] > 0
    assert "stale" not in rec.points and not any("stale" in o for o in rec._shot_obs.values())
    assert _observation_sets(rec) == _observation_sets(ref)
    for p, lm in rec.points.items():
        assert np.abs(lm.coordinates - ref.points[p].coordinates).max() <= 1e-8
    for p, lm in list(rec.points.items())[:50]:
        for shot in lm.get_observations():
            a, b = shot.get_landmark_observation(lm), ref.shots[shot.id].get_landmark_observation(ref.points[p])
            assert np.array_equal(a.point, b.point) and a.id == b.id


def test_triangulate_shot_features_touches_only_new_tracks_of_the_shots(cube):
    sc, camera, in_rec, tm = cube
    rec = sc.reconstruction(camera, in_rec, np.random.RandomState(5), 1e-4, 1e-3)
    ref = sc.reconstruction(camera, in_rec, np.random.RandomState(5), 1e-4, 1e-3)
    shot_ids = [in_rec[2], in_rec[3], "not-a-shot"]
    seen = set(tm.get_shot_observations(in_rec[2])) | set(tm.get_shot_observations(in_rec[3]))
    existing = sorted(seen, key=int)[:5]
    for r in (rec, ref):
        for p in existing:
            r.create_point(p, [7.0, 7.0, 7.0])
    triangulation.triangulate_shot_features(tm, rec, shot_ids, tc.CONFIG)
    to.triangulate_shot_features(tm, ref, shot_ids, tc.CONFIG)
    for p in existing:
        assert np.array_equal(rec.points[p].coordinates, [7.0, 7.0, 7.0]) and rec.points[p].number_of_observations() == 0
    assert set(rec.points) <= seen and len(rec.points) > len(existing)
    assert _observation_sets(rec) == _observation_sets(ref)


@pytest.mark.parametrize("case", tc.known_answers()["tracks"], ids=lambda c: c["name"])
def test_known_answers_on_the_engine(case):
    features, colors, matches = tc.known_answer_inputs(case)
    tm = tracking.create_tracks_manager(features, colors, {}, {}, matches, 2)
    rec = tc.reconstruction_from_json(case, tc.SphericalCamera())
    o = case["options"]
    config = dict(tc.CONFIG, triangulation_threshold=o["reproj_threshold"],
                  triangulation_min_ray_angle=o["min_ray_angle_degrees"], triangulation_min_depth=o["min_depth"],
                  triangulation_refinement_iterations=o["iterations"])
    triangulation.triangulate_shot_features(tm, rec, ["im1", "im2"], config)
    if case["expected_point"] is None:
        assert not rec.points
    else:
        assert list(rec.points) == ["0"]
        assert np.allclose(rec.points["0"].coordinates, case["expected_point"])
        assert len(rec.points["0"].get_observations()) == case["expected_observations"]


def test_sizes_that_are_not_the_handles_are_refused(cube):
    sc, camera, in_rec, tm = cube
    rec = sc.reconstruction(camera, in_rec, np.random.RandomState(0))
    rays = triangulation.shot_rays(tm, rec)
    h = tm._handle
    from opensfm_b200._lib import ptr

    status = np.zeros(tm.num_tracks(), dtype=np.int8)
    X = np.zeros((tm.num_tracks(), 3))
    sel = np.ones(tm.num_tracks(), dtype=np.uint8)
    code = h.L.osfm_tracks_triangulate(h.h, len(tm.images), ptr(rays["image_rt"]), ptr(rays["image_origin"]),
                                       ptr(rays["image_in"]), len(tm.obs_track) - 1, ptr(rays["bearings"]),
                                       tm.num_tracks(), ptr(sel), 0.006, 0.01, 0.001, 10, ptr(status), ptr(X))
    assert code != 0 and b"differ from the handle's" in h.L.osfm_last_error()
