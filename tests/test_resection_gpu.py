"""Resection on the GPU (opensfm_b200/csrc/resect.cu) against oracle/absolute_pose_oracle.py (its results on the
batch are kept in tests/golden/resection_oracle.npz, made by tests/golden/make_resection_golden.py), shot by
shot: the drawn sample indices, the generator outputs used, the RANSAC and chord inlier counts and the chord mask
exactly, lo_model to 1e-10 of the scene scale; the reference's RANSAC known answer; and resect_candidates against a
sequential loop of resect on copies of the same map.

A shot is left out of the exact comparison only when the oracle meets an error or a chord within 1e-12 of its
threshold, a relative change of Lu's translation within 1e-12 of 1e-7, or a stopping bound within 1e-9 of the
iteration it is compared with: there the last bits of fp64 arithmetic decide, and the device contracts to fused
multiply-adds where numpy does not.  Lu's band is absolute like the others: the engine's and the oracle's iterates
agree to about 1e-13, and a shot runs thousands of Lu steps, so a band of 1e-9 (1 % of the tolerance) would set
most shots aside."""
import os
from dataclasses import dataclass

import numpy as np
import pytest

import resection_cases as C
from opensfm_b200 import map_types as M
from opensfm_b200 import reconstruction as rec
from opensfm_b200 import resection as rs
from opensfm_b200 import synthetic as syn
pytestmark = pytest.mark.gpu

THRESHOLD = C.THRESHOLD
STAGE_ROWS = 1024              # RANSAC_STAGE_ROWS: larger shots are read through L2
SCENE_SCALE = 2.0              # cameras on a sphere of radius 2 around the unit cube


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resection_oracle.npz")


@dataclass
class Want:
    """One shot's oracle result, as tests/golden/make_resection_golden.py stored it."""
    draws: np.ndarray
    stream_used: int
    ransac_inliers: int
    chord_inliers: int
    chord_mask: np.ndarray
    lo_model: np.ndarray
    margins: np.ndarray            # error, chord, stop bound, Lu's relative change

    def marginal(self) -> bool:
        return min(self.margins[0], self.margins[1], self.margins[3]) < 1e-12 or self.margins[2] < 1e-9


def run_traced(bs, Xs, threshold, want, prefix=None):
    h = rs.Resection()
    if prefix is not None:
        h.set_stream_prefix(prefix)
    h.set_trace(max(len(r.draws) for r in want) + 1)
    res = h.run(*rs.pack_lists(bs, Xs), threshold)
    draws, count, used = h.trace()
    return res, draws, count, used


def compare(res, draws, count, used, want):
    """Exact agreement on every shot the oracle does not mark as marginal; returns how many it marked."""
    excluded = 0
    for s, r in enumerate(want):
        if r.marginal():
            excluded += 1
            continue
        assert count[s] == len(r.draws) and np.array_equal(draws[s], r.draws), s
        assert used[s] == r.stream_used, s
        assert res.ransac_inliers[s] == r.ransac_inliers, s
        assert res.chord_inliers[s] == r.chord_inliers, s
        assert np.array_equal(res.inliers(s), r.chord_mask), s
        err = np.abs(res.lo_model[s] - r.lo_model).max()
        assert err <= 1e-10 * SCENE_SCALE, (s, err)
    return excluded


@pytest.fixture(scope="module")
def batch():
    """resection_cases.batch_shots() and the oracle's result on every shot (tests/golden/resection_oracle.npz)."""
    bs, Xs = C.batch_shots()
    g = np.load(GOLDEN)
    assert str(g["inputs_digest"]) == C.digest(bs, Xs), "the fixture was made from other inputs"
    n = np.array([len(b) for b in bs])
    row_start = np.concatenate([[0], np.cumsum(n)])
    mask = np.unpackbits(g["chord_mask"])[:row_start[-1]].astype(bool)
    ds = g["draw_start"]
    want = [Want(g["draws"][ds[k]:ds[k + 1]].astype(np.int32), int(g["stream_used"][k]), int(g["ransac_inliers"][k]),
                 int(g["chord_inliers"][k]), mask[row_start[k]:row_start[k + 1]], g["lo_model"][k], g["margins"][k])
            for k in range(len(bs))]
    return bs, Xs, want


def test_engine_equals_oracle(batch):
    bs, Xs, want = batch
    n = np.array([len(b) for b in bs])
    assert len(bs) >= 200 and {5, 6, 12, 50, 600, 3000} <= set(n.tolist()) and (n > STAGE_ROWS).any()
    res, draws, count, used = run_traced(bs, Xs, THRESHOLD, want)
    excluded = compare(res, draws, count, used, want)
    print("resection: %d shots, %d left out as marginal, device %.2f ms" % (len(bs), excluded, res.device_ms))
    assert excluded <= len(bs) // 20
    assert sum(r.chord_inliers >= 10 for r in want) >= 100


def test_exhausted_stream_continues_exactly(batch):
    """With 700 generator outputs kept on the device, shots that run past them continue from the saved state."""
    bs, Xs, want = batch
    pick = [s for s, r in enumerate(want) if r.stream_used > 700][:60] + list(range(10))
    bs, Xs, want = [bs[s] for s in pick], [Xs[s] for s in pick], [want[s] for s in pick]
    res, draws, count, used = run_traced(bs, Xs, THRESHOLD, want, prefix=700)
    assert (used > 700).sum() >= 20
    assert compare(res, draws, count, used, want) <= len(pick) // 20


def test_known_answer_absolute_pose_ransac():
    """test_robust.py's test_outliers_absolute_pose_ransac on the engine: 30 % outliers, inliers within 5 % of 70 %,
    lo_model within 8e-2 of the pose."""
    sc = syn.cube_scene(6, 400, projection_noise=0.0, seed=11, with_descriptors=False)
    rng = np.random.RandomState(3)
    bs, Xs, poses = [], [], []
    for s in range(sc.num_shots):
        X = sc.points[sc.obs_point[sc.obs_shot == s]]
        b = C.unit((X - sc.origins[s]) @ sc.R_wc[s].T)
        bad = rng.permutation(len(b))[:int(0.3 * len(b))]
        b[bad] = C.unit(rng.randn(len(bad), 3))
        bs.append(b)
        Xs.append(X)
        poses.append(np.column_stack([sc.R_wc[s], -sc.R_wc[s] @ sc.origins[s]]))
    res = rs.ransac_lists(bs, Xs, 0.01)
    for s in range(len(bs)):
        assert np.isclose(res.ransac_inliers[s], 0.7 * len(bs[s]), rtol=0.05), s
        assert np.linalg.norm(res.lo_model[s] - poses[s]) < 8e-2, s
    T = rs.absolute_pose_ransac(bs[0], Xs[0], 0.01, 1000, 0.999)
    assert np.abs(T[:, :3] - sc.R_wc[0].T).max() < 8e-2 and np.abs(T[:, 3] - sc.origins[0]).max() < 8e-2


def test_error_names_the_shot():
    b = C.unit(np.random.RandomState(0).randn(10, 3))
    with pytest.raises(ValueError, match="shot 1 has 2 rows"):
        rs.ransac_lists([b[:5], b[:2], b[:4]], [b[5:], b[2:4], b[6:]], THRESHOLD)
    bearings, points, start, rb, rx = rs.pack_lists([b[:5], b[:4]], [b[5:], b[6:]])
    rx[6] = 99
    with pytest.raises(ValueError, match="row 1 of shot 1 names a point outside"):
        rs.ransac_shots(bearings, points, start, rb, rx, THRESHOLD)


# ---------------------------------------------------------------------------------------------------------------
# resect and resect_candidates on a map
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scene():
    return C.incremental_scene(24, 4000, seed=2)


def sequential(data, tm, r, candidates, threshold, min_inliers):
    """The grow_reconstruction loop: resect the candidates in order until one succeeds."""
    reports = []
    for image, _ in candidates:
        ok, new_shots, report = rec.resect(data, tm, r, image, threshold, min_inliers)
        reports.append(report)
        if ok:
            return image, new_shots, report, reports
    return None, set(), None, reports


def test_resect_candidates_equals_sequential_resect(scene):
    tm, r0, _ = scene
    data = C.Dataset()
    candidates = rec.reconstructed_points_for_images(tm, r0, set(tm.images))
    assert len(candidates) == 12
    for min_inliers in (10, 10 ** 6, None):
        a, b = C.clone(r0), C.clone(r0)
        if min_inliers is None:
            # the best candidates fail on their inlier count: the choice falls further down the list
            counts = [rep["num_inliers"] for rep in rec.resect_candidates(data, tm, C.clone(r0), candidates,
                                                                            THRESHOLD, 10 ** 6)[3]]
            min_inliers = sorted(counts)[-3]
        got = rec.resect_candidates(data, tm, a, candidates, THRESHOLD, min_inliers)
        want = sequential(data, tm, b, candidates, THRESHOLD, min_inliers)
        assert got[0] == want[0] and got[1] == want[1] and got[2] == want[2]
        assert got[3][:len(want[3])] == want[3]
        assert C.map_state(a) == C.map_state(b)
        if want[0] is None:
            assert C.map_state(a) == C.map_state(r0), "a failed resection changed the map"
        else:
            assert want[0] in a.shots and len(a._shot_obs[want[0]]) == want[2]["num_inliers"]


def test_few_rows_reported_not_launched(scene):
    tm, r0, sc = scene
    r = C.clone(r0)
    target = tm.images[-1]
    # keep only 4 of the points the target sees
    seen = [t for t in tm.get_shot_observations(target) if t in r.points]
    for t in seen[4:]:
        r.remove_landmark(r.points[t])
    ok, new_shots, report = rec.resect(C.Dataset(), tm, r, target, THRESHOLD, 10)
    assert (ok, new_shots, report) == (False, set(), {"num_common_points": 4})
    assert rec.last_resect_times()["device_ms"] == 0.0


def test_rig_candidate_triangulates_before_adding_inliers(scene, monkeypatch):
    tm, r0, sc = scene
    rigs = {"rig0": [(tm.images[-1], "cam"), (tm.images[-2], "right")]}
    data = C.Dataset(rigs)
    # the second rig camera sits where the scene's second shot is, relative to the first
    R1, R2 = sc.R_wc[-1], sc.R_wc[-2]
    t1, t2 = -R1 @ sc.origins[-1], -R2 @ sc.origins[-2]
    rc = rec.T.Pose()
    rc.set_rotation_matrix(R2 @ R1.T)
    rc.translation = t2 - R2 @ R1.T @ t1
    r0 = C.clone(r0)
    r0.add_rig_camera(M.RigCamera(rc, "right"))
    # points only the second shot sees are left for the triangulation of the new shots to make
    only_second = set(tm.get_shot_observations(tm.images[-2])) - set(tm.get_shot_observations(tm.images[-1]))
    for t in only_second & set(r0.points):
        r0.remove_landmark(r0.points[t])
    a = C.clone(r0)
    poses = []
    add_shot = rec.add_shot
    monkeypatch.setattr(rec, "add_shot", lambda *args: poses.append(args[-1]) or add_shot(*args))
    ok, new_shots, report = rec.resect(data, tm, a, tm.images[-1], THRESHOLD, 10)
    assert ok and new_shots == {tm.images[-1], tm.images[-2]} and set(report["shots"]) == new_shots
    # the same steps by hand: add the instance at the resected pose, triangulate its shots, then the inliers
    b = C.clone(r0)
    add_shot(data, b, rec.rig_assignments_per_image(rigs), tm.images[-1], poses[0])
    before = set(b.points)
    rec.triangulate_shot_features(tm, b, new_shots, data.config)
    assert len(set(b.points) - before) > 0
    inliers = set(a._shot_obs[tm.images[-1]]) - set(b._shot_obs.get(tm.images[-1], {}))
    for t in sorted(inliers, key=int):
        b.add_observation(tm.images[-1], t, tm.get_observation(tm.images[-1], t))
    assert C.map_state(a) == C.map_state(b)
