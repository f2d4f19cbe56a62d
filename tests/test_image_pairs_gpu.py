"""The rotation-only RANSAC of image pairs on the GPU (opensfm_b200/csrc/rotransac.cu) against
oracle/rotation_ransac_oracle.py, pair by pair: the drawn sample indices, the RANSAC and chord inlier counts, the
chord mask and the score exactly, lo_model to 1e-12; and the ranked outputs of compute_image_pairs,
compute_image_pairs_sequential and compute_image_pairs_from_tracks.

A pair is left out of the exact comparison only when the oracle meets an error within 1e-12 of a threshold or a
stopping bound within 1e-9 of the iteration it is compared with: there the last bits of fp64 arithmetic decide,
and the device contracts to fused multiply-adds where numpy does not."""
import multiprocessing
import os
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

import image_pair_cases as C
from opensfm_b200 import reconstruction as rec
from opensfm_b200 import rotation_ransac as rr
from opensfm_b200 import synthetic as syn
from opensfm_b200 import tracking
from oracle import rotation_ransac_oracle as o

pytestmark = pytest.mark.gpu

THRESHOLD = 4 * 0.004          # 4 * five_point_algo_threshold, OpenSfM's default
STAGE_ROWS = 1024              # RANSAC_STAGE_ROWS: larger pairs are read through L2


def oracle_all(b1s, b2s, threshold):
    workers = max(1, min(16, os.cpu_count() or 1))
    with ProcessPoolExecutor(workers, mp_context=multiprocessing.get_context("spawn")) as ex:
        return list(ex.map(o.ransac_rotation, b1s, b2s, [threshold] * len(b1s), chunksize=4))


def marginal(r: o.PairResult) -> bool:
    return min(r.error_margin, r.chord_margin) < 1e-12 or r.stop_margin < 1e-9


def run_traced(b1s, b2s, threshold, want, prefix=None):
    h = rr.RotationRansac()
    if prefix is not None:
        h.set_stream_prefix(prefix)
    h.set_trace(max(len(r.draws) for r in want) + 1)
    res = h.run(*rr.pack_lists(b1s, b2s), threshold)
    draws, count, used = h.trace()
    return res, draws, count, used


def compare(res, draws, count, used, want):
    """Exact agreement on every pair the oracle does not mark as marginal; returns how many it marked."""
    excluded = 0
    for p, r in enumerate(want):
        if marginal(r):
            excluded += 1
            continue
        assert count[p] == len(r.draws) and np.array_equal(draws[p], r.draws), p
        assert used[p] == r.stream_used, p
        assert res.ransac_inliers[p] == r.ransac_inliers, p
        assert res.chord_inliers[p] == r.chord_inliers, p
        b, e = res.pair_start[p], res.pair_start[p + 1]
        assert np.array_equal(res.chord_mask[b:e], r.chord_mask), p
        assert np.abs(res.lo_model[p] - r.lo_model).max() <= 1e-12, (p, np.abs(res.lo_model[p] - r.lo_model).max())
        assert res.scores()[p] == r.score, p
    return excluded


@pytest.fixture(scope="module")
def batch():
    """Pairs of a cube scene with 0 .. 65 % injected outliers, near-rotational and (every 40th) translational, of
    3, 4, 7, 12, 50, 200, 600, 1025 and 3000 rows."""
    b1s, b2s = C.cube_pairs(8, 3000, 5, sizes=(3, 4, 7, 12, 50, 200, 600, 1025, 3000), translational_every=40)
    return b1s, b2s, oracle_all(b1s, b2s, THRESHOLD)


def test_engine_equals_oracle(batch):
    b1s, b2s, want = batch
    n = np.array([len(b) for b in b1s])
    assert len(b1s) >= 250 and {3, 4, 50, 3000} <= set(n.tolist()) and (n > STAGE_ROWS).any()
    res, draws, count, used = run_traced(b1s, b2s, THRESHOLD, want)
    excluded = compare(res, draws, count, used, want)
    print("rotation RANSAC: %d pairs, %d left out as marginal, device %.2f ms" % (len(b1s), excluded, res.device_ms))
    assert excluded <= len(b1s) // 20
    assert sum(r.score > 0 for r in want) >= 50 and sum(r.score == 0 for r in want) >= 50


def test_exhausted_stream_continues_exactly(batch):
    """With 700 generator outputs kept on the device, most pairs run past them and continue from the saved state."""
    b1s, b2s, want = batch
    pick = [p for p, r in enumerate(want) if r.stream_used > 700][:60] + list(range(10))
    b1s, b2s, want = [b1s[p] for p in pick], [b2s[p] for p in pick], [want[p] for p in pick]
    res, draws, count, used = run_traced(b1s, b2s, THRESHOLD, want, prefix=700)
    assert (used > 700).sum() >= 50
    assert compare(res, draws, count, used, want) <= len(pick) // 20


def test_known_answer_relative_rotation():
    """test_robust.py's test_outliers_relative_rotation_ransac on the engine: 30 % outliers, inliers within 4 % of
    70 %, the model within 8e-2 of the true rotation."""
    cases = [C.robust_case(seed) for seed in range(20)]
    res = rr.ransac_pairs_lists([c[0] for c in cases], [c[1] for c in cases], cases[0][3])
    for p, (b1, _, rotation, _) in enumerate(cases):
        assert np.isclose(res.ransac_inliers[p], 0.7 * len(b1), rtol=0.04), p
        assert np.linalg.norm(rotation - res.lo_model[p], ord="fro") < 8e-2, p


def test_fewer_than_three_rows_names_the_pair():
    b = C.unit(np.random.RandomState(0).randn(10, 3))
    with pytest.raises(ValueError, match="pair 1 has 2 correspondences"):
        rr.ransac_pairs_lists([b[:5], b[:2], b[:4]], [b[5:], b[2:4], b[6:]], THRESHOLD)


@pytest.fixture(scope="module")
def tracks_scene():
    """A TracksManager of a cube scene matched on its true correspondences, 15 % of each pair's second features
    moved to a wrong position, and the dataset stand-in whose camera turns those positions into bearings."""
    sc = syn.cube_scene(8, 400, seed=9)
    rows = [np.nonzero(sc.obs_shot == s)[0] for s in range(sc.num_shots)]
    rng = np.random.RandomState(9)
    feats = {}
    for s, r in enumerate(rows):
        xy = sc.obs_xy[r].copy()
        bad = rng.rand(len(xy)) < 0.15
        xy[bad] += rng.uniform(-0.2, 0.2, (int(bad.sum()), 2))
        feats["im%02d" % s] = np.column_stack([xy, sc.obs_sigma[r]])
    matches = {}
    for i in range(sc.num_shots):
        for j in range(i + 1, sc.num_shots):
            _, ki, kj = np.intersect1d(sc.obs_point[rows[i]], sc.obs_point[rows[j]], return_indices=True)
            matches["im%02d" % i, "im%02d" % j] = np.column_stack([ki, kj]).astype(np.int32)
    tm = tracking.create_tracks_manager(feats, {}, {}, {}, matches, 2)
    return tm, C.Dataset(0.004)


def test_compute_image_pairs_orders(tracks_scene):
    tm, data = tracks_scene
    cam = data.camera
    track_dict = tracking.all_common_tracks_with_features(tm)
    keys = list(track_dict)
    want = oracle_all([cam.pixel_bearing_many(v[1]) for v in track_dict.values()],
                      [cam.pixel_bearing_many(v[2]) for v in track_dict.values()], THRESHOLD)
    assert len(keys) >= 20 and not any(marginal(r) for r in want)
    scores = [r.score for r in want]
    assert len(set(s for s in scores if s > 0)) >= 10

    pairs = [k for k, s in zip(keys, scores) if s > 0]
    positive = [s for s in scores if s > 0]
    expected = [pairs[i] for i in np.argsort(-np.array(positive))]
    assert rec.compute_image_pairs(track_dict, data) == expected

    by_key = dict(zip(keys, scores))
    conn = [k for k, size in tm.get_all_pairs_connectivity().items() if size >= 50]
    results = [(a, b, by_key[a, b]) for a, b in conn if by_key[a, b] > 0]
    results.sort(key=lambda x: x[2], reverse=True)
    assert rec.compute_image_pairs_sequential(data, tm) == [(a, b) for a, b, _ in results]

    cameras = {im: cam for im in tm.images}
    assert rec.compute_image_pairs_from_tracks(tm, cameras, data.config) == rec.compute_image_pairs(track_dict, data)


def test_two_view_reconstruction_rotation_only(tracks_scene):
    tm, data = tracks_scene
    (im1, im2), (_, p1, p2) = next(iter(tracking.all_common_tracks_with_features(tm).items()))
    rvec, inliers = rec.two_view_reconstruction_rotation_only(p1, p2, data.camera, data.camera, THRESHOLD)
    r = o.ransac_rotation(data.camera.pixel_bearing_many(p1), data.camera.pixel_bearing_many(p2), THRESHOLD)
    assert np.array_equal(inliers, np.nonzero(r.chord_mask)[0])
    assert np.abs(syn.angle_axis_to_rotation(rvec) - r.R.T).max() < 1e-9
