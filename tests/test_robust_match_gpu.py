"""Geometric verification of calibrated pairs on the GPU (rp_match_filter in opensfm_b200/csrc/relpose.cu,
osfm_relpose_robust_match) against oracle/robust_match_oracle.py, pair by pair, the oracle starting from the engine's
own lo_model so that the stage after RANSAC is compared on identical inputs: the round that empties a pair, the four
counts and the final mask exactly, the refined pose within 1e-7.

The batch is tests/relative_pose_cases.batch_pairs' 196 pairs without the 42 of fewer than 8 rows, which the entry
refuses (and robust_match_calibrated answers on the host).  A pair is set aside only when the oracle meets a chord
within 1e-9 of a round's bound: there the last bits decide a row.  The test reports how many were and fails above
SET_ASIDE_MAX.

Also: the RANSAC is osfm_relpose_run's, bit for bit; the batch equals per-pair robust_match_calibrated calls; the
pair driver with `verify` equals the per-pair composition of the matcher and robust_match on a cube scene with the
scene's radial distortion; the error messages."""
import numpy as np
import pytest

import relative_pose_cases as C
import robust_match_cases as RC
from opensfm_b200 import matching
from opensfm_b200 import relative_pose as rp
from opensfm_b200 import synthetic as syn
from oracle import robust_match_oracle as rmo

pytestmark = pytest.mark.gpu

THRESHOLD = 0.004
SET_ASIDE_MAX = 4


@pytest.fixture(scope="module")
def batch():
    b1s, b2s = C.batch_pairs()
    keep = [p for p in range(len(b1s)) if len(b1s[p]) >= 8]
    assert len(keep) == 154
    return [b1s[p] for p in keep], [b2s[p] for p in keep]


@pytest.fixture(scope="module")
def result(batch):
    return rp.robust_match_lists(*batch, THRESHOLD)


def test_engine_equals_oracle(batch, result):
    b1s, b2s = batch
    set_aside, empty, worst = 0, {0: 0, 1: 0, 2: 0}, 0.0
    for p in range(len(b1s)):
        o = rmo.robust_match(b1s[p], b2s[p], result.lo_model[p], THRESHOLD, rmo.REFINE_ITERATIONS)
        if o.margins.chord < 1e-9:
            set_aside += 1
            continue
        assert result.empty_round(p) == o.empty_round, (p, result.counts[p], o.counts)
        assert result.counts[p].tolist() == o.counts, (p, result.counts[p], o.counts)
        assert np.array_equal(result.mask(p), o.mask), p
        if o.empty_round is None:
            err = np.abs(result.pose[p] - o.pose).max()
            assert err <= 1e-7, (p, err)
            worst = max(worst, err)
        else:
            assert np.isnan(result.pose[p]).all()
            empty[o.empty_round] += 1
    print("robust match: %d pairs, %d set aside, emptied per round %s, largest pose difference %.3g, RANSAC %.2f ms, "
          "filter %.2f ms" % (len(b1s), set_aside, empty, worst, result.ransac_ms, result.filter_ms))
    assert set_aside <= SET_ASIDE_MAX
    assert sum(empty.values()) >= 1 and (result.counts[:, 3] > 0).sum() >= 100


def test_ransac_is_relpose_run(batch, result):
    """lo_model and the RANSAC inlier counts are osfm_relpose_run's, bit for bit."""
    run = rp.ransac_lists(*batch, THRESHOLD)
    assert np.array_equal(run.lo_model, result.lo_model)
    assert np.array_equal(run.ransac_inliers, result.ransac_inliers)


def test_batch_equals_single_pair_drop_in(batch, result):
    """robust_match_calibrated per pair, through a camera whose pixel_bearing_many gives the batch's bearings."""
    b1s, b2s = batch
    cam = RC.RadialCamera(0.0, 0.0, 1.0)
    config = dict(RC.CONFIG)
    pick = list(range(0, len(b1s), 7))
    p1s = [b[:, :2] / b[:, 2:] for b in b1s]
    p2s = [b[:, :2] / b[:, 2:] for b in b2s]
    whole = rp.robust_match_lists([cam.pixel_bearing_many(p1s[p]) for p in pick],
                                  [cam.pixel_bearing_many(p2s[p]) for p in pick], THRESHOLD)
    for k, p in enumerate(pick):
        m = np.column_stack([np.arange(len(p1s[p])), np.arange(len(p1s[p]))])
        got = matching.robust_match_calibrated(p1s[p], p2s[p], cam, cam, m, config)
        assert np.array_equal(got, m[whole.mask(k)]), p


def test_pair_driver_equals_per_pair_composition():
    """match_images_with_pairs(..., verify=...) on a cube scene (k1 = -0.1, k2 = 0.01, so the calibrated branch)
    equals the engine matcher followed by robust_match pair by pair.  Every pair keeps more than 25 matches, and at
    least 99.5 % of all kept matches join two observations of the same point."""
    sc = syn.cube_scene(8, 600, seed=17)
    desc, points, ids, cam = RC.cube_images(sc)
    images = sorted(desc)
    pairs = [(a, b) for i, a in enumerate(images) for b in images[i + 1:]]
    cameras = {im: cam for im in images}
    got = matching.match_images_with_pairs(desc, pairs, RC.CONFIG, verify={"cameras": cameras, "points": points})
    pm = matching.PairMatcher()
    pm.add_many([(im, desc[im]) for im in images])
    raw = pm.match_pairs(pairs, RC.CONFIG)
    kept = true = 0
    for p in pairs:
        m = raw[p]
        want = np.zeros((0, 2), dtype=np.int64)
        if len(m) >= 20:
            want = np.asarray(matching.robust_match(points[p[0]], points[p[1]], cam, cam, m, RC.CONFIG),
                              dtype=np.int64).reshape(-1, 2)
            if len(want) < 20:
                want = np.zeros((0, 2), dtype=np.int64)
        assert np.array_equal(got[p], want), p
        assert len(got[p]) > 25, (p, len(got[p]))
        kept += len(got[p])
        true += int((ids[p[0]][got[p][:, 0]] == ids[p[1]][got[p][:, 1]]).sum())
    print("pair driver: %d pairs, %d matches kept, %d true" % (len(pairs), kept, true))
    assert true >= 0.995 * kept


def test_errors_name_the_pair():
    b = C.unit(np.random.RandomState(0).randn(40, 3) + [0, 0, 3])
    with pytest.raises(ValueError, match="pair 1 has 7 rows; at least 8"):
        rp.robust_match_lists([b[:8], b[:7], b[:9]], [b[8:16], b[16:23], b[23:32]], THRESHOLD)
    bearings, start, ra, rb = rp.pack_lists([b[:8], b[:9]], [b[8:16], b[16:25]])
    rb[9] = 99
    with pytest.raises(ValueError, match="row 1 of pair 1 names a bearing outside"):
        rp.robust_match_pairs(bearings, start, ra, rb, THRESHOLD)
    with pytest.raises(ValueError, match="refine_iterations must be at least 1"):
        rp.robust_match_lists([b[:8]], [b[8:16]], THRESHOLD, refine_iterations=0)
    with pytest.raises(ValueError, match="robust_filter or verify"):
        matching.match_images_with_pairs({}, [], RC.CONFIG, robust_filter=lambda a, b, m: m,
                                         verify={"cameras": {}, "points": {}})
