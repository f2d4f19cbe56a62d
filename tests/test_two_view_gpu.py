"""The two-view stage on the GPU (rp_two_view in opensfm_b200/csrc/relpose.cu, osfm_relpose_two_view) against
oracle/two_view_oracle.py, pair by pair, the oracle starting from the engine's own lo_model and plane motion so that
this stage is compared on identical inputs: every final count, mask, kept configuration and method exactly, each
kept configuration's refined pose to 1e-7 (TinySolver's parameter stop leaves about 1e-8 relative).  The
configuration a Necker check drops is a wrong pose, where the cost is flat and ill-conditioned: the summation orders
of the engine and the oracle take the solver to points up to about 5e-3 apart (measured on the batch), which
can move its count by a row; the test bounds that at 1e-2 and a 2 % count change.

A pair is set aside only when the oracle meets a chord within 1e-9 of the threshold or a midpoint |det| within
1e-9 of 1e-10: there the last bits decide a row, and every count gap behind a decision moves with it.  The test
reports how many were set aside and fails above 5 %.

Also: noise-free pairs against their true pose, the batch against a loop of the single-pair drop-in, the tracks
form against the per-pair drop-in, and the error messages."""
import numpy as np
import pytest

import image_pair_cases as IC
import relative_pose_cases as C
from opensfm_b200 import reconstruction as rec
from opensfm_b200 import relative_pose as rp
from opensfm_b200 import synthetic as syn
from opensfm_b200 import tracking
from oracle import two_view_oracle as tv

pytestmark = pytest.mark.gpu

ITERATIONS = 1000


def marginal(m: tv.Margins) -> bool:
    return m.chord < 1e-9 or m.det < 1e-9


def compare(res: rp.TwoViewResult, b1s, b2s, check_reversal: bool, reversal_ratio: float):
    set_aside, configs = 0, 2 if check_reversal else 1
    methods = {}
    other, moved = 0.0, []
    for p in range(len(b1s)):
        o = tv.two_view(b1s[p], b2s[p], res.lo_model[p], res.plane[p], C.THRESHOLD, ITERATIONS, check_reversal,
                        reversal_ratio)
        if marginal(o.margins):
            set_aside += 1
            continue
        rows = res.rows(p)
        for c in range(configs):
            if c == o.chosen or configs == 1:
                assert res.counts[p, c] == o.counts[c], (p, c, res.counts[p], o.counts)
            elif res.counts[p, c] != o.counts[c]:
                # the dropped configuration's endpoint moves (see above); its count may move by a row or two, but
                # never across the Necker decision, which `chosen` pins
                assert abs(int(res.counts[p, c]) - int(o.counts[c])) <= max(2, o.counts[c] // 50), (p, c)
                moved.append(p)
        assert res.counts[p, 2] == o.counts[2], p
        assert res.chosen[p] == o.chosen, p
        assert np.array_equal(res.mask_5pt[rows], o.mask_5pt), p
        assert np.array_equal(res.mask_plane[rows], o.mask_plane), p
        assert res.method(p) == o.method, p
        for c in range(configs):
            err = np.abs(res.pose[p, c] - o.pose[c]).max()
            if c == o.chosen or configs == 1:
                assert err <= 1e-7, (p, c, err)
            else:
                other = max(other, err)
        if configs == 1:
            assert np.isnan(res.pose[p, 1]).all()
        methods[o.method] = methods.get(o.method, 0) + 1
    print("dropped configurations: largest pose difference %.3g, counts moved on pairs %s" % (other, moved))
    assert len(moved) <= len(b1s) // 20
    assert other <= 1e-2
    return set_aside, methods


@pytest.fixture(scope="module")
def batch():
    return C.batch_pairs()


@pytest.mark.parametrize("check_reversal,reversal_ratio", [(False, 1.0), (True, 0.95)])
def test_engine_equals_oracle(batch, check_reversal, reversal_ratio):
    b1s, b2s = batch
    res = rp.two_view_lists(b1s, b2s, C.THRESHOLD, ITERATIONS, check_reversal, reversal_ratio)
    set_aside, methods = compare(res, b1s, b2s, check_reversal, reversal_ratio)
    print("two-view (check_reversal=%s): %d pairs, %d set aside, methods %s, RANSAC %.2f ms, two-view %.2f ms" % (
        check_reversal, len(b1s), set_aside, methods, res.ransac_ms, res.two_view_ms))
    assert set_aside <= len(b1s) // 20
    assert methods.get("5_point", 0) >= 50 and methods.get("plane_based", 0) >= 10
    if check_reversal:
        assert (res.chosen == 1).any() or (res.counts[:, 1] > 0).any()


@pytest.mark.parametrize("outliers", [0.0, 0.3])
def test_true_pose(outliers):
    """Noise-free pairs: R (angle-axis) and t of the second camera near the truth.  When the plane motion has as many
    inliers as the 5-point pose, equal counts go to the plane (the reference's rule); with 30 % outliers the 5-point
    method wins on most pairs.  The bar is 1e-2 (as for RANSAC's lo_model), not 1e-6: the residuals 1 - cos are quadratic in the angular error, so
    TinySolver's stops end where the quartic cost is flat, and outliers inside the threshold pull on it."""
    seed, cams = 11, 8
    b1s, b2s = C.cube_pairs(cams, 400, seed, count=8, sizes=(400,), outlier_ratios=(outliers,), noise=0.0,
                            planar_every=0)
    sc = syn.cube_scene(cams, 400, seed=seed, with_descriptors=False)
    res = rp.two_view_lists(b1s, b2s, C.THRESHOLD, ITERATIONS)
    planes = 0
    for k in range(len(b1s)):
        s, o = k % cams, (k + 1 + k % 3) % cams
        R = sc.R_wc[o] @ sc.R_wc[s].T
        t = sc.R_wc[o] @ (sc.origins[s] - sc.origins[o])
        r, tt, inliers, report = res.result(k)
        if report["method"] == "plane_based":
            # equal counts go to the plane: every true inlier is an inlier of both
            assert report["plane_based_inliers"] == report["5_point_inliers"] >= 0.65 * len(b1s[k]), (k, report)
            planes += 1
            continue
        assert report["method"] == "5_point", (k, report)
        assert np.abs(syn.angle_axis_to_rotation(r) - R).max() < 1e-2, k
        assert np.abs(tt - t / np.linalg.norm(t)).max() < 1e-2, k
    assert outliers == 0.0 or planes <= len(b1s) // 2


def test_batch_equals_single_pair_drop_in(batch):
    b1s, b2s = batch
    pick = list(range(0, len(b1s), 7))
    res = rp.two_view_lists([b1s[p] for p in pick], [b2s[p] for p in pick], C.THRESHOLD, ITERATIONS, True, 0.95)
    for k, p in enumerate(pick):
        one = rp.two_view_lists([b1s[p]], [b2s[p]], C.THRESHOLD, ITERATIONS, True, 0.95).result(0)
        got = res.result(k)
        assert got[3] == one[3], p
        assert (got[0] is None) == (one[0] is None), p
        if got[0] is not None:
            assert np.array_equal(got[0], one[0]) and np.array_equal(got[1], one[1]), p
        assert np.array_equal(got[2], one[2]), p


def test_tracks_form_equals_drop_in():
    sc = syn.cube_scene(6, 300, seed=9)
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
    cam = IC.PinholeCamera()
    config = {"five_point_algo_threshold": 0.004, "five_point_refine_rec_iterations": 1000,
              "five_point_reversal_check": True, "five_point_reversal_ratio": 0.95}
    pairs = [(a, b) for (a, b), n in tm.get_all_pairs_connectivity().items() if n >= 20]
    pairs = pairs + [(b, a) for a, b in pairs[:3]]
    got = rec.two_view_reconstructions(tm, pairs, {im: cam for im in tm.images}, config)
    assert len(got) == len(pairs) >= 10
    methods = set()
    for (im1, im2), g in zip(pairs, got):
        p1, p2 = rec._get_common_feature_arrays(tm, im1, im2)
        want = rec.two_view_reconstruction_general(p1, p2, cam, cam, 0.004, 1000, True, 0.95)
        assert g[3] == want[3], (im1, im2)
        methods.add(g[3].get("method"))
        if want[0] is None:
            assert g[0] is None and len(g[2]) == 0
        else:
            assert np.array_equal(g[0], want[0]) and np.array_equal(g[1], want[1]) and np.array_equal(g[2], want[2])
    assert "5_point" in methods


def test_errors_name_the_pair():
    b = C.unit(np.random.RandomState(0).randn(20, 3) + [0, 0, 3])
    with pytest.raises(ValueError, match="pair 1 has 4 rows; at least 5"):
        rp.two_view_lists([b[:5], b[:4], b[:6]], [b[5:10], b[10:14], b[14:20]], C.THRESHOLD)
    bearings, start, ra, rb = rp.pack_lists([b[:5], b[:6]], [b[5:10], b[10:16]])
    rb[6] = 99
    with pytest.raises(ValueError, match="row 1 of pair 1 names a bearing outside"):
        rp.two_view_pairs(bearings, start, ra, rb, C.THRESHOLD)
    with pytest.raises(ValueError, match="refine_iterations must be at least 1"):
        rp.two_view_lists([b[:6]], [b[6:12]], C.THRESHOLD, iterations=0)
