"""Five-point relative-pose RANSAC on the GPU (opensfm_b200/csrc/relpose.cu) against oracle/relative_pose_oracle.py
(its results on the batch are kept in tests/golden/relative_pose_oracle.npz, made by
tests/golden/make_relative_pose_golden.py), pair by pair: the drawn sample indices, the generator outputs used, the
RANSAC inlier count and the inlier mask exactly, lo_model to 1e-8; the batched form against a loop of the single-pair
drop-in; an exhausted stream prefix; error messages.

A pair is left out of the exact comparison only when the oracle meets an error within 1e-12 of its threshold, a
stopping bound within 1e-9 of the iteration it is compared with, an eigenvalue whose |Im| is within 1e-8 (relative)
of the real-root rule, two decompositions whose scores are within 1e-9, or a singular-value ratio within 1e-9 of 4:
there the last bits of fp64 arithmetic decide.  lo_model's bar is 1e-8 because the engine's eigenvalues come from
its own QR iteration and the oracle's from LAPACK: the essentials of a sample agree to about 1e-12, and the
decomposition and the N-point fit amplify that by the conditioning of the sample."""
import os
from dataclasses import dataclass

import numpy as np
import pytest

import relative_pose_cases as C
from opensfm_b200 import relative_pose as rp
from opensfm_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

STAGE_ROWS = 1024              # RANSAC_STAGE_ROWS: larger pairs are read through L2
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "relative_pose_oracle.npz")


@dataclass
class Want:
    """One pair's oracle result, as tests/golden/make_relative_pose_golden.py stored it."""
    draws: np.ndarray
    stream_used: int
    ransac_inliers: int
    inlier_mask: np.ndarray
    lo_model: np.ndarray
    margins: np.ndarray            # error, stop bound, root classification, decomposition, singular-value ratio

    def marginal(self) -> bool:
        m = self.margins
        return m[0] < 1e-12 or m[1] < 1e-9 or m[2] < 1e-8 or m[3] < 1e-9 or m[4] < 1e-9


def run_traced(b1s, b2s, want, prefix=None):
    h = rp.RelativePose()
    if prefix is not None:
        h.set_stream_prefix(prefix)
    h.set_trace(max(len(r.draws) for r in want) + 1)
    res = h.run(*rp.pack_lists(b1s, b2s), C.THRESHOLD)
    draws, count, used = h.trace()
    return res, draws, count, used


def compare(res, draws, count, used, want):
    """Exact agreement on every pair the oracle does not mark as marginal; returns how many it marked."""
    excluded = 0
    for p, r in enumerate(want):
        if r.marginal():
            excluded += 1
            continue
        assert count[p] == len(r.draws) and np.array_equal(draws[p], r.draws), p
        assert used[p] == r.stream_used, p
        assert res.ransac_inliers[p] == r.ransac_inliers, p
        assert np.array_equal(res.inliers(p), r.inlier_mask), p
        err = np.abs(res.lo_model[p] - r.lo_model).max()
        assert err <= 1e-8, (p, err)
    return excluded


@pytest.fixture(scope="module")
def batch():
    b1s, b2s = C.batch_pairs()
    g = np.load(GOLDEN)
    assert str(g["inputs_digest"]) == C.digest(b1s, b2s), "the fixture was made from other inputs"
    n = np.array([len(b) for b in b1s])
    row_start = np.concatenate([[0], np.cumsum(n)])
    mask = np.unpackbits(g["inlier_mask"])[:row_start[-1]].astype(bool)
    ds = g["draw_start"]
    want = [Want(g["draws"][ds[k]:ds[k + 1]].astype(np.int32), int(g["stream_used"][k]), int(g["ransac_inliers"][k]),
                 mask[row_start[k]:row_start[k + 1]], g["lo_model"][k], g["margins"][k]) for k in range(len(b1s))]
    return b1s, b2s, want


def test_engine_equals_oracle(batch):
    b1s, b2s, want = batch
    n = np.array([len(b) for b in b1s])
    assert len(b1s) >= 190 and {5, 6, 12, 50, 600, 3000} <= set(n.tolist()) and (n > STAGE_ROWS).any()
    res, draws, count, used = run_traced(b1s, b2s, want)
    excluded = compare(res, draws, count, used, want)
    print("relative pose: %d pairs, %d left out as marginal, device %.2f ms" % (len(b1s), excluded, res.device_ms))
    assert excluded <= len(b1s) // 20
    assert sum(r.ransac_inliers >= 50 for r in want) >= 80


def test_exhausted_stream_continues_exactly(batch):
    """With 700 generator outputs kept on the device, pairs that run past them continue from the saved state."""
    b1s, b2s, want = batch
    pick = [p for p, r in enumerate(want) if r.stream_used > 700][:60] + list(range(10))
    b1s, b2s, want = [b1s[p] for p in pick], [b2s[p] for p in pick], [want[p] for p in pick]
    res, draws, count, used = run_traced(b1s, b2s, want, prefix=700)
    assert (used > 700).sum() >= 20
    assert compare(res, draws, count, used, want) <= len(pick) // 20


def test_batched_equals_single_pair_drop_in(batch):
    b1s, b2s, _ = batch
    pick = list(range(0, len(b1s), 9))
    res = rp.ransac_lists([b1s[p] for p in pick], [b2s[p] for p in pick], C.THRESHOLD)
    for k, p in enumerate(pick):
        T = rp.relative_pose_ransac(b1s[p], b2s[p], C.THRESHOLD, 1000, 0.999)
        assert np.array_equal(T, res.poses()[k]), p


def test_known_answer_pose():
    """Noise-free pairs with 30 % outliers: about 70 % of the rows are inliers, and lo_model is the true [R | t]
    (unit t, x2 = R x1 + t) up to the pull of the few outliers that fall within the threshold."""
    seed, cams = 11, 8
    b1s, b2s = C.cube_pairs(cams, 400, seed, count=8, sizes=(400,), outlier_ratios=(0.3,), noise=0.0,
                            planar_every=0)
    sc = syn.cube_scene(cams, 400, seed=seed, with_descriptors=False)
    res = rp.ransac_lists(b1s, b2s, 0.004)
    for k in range(len(b1s)):
        s, o = k % cams, (k + 1 + k % 3) % cams
        R = sc.R_wc[o] @ sc.R_wc[s].T
        t = sc.R_wc[o] @ (sc.origins[s] - sc.origins[o])
        assert np.isclose(res.ransac_inliers[k], 0.7 * len(b1s[k]), rtol=0.1), k
        assert np.abs(res.lo_model[k] - np.column_stack([R, t / np.linalg.norm(t)])).max() < 1e-2, k


def test_error_names_the_pair():
    b = C.unit(np.random.RandomState(0).randn(20, 3))
    with pytest.raises(ValueError, match="pair 1 has 4 rows; at least 5"):
        rp.ransac_lists([b[:5], b[:4], b[:6]], [b[5:10], b[10:14], b[14:20]], C.THRESHOLD)
    bearings, start, ra, rb = rp.pack_lists([b[:5], b[:6]], [b[5:10], b[10:16]])
    rb[6] = 99
    with pytest.raises(ValueError, match="row 1 of pair 1 names a bearing outside"):
        rp.ransac_pairs(bearings, start, ra, rb, C.THRESHOLD)
