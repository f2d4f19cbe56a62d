"""GPU parity of VLAD pair selection (csrc/vlad.cu) with the reference's arithmetic (oracle/vlad_oracle.py)."""
import math
import os

import numpy as np
import pytest

from oracle import vlad_oracle as vo
from opensfm_b200 import matching, pairs_selection as ps, synthetic as syn

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vlad_words_64.npz")
CFG = {"lowes_ratio": 0.8}


def _words():
    return np.load(GOLDEN)["words"]


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _engine_unnormalized(features, centers, u8=False):
    pm = matching.PairMatcher()
    pm.add("a", features.astype(np.uint8) if u8 else features, uint8_is_l2=u8)
    assert pm.compute_vlad(["a"], centers) == ["a"]
    return pm.vlad_descriptor("a", normalized=False), pm.vlad_descriptor("a")


# ---- unnormalised VLAD, bit for bit ------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 31, 4000, 8000])
@pytest.mark.parametrize("u8", [False, True])
def test_unnormalized_vlad_bit_exact_hahog(n, u8):
    words = _words()
    f = syn.hahog_like_descriptors(n, 100 + n)
    got, _ = _engine_unnormalized(f, words, u8)
    assert np.array_equal(_bits(got), _bits(vo.compute_vlad_descriptor(f, words)))


@pytest.mark.parametrize("dim,nc", [(2, 2), (3, 5), (3, 40), (128, 64), (128, 70)])
def test_unnormalized_vlad_bit_exact_dims(dim, nc):
    rng = np.random.RandomState(dim * 100 + nc)
    f = rng.normal(0, 3, (2500, dim)).astype(np.float32)
    c = rng.normal(0, 3, (nc, dim)).astype(np.float32)
    got = ps.unnormalized_vlad(f, c)
    assert np.array_equal(_bits(got), _bits(vo.compute_vlad_descriptor(f, c)))


def test_exact_ties_first_centre_wins():
    words = _words().copy()
    words[40] = words[7]                       # two identical centres: every feature of 7 ties with 40
    f = np.repeat(words[7:8], 50, axis=0) + np.arange(50, dtype=np.float32)[:, None] * 0.05
    f[25:] = (words[3] + words[9]) / 2         # midway between two centres: equal squared distances
    got, _ = _engine_unnormalized(f, words)
    want = vo.compute_vlad_descriptor(f, words)
    assert np.array_equal(_bits(got), _bits(want))
    assert np.all(got.reshape(64, 128)[40] == 0) and np.any(got.reshape(64, 128)[7] != 0)


def test_near_ties_one_ulp_apart():
    """Features whose two best float32 squared distances differ by one ulp: centres (0, 0) and (2, 0), features
    (x, ~4096) with x in (0.5, 1.5), where the y term (~2^24) absorbs all but the last bit of the x terms' difference."""
    rng = np.random.RandomState(11)
    c = np.array([[0.0, 0.0], [2.0, 0.0]], np.float32)
    f = np.stack([rng.uniform(0.5, 1.5, 4000), 4096 + rng.uniform(-64, 64, 4000)], 1).astype(np.float32)
    d = [(f[:, 0] - cc[0]) * (f[:, 0] - cc[0]) + (f[:, 1] - cc[1]) * (f[:, 1] - cc[1]) for cc in c]
    f = f[np.abs(d[0].view(np.int32).astype(np.int64) - d[1].view(np.int32)) == 1]
    assert len(f) > 1000
    got = ps.unnormalized_vlad(f, c)
    assert np.array_equal(_bits(got), _bits(vo.compute_vlad_descriptor(f, c)))
    assert np.all(got != 0)   # both centres receive features


# ---- the reference's known-answer tests on the engine (opensfm/test/test_vlad.py) -------------------------------
def test_known_answer_unnormalized_vlad():
    res = ps.unnormalized_vlad(np.array([[0, 1.1]]), np.array([[1.0, 0.0], [0.0, 1.0]]))
    assert res is not None
    assert res[0] == res[1] == res[2] == 0
    assert pytest.approx(res[3], 1e-6) == 0.1
    assert ps.unnormalized_vlad(np.zeros((3, 4), np.float32), np.zeros((2, 3), np.float32)) is None
    assert ps.unnormalized_vlad(np.zeros((3, 3), np.uint8), np.zeros((2, 3), np.float32)) is None


def test_known_answer_signed_square_root_normalize():
    v = np.array([1, 0.01])
    pm = matching.PairMatcher()
    pm.add("x", v[None].astype(np.float32))
    res = pm.vlad_histograms(["x"], np.zeros((1, 2), np.float32))["x"]
    assert pytest.approx(np.linalg.norm(res), 1e-6) == 1
    assert pytest.approx(v[0] / v[1], 1e-6) == 10 * res[0] / res[1]


def test_known_answer_vlad_distances_order():
    histograms = {"im1": np.array([1, 0, 0]), "im2": np.array([0, 1, 0]),
                  "im3": np.array([1, 1, 0]) / np.linalg.norm([1, 1, 0])}
    im_res, distance_res, other_res = matching.vlad_distances("im1", ["im2", "im3"], histograms)
    assert im_res == "im1" and len(distance_res) == 2 and other_res == ["im2", "im3"]
    order_res = np.argsort(distance_res)
    assert other_res[order_res[0]] == "im3" and other_res[order_res[1]] == "im2"


# ---- normalised histograms ----------------------------------------------------------------------------------------
def test_histograms_normalised_and_skipped_sets():
    words = _words()
    pm = matching.PairMatcher()
    for i, n in enumerate([0, 1, 31, 4000, 8000]):
        pm.add(i, syn.hahog_like_descriptors(n, 300 + i))
    pm.add("u8", syn.hahog_like_descriptors(500, 9).astype(np.uint8), uint8_is_l2=True)
    pm.add("hamming", syn.binary_descriptors(200, 1, 61))
    pm.add("dim64", syn.hahog_like_descriptors(100, 2, 64))
    keys = [0, 1, 2, 3, 4, "u8", "hamming", "dim64"]
    hist = pm.vlad_histograms(keys, words)
    assert sorted(hist, key=str) == sorted([0, 1, 2, 3, 4, "u8"], key=str)
    assert pm.has_vlad("hamming") is False and pm.has_vlad("dim64") is False and pm.has_vlad("never") is None
    assert np.isnan(hist[0]).all()
    ulps = 0
    for k in [1, 2, 3, 4, "u8"]:
        un = pm.vlad_descriptor(k, normalized=False)
        want = vo.signed_square_root_normalize(un.copy(), fp64_sum=True)
        ulp = np.spacing(np.abs(want).astype(np.float32))
        assert np.all(np.abs(hist[k] - want) <= 2 * ulp), k
        ulps = max(ulps, int((np.abs(hist[k] - want) / ulp).max()))
        ref = vo.signed_square_root_normalize(un.copy())   # the reference's float32 BLAS norm
        assert np.allclose(hist[k], ref, rtol=2e-6, atol=0)
    print("normalised histograms: max %d ulp from the oracle" % ulps)


def test_non_finite_descriptors_and_centres_rejected():
    words = _words()
    pm = matching.PairMatcher()
    bad = syn.hahog_like_descriptors(10, 1)
    bad[3, 5] = np.inf
    pm.add("bad", bad)
    with pytest.raises(ValueError):
        pm.compute_vlad(["bad"], words)
    pm.add("ok", syn.hahog_like_descriptors(10, 2))
    w = words.copy()
    w[2, 2] = np.nan
    with pytest.raises(ValueError):
        pm.compute_vlad(["ok"], w)
    assert pm.compute_vlad(["ok"], words) == ["ok"]


# ---- distances and selection over 500 images ----------------------------------------------------------------------
N_IMAGES = 500


@pytest.fixture(scope="module")
def scene():
    words = _words()
    pm = matching.PairMatcher()
    rng = np.random.RandomState(21)
    base = [syn.hahog_like_descriptors(300, 1000 + g) for g in range(25)]
    items = []
    for i in range(N_IMAGES):
        g = base[i % 25]
        n = int(rng.randint(150, 300))
        f = np.clip(g[rng.choice(300, n, replace=False)] + rng.randint(-3, 4, (n, 128)), 0, 255).astype(np.float32)
        if i % 97 == 5:
            f = f[:0]                                   # no features: an all-NaN histogram
        items.append(("im%03d" % i, f))
    items.append(("im%03d" % N_IMAGES, items[10][1].copy()))   # a duplicate image: distance 0 to im010
    pm.add_many(items)
    names = [k for k, _ in items]
    hist = pm.vlad_histograms(names, words)
    exifs = {n: {"camera": "cam%d" % (i % 3)} for i, n in enumerate(names)}
    # the engine's fp64 distances, row by row, through matching.vlad_distances (same kernel and summation order)
    H = np.stack([hist[n] for n in names])
    D = np.empty((len(names), len(names)))
    for i, n in enumerate(names):
        _, d, others = matching.vlad_distances(n, names, hist)
        D[i, [names.index(o) for o in others]] = d
        D[i, i] = 0.0
    return dict(pm=pm, names=names, hist=hist, exifs=exifs, H=H, D=D, items=items)


def test_distances_fp64_and_symmetric(scene):
    H, D = scene["H"].astype(np.float64), scene["D"]
    ok = ~np.isnan(H).any(axis=1)
    sub = np.flatnonzero(ok)[:120]
    ref = np.sqrt(((H[sub][:, None, :] - H[sub][None, :, :]) ** 2).sum(axis=2))
    got = D[np.ix_(sub, sub)]
    assert np.all(np.abs(got - ref) <= 1e-12 * np.maximum(ref, 1e-300))
    Dm = np.where(np.isnan(D), -1.0, D)
    assert np.array_equal(Dm.view(np.uint64), Dm.T.view(np.uint64))
    assert np.isnan(D[~ok][:, ok]).all()
    assert D[10, N_IMAGES] == 0.0


def _same(got, want):
    assert set(got) == set(want), (len(set(got) ^ set(want)), sorted(set(got) ^ set(want))[:5])
    for p, d in want.items():
        assert (math.isnan(d) and math.isnan(got[p])) or got[p] == d, (p, got[p], d)


@pytest.mark.parametrize("enforce", [False, True])
@pytest.mark.parametrize("k", [0, 1, 10, 600])
@pytest.mark.parametrize("masked", [False, True])
def test_selection_matches_oracle(scene, k, enforce, masked):
    names, D, exifs = scene["names"], scene["D"], scene["exifs"]
    idx = {n: i for i, n in enumerate(names)}
    refs, cands = names[:300], names[100:]
    candidates = None
    if masked:
        rng = np.random.RandomState(k + 3 * enforce)
        candidates = {r: [c for c in cands if rng.rand() < 0.3] for r in refs[::2]}
    got = ps.match_candidates_with_vlad(scene["pm"], refs, cands, exifs, k, enforce, candidates)
    want = vo.match_candidates_with_vlad(scene["hist"], refs, cands, exifs, k, enforce, candidates,
                                         distance=lambda a, b: float(D[idx[a], idx[b]]))
    _same(got, want)
    if k:
        assert len(got) > 0


def test_selection_against_reference_float32_pipeline(scene):
    """The reference's own distances are float32 norms ordered by np.argsort (unstable): per reference image the
    selected sets agree except for candidates whose float32 distance lies within 1e-6 relative of the row's k-th."""
    pm, names, hist = scene["pm"], scene["names"], scene["hist"]
    k = 10
    refs = [n for n in names if not np.isnan(hist[n]).any()]   # all-NaN rows: covered by the stable oracle above
    cands = sorted(names)
    excluded = 0
    for im, (cols, _) in zip(refs, pm.vlad_select(refs, cands, k)):
        d32, others = vo.compute_vlad_distances(hist, im, names, lambda a, b: vo.vlad_distance(hist[a], hist[b], False))
        order = np.argsort(d32)
        kth = d32[order[k - 1]]
        want = {others[i] for i in order[:k]}
        mine = {cands[j] for j in cols}
        near = {o for o, d in zip(others, d32) if abs(d - kth) <= 1e-6 * kth}
        assert (want ^ mine) <= near, (im, want ^ mine)
        excluded += len(want - mine)
    print("reference float32 pipeline: %d candidates at the cut differ" % excluded)


def test_selected_pairs_feed_the_matcher(scene):
    pm, names, exifs = scene["pm"], scene["names"], scene["exifs"]
    pairs = sorted(ps.match_candidates_with_vlad(pm, names[:60], names, exifs, 4, True))
    got = pm.match_pairs(pairs, CFG)
    fresh = matching.PairMatcher()
    needed = sorted({i for p in pairs for i in p})
    items = dict(scene["items"])
    fresh.add_many([(k, items[k]) for k in needed])
    want = fresh.match_pairs(pairs, CFG)
    assert len(pairs) > 60
    for p in pairs:
        assert np.array_equal(got[p], want[p]), p


def test_selection_over_several_row_blocks():
    """20000 candidates: a 256 MB distance block holds 1664 reference rows, so 4000 references take three blocks.
    Each reference must get the same selection as in a call of its own 500-reference chunk (one block), with its
    rows of the candidate mask and its camera label.  Integer descriptors give many exactly tied distances."""
    rng = np.random.RandomState(5)
    n, nref, k = 20000, 4000, 10
    pm = matching.PairMatcher()
    pm.add_many([(i, rng.randint(0, 4, (3, 2)).astype(np.float32)) for i in range(n)])
    assert len(pm.compute_vlad(range(n), np.array([[0.5, 0.5], [2.5, 2.5]], np.float32))) == n
    cands = list(range(n))
    refs = list(range(0, 2 * nref, 2))
    labels = np.array(refs + cands) % 3
    mask = rng.rand(nref, n) < 0.5
    whole = pm.vlad_select(refs, cands, k, mask, labels)
    assert all(0 < len(c) <= 2 * k for c, _ in whole)
    for r0 in range(0, nref, 500):
        part = pm.vlad_select(refs[r0:r0 + 500], cands, k, mask[r0:r0 + 500],
                              np.concatenate([labels[r0:r0 + 500], labels[nref:]]))
        for r, ((c1, d1), (c2, d2)) in enumerate(zip(whole[r0:r0 + 500], part)):
            assert np.array_equal(c1, c2) and np.array_equal(d1, d2), r0 + r
