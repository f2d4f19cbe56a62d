"""GPU parity of BoW pair selection (csrc/bow.cu): words against live cv2 BruteForce knnMatch, histograms, distances
and the selection against the reference's formulas (oracle/bow_oracle.py)."""
import math
import os

import cv2
import numpy as np
import pytest

from oracle import bow_oracle as bo
from opensfm_b200 import bow, matching, pairs_selection as ps, synthetic as syn

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bow_words_1024.npz")
CFG = {"lowes_ratio": 0.8, "bow_num_checks": 20}


def _fixture():
    z = np.load(GOLDEN)
    return z["words"], z["frequencies"]


def _vocab_10000():
    """10000 words synthesised from the fixture: its 1024 words and seeded perturbations of them."""
    w, f = _fixture()
    rng = np.random.RandomState(10000)
    extra = w[rng.randint(0, len(w), 10000 - len(w))] + rng.normal(0, 4, (10000 - len(w), w.shape[1]))
    words = np.concatenate([w, np.clip(extra, 0, 255)]).astype(np.float32)
    freq = np.concatenate([f, rng.randint(1, 3000, 10000 - len(w))]).astype(np.int64)
    return words, freq


def _cv2_words(desc, vocab, k):
    m = cv2.DescriptorMatcher_create("BruteForce")
    kout = min(k, len(vocab))
    if len(desc) == 0:
        return np.zeros((0, kout), np.int32)
    return np.array([[n.trainIdx for n in row] for row in m.knnMatch(np.asarray(desc, np.float32), vocab, k=k)],
                    dtype=np.int32).reshape(len(desc), kout)


def _descriptors(kind, n, seed, dim=128):
    if kind == "hahog":
        return syn.hahog_like_descriptors(n, seed, dim)
    if kind == "float":
        return np.random.RandomState(seed).normal(30, 20, (n, dim)).astype(np.float32)
    raise ValueError(kind)


def _engine_words(desc, vocab, k, u8=False):
    pm = matching.PairMatcher()
    pm.add("a", desc.astype(np.uint8) if u8 else desc, uint8_is_l2=u8)
    return pm.compute_words(["a"], bow.BagOfWords(vocab, np.ones(len(vocab))), k)["a"]


# ---- words, index for index -----------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 2, 50, 64])
@pytest.mark.parametrize("kind", ["hahog", "u8", "float"])
def test_words_match_cv2_fixture(k, kind):
    vocab, _ = _fixture()
    desc = _descriptors("float" if kind == "float" else "hahog", 4000, 7 + k)
    if kind == "u8":
        desc = np.clip(desc, 0, 255).astype(np.uint8).astype(np.float32)
    got = _engine_words(desc, vocab, k, u8=(kind == "u8"))
    assert np.array_equal(got, _cv2_words(desc, vocab, k))


@pytest.mark.parametrize("dim", [3, 61, 128, 130])
@pytest.mark.parametrize("nwords", [1, 49, 50, 51])
def test_words_match_cv2_dims(dim, nwords):
    rng = np.random.RandomState(dim * 100 + nwords)
    vocab = rng.normal(0, 3, (nwords, dim)).astype(np.float32)
    desc = rng.normal(0, 3, (700, dim)).astype(np.float32)
    got = bow.BagOfWords(vocab, np.ones(nwords)).map_to_words(desc, 50, "BRUTEFORCE")
    assert got.shape == (700, min(50, nwords))
    assert np.array_equal(got, _cv2_words(desc, vocab, 50))


@pytest.mark.parametrize("n", [0, 1, 4000])
def test_words_match_cv2_10000_vocabulary(n):
    vocab, freq = _vocab_10000()
    desc = syn.hahog_like_descriptors(n, 40 + n)
    got = bow.BagOfWords(vocab, freq).map_to_words(desc, 50)
    assert got.shape == (n, 50)
    assert np.array_equal(got, _cv2_words(desc, vocab, 50))


def test_word_ties_go_to_the_lower_index():
    vocab, _ = _fixture()
    v = vocab[:200].copy()
    v[150] = v[20]                                  # exact duplicates
    v[151] = v[3]
    desc = np.concatenate([v[[20, 3, 150]] + 0.25, syn.hahog_like_descriptors(300, 3)]).astype(np.float32)
    got = bow.BagOfWords(v, np.ones(len(v))).map_to_words(desc, 50)
    assert np.array_equal(got, _cv2_words(desc, v, 50))
    assert got[0, 0] == 20 and got[1, 0] == 3


def test_sqrt_space_ties_one_ulp_apart():
    """Words (0, 0) and (2, 0), features (x, ~4096): the two squared distances (~2^24) differ by one ulp and have the
    same float32 square root, so cv2 ranks them equal and takes the lower word."""
    rng = np.random.RandomState(11)
    v = np.array([[2.0, 0.0], [0.0, 0.0], [2.0, 0.0], [0.0, -3.0]], np.float32)
    f = np.stack([rng.uniform(0.5, 1.5, 4000), 4096 + rng.uniform(-64, 64, 4000)], 1).astype(np.float32)
    d = [(f[:, 0] - c[0]) * (f[:, 0] - c[0]) + (f[:, 1] - c[1]) * (f[:, 1] - c[1]) for c in v[:2]]
    f = f[(np.abs(d[0].view(np.int32).astype(np.int64) - d[1].view(np.int32)) == 1) & (np.sqrt(d[0]) == np.sqrt(d[1]))]
    assert len(f) > 500
    got = bow.BagOfWords(v, np.ones(4)).map_to_words(f, 3)
    assert np.array_equal(got, _cv2_words(f, v, 3))
    assert np.array_equal(got[:, :3], np.tile([0, 1, 2], (len(f), 1)))


def test_many_sets_in_one_call_and_invalid_sets():
    vocab, freq = _fixture()
    bows = bow.BagOfWords(vocab, freq)
    pm = matching.PairMatcher()
    sizes = [0, 1, 5, 63, 64, 65, 4000, 129]
    items = [(i, syn.hahog_like_descriptors(n, 60 + i)) for i, n in enumerate(sizes)]
    pm.add_many(items)
    pm.add("u8", syn.hahog_like_descriptors(500, 9).astype(np.uint8), uint8_is_l2=True)
    pm.add("hamming", syn.binary_descriptors(200, 1, 61))
    pm.add("dim64", syn.hahog_like_descriptors(100, 2, 64))
    keys = [k for k, _ in items] + ["u8", "hamming", "dim64"]
    together = pm.compute_words(keys, bows, 50)
    assert sorted(together, key=str) == sorted([k for k, _ in items] + ["u8"], key=str)
    for k, f in items + [("u8", syn.hahog_like_descriptors(500, 9).astype(np.uint8).astype(np.float32))]:
        assert np.array_equal(together[k], _cv2_words(f, vocab, 50)), k
        alone = pm.compute_words([k], bows, 50)[k]
        assert np.array_equal(together[k], alone), k


def test_non_finite_inputs_rejected():
    vocab, freq = _fixture()
    pm = matching.PairMatcher()
    bad = syn.hahog_like_descriptors(10, 1)
    bad[3, 5] = np.nan
    pm.add("bad", bad)
    with pytest.raises(ValueError):
        pm.compute_words(["bad"], bow.BagOfWords(vocab, freq), 50)
    pm.add("ok", syn.hahog_like_descriptors(10, 2))
    v = vocab.copy()
    v[7, 1] = np.inf
    with pytest.raises(ValueError):
        pm.compute_words(["ok"], bow.BagOfWords(v, freq), 50)
    assert list(pm.compute_words(["ok"], bow.BagOfWords(vocab, freq), 50)) == ["ok"]
    with pytest.raises(ValueError):
        pm.compute_words(["ok"], bow.BagOfWords(vocab, freq), 65)


# ---- histograms and distances -----------------------------------------------------------------------------------
def test_histograms_equal_the_reference_formula():
    vocab, freq = _fixture()
    bows = bow.BagOfWords(vocab, freq)
    pm = matching.PairMatcher()
    sizes = [0, 1, 8, 9, 300, 4000]
    pm.add_many([(i, syn.hahog_like_descriptors(n, 80 + i)) for i, n in enumerate(sizes)])
    words = pm.compute_words(range(len(sizes)), bows, 50)
    hist = pm.bow_histograms(range(len(sizes)), bows)
    assert sorted(hist) == [3, 4, 5]
    assert pm.has_bow(0) is False and pm.has_bow(2) is False and pm.has_bow(3) is True and pm.has_bow("x") is None
    w = bo.weights(freq)
    for i in hist:
        want = bo.histogram(words[i][:, 0], w)
        assert np.array_equal(hist[i].view(np.uint64), want.view(np.uint64)), i
        assert np.array_equal(bows.histogram(words[i][:, 0]).view(np.uint64), want.view(np.uint64))
    # frequencies equal to their sum: zero weights, 0/0 = NaN as numpy gives
    with np.errstate(divide="ignore", invalid="ignore"):
        z = bow.BagOfWords(vocab[:4], np.array([0, 0, 5, 0]))
        want = bo.histogram(np.array([2, 2, 2]), bo.weights(np.array([0, 0, 5, 0])))
    got = z.histogram(np.array([2, 2, 2]))
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.all(got[~np.isnan(got)] == want[~np.isnan(want)])


N_IMAGES = 300


@pytest.fixture(scope="module")
def scene():
    vocab, freq = _fixture()
    bows = bow.BagOfWords(vocab, freq)
    pm = matching.PairMatcher()
    rng = np.random.RandomState(21)
    base = [syn.hahog_like_descriptors(300, 1000 + g) for g in range(15)]
    items = []
    for i in range(N_IMAGES):
        g = base[i % 15]
        n = int(rng.randint(100, 300))
        f = np.clip(g[rng.choice(300, n, replace=False)] + rng.randint(-3, 4, (n, 128)), 0, 255).astype(np.float32)
        if i % 97 == 5:
            f = f[:6]                                   # too few words: no histogram
        items.append(("im%03d" % i, f))
    items.append(("im%03d" % N_IMAGES, items[10][1].copy()))   # a duplicate image: distance 0 to im010
    pm.add_many(items)
    names = [k for k, _ in items]
    words = pm.compute_words(names, bows, 50)
    hist = pm.bow_histograms(names, bows)
    exifs = {n: {"camera": "cam%d" % (i % 3)} for i, n in enumerate(names)}
    return dict(pm=pm, names=names, hist=hist, exifs=exifs, items=items, words=words, bows=bows)


def test_distances_bit_exact_and_symmetric(scene):
    hist = scene["hist"]
    keys = sorted(hist)[:150]
    H = np.stack([hist[k] for k in keys])
    for i, k in enumerate(keys):
        _, d, others = ps.bow_distances(k, keys, hist)
        assert others == keys[:i] + keys[i + 1:]
        want = [np.fabs(H[i] - hist[o]).sum() for o in others]
        assert np.array_equal(np.array(d).view(np.uint64), np.array(want).view(np.uint64)), k
    D = np.stack([bow.bow_distance_rows(H, i) for i in range(len(keys))])
    assert np.array_equal(D.view(np.uint64), D.T.view(np.uint64))
    assert scene["bows"].bow_distance(None, None, H[0], H[1]) == np.fabs(H[0] - H[1]).sum()


def _same(got, want):
    assert set(got) == set(want), (len(set(got) ^ set(want)), sorted(set(got) ^ set(want))[:5])
    for p, d in want.items():
        assert (math.isnan(d) and math.isnan(got[p])) or got[p] == d, (p, got[p], d)


@pytest.mark.parametrize("enforce", [False, True])
@pytest.mark.parametrize("k", [0, 1, 10, 600])
@pytest.mark.parametrize("cands", ["all", "dict", "shuffled"])
def test_selection_matches_oracle(scene, k, enforce, cands):
    names, exifs, hist = scene["names"], scene["exifs"], scene["hist"]
    refs, pool = names[:200], names[50:]
    candidates = None
    if cands == "shuffled":
        rng = np.random.RandomState(3 + k)
        pool = [pool[i] for i in rng.permutation(len(pool))]
    if cands == "dict":
        rng = np.random.RandomState(k + 3 * enforce)
        candidates = {r: [pool[i] for i in rng.permutation(len(pool)) if rng.rand() < 0.3] for r in refs[::2]}
    got = ps.match_candidates_with_bow(scene["pm"], refs, pool, exifs, k, enforce, candidates)
    want = bo.match_candidates_with_bow(hist, refs, pool, exifs, k, enforce, candidates)
    _same(got, want)
    if k:
        assert len(got) > 0


def test_empty_preemption_gives_no_pairs(scene):
    names, exifs = scene["names"], scene["exifs"]
    assert ps.match_candidates_with_bow(scene["pm"], names, names, exifs, 10, False, {}) == {}
    got = ps.match_candidates_with_bow(scene["pm"], names[:3], names, exifs, 10, False, None)
    assert got == bo.match_candidates_with_bow(scene["hist"], names[:3], names, exifs, 10, False, None) and len(got) > 10


def test_words_and_pairs_feed_the_matchers(scene):
    pm, names, exifs, items = scene["pm"], scene["names"], scene["exifs"], dict(scene["items"])
    vocab = scene["bows"].words32
    for a, b in [(names[0], names[15]), (names[1], names[2])]:
        wa, wb = scene["words"][a], scene["words"][b]
        assert np.array_equal(wa, _cv2_words(items[a], vocab, 50)) and np.array_equal(wb, _cv2_words(items[b], vocab, 50))
        got = matching.match_words(items[a], wa, items[b], wb, CFG)
        want = matching.match_words(items[a], _cv2_words(items[a], vocab, 50), items[b], _cv2_words(items[b], vocab, 50), CFG)
        assert np.array_equal(got, want)
    pairs = sorted(ps.match_candidates_with_bow(pm, names[:60], names, exifs, 4, True))
    got = pm.match_pairs(pairs, {"lowes_ratio": 0.8})
    fresh = matching.PairMatcher()
    fresh.add_many([(k, items[k]) for k in sorted({i for p in pairs for i in p})])
    want = fresh.match_pairs(pairs, {"lowes_ratio": 0.8})
    assert len(pairs) > 60
    for p in pairs:
        assert np.array_equal(got[p], want[p]), p


def test_selection_over_several_row_blocks():
    """20000 candidates: a 256 MB distance block holds 1664 reference rows, so 4000 references take three blocks.
    Each reference must get the same selection as in a call of its own 500-reference chunk (one block), with its
    candidate order and its camera label.  Few words give many exactly tied distances."""
    rng = np.random.RandomState(5)
    n, nref, k = 20000, 4000, 10
    vocab = np.array([[0.0, 0.0], [3.0, 0.0], [0.0, 3.0], [3.0, 3.0]], np.float32)
    bows = bow.BagOfWords(vocab, np.array([5, 3, 2, 7]))
    pm = matching.PairMatcher()
    pm.add_many([(i, rng.randint(0, 4, (9 + i % 3, 2)).astype(np.float32)) for i in range(n)])
    pm.compute_words(range(n), bows, 1)
    assert len(pm.bow_histograms(range(n), bows)) == n
    cands = list(range(n))
    refs = list(range(0, 2 * nref, 2))
    labels = np.array(refs + cands) % 3
    order = np.where(rng.rand(nref, n) < 0.5, rng.randint(0, 1 << 20, (nref, n)), -1)
    for r in range(nref):   # distinct positions per reference
        sel = order[r] >= 0
        order[r, sel] = rng.permutation(int(sel.sum()))
    whole = pm.bow_select(refs, cands, k, order, labels)
    assert all(0 < len(c) <= 2 * k for c, _ in whole)
    for r0 in range(0, nref, 500):
        part = pm.bow_select(refs[r0:r0 + 500], cands, k, order[r0:r0 + 500],
                             np.concatenate([labels[r0:r0 + 500], labels[nref:]]))
        for r, ((c1, d1), (c2, d2)) in enumerate(zip(whole[r0:r0 + 500], part)):
            assert np.array_equal(c1, c2) and np.array_equal(d1, d2), r0 + r
