"""CPU pins of the BoW oracle (oracle/bow_oracle.py): numpy's pairwise summation order, cv2's word ranking, and
the reference's pair construction against brute force."""
import math
import os

import cv2
import numpy as np
import pytest

from oracle import bow_oracle as bo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bow_words_1024.npz")


@pytest.mark.parametrize("n", [1, 7, 8, 9, 127, 128, 129, 1000, 8192, 8193, 10000, 65536])
def test_pairwise_sum_is_numpy_sum(n):
    rng = np.random.RandomState(n)
    for t in range(5):
        a = rng.gamma(0.3, 1.0, n) * (rng.rand(n) < 0.2) * np.exp(rng.normal(0, 3, n))
        assert bo.pairwise_sum(a) == np.sum(a) == np.fabs(a).sum()
        leaves, prog = bo.pairwise_leaves(n)
        st = []
        for op in prog:
            if op >= 0:
                s, m = leaves[op]
                st.append(bo.pairwise_sum(a[s:s + m]))
            else:
                b = st.pop()
                st.append(np.float64(st.pop() + b))
        assert len(st) == 1 and st[0] == np.sum(a)


@pytest.mark.parametrize("k", [1, 2, 50])
def test_cv2_knn_is_a_stable_argsort(k):
    z = np.load(GOLDEN)
    vocab = z["words"].copy()
    vocab[900] = vocab[17]                      # duplicated rows: exact ties go to the lower index
    vocab[901] = vocab[400]
    rng = np.random.RandomState(k)
    desc = np.round(rng.gamma(0.6, 30.0, (400, 128))).clip(0, 255).astype(np.float32)
    desc[:10] = vocab[[17, 400, 900, 901, 3, 5, 7, 9, 11, 13]] + 0.5
    got = np.array([[m.trainIdx for m in row] for row in
                    cv2.DescriptorMatcher_create("BruteForce").knnMatch(desc, vocab, k=k)], dtype=np.int32)
    assert np.array_equal(got, bo.knn_words(desc, vocab, k))
    assert got[0, 0] == 17 and got[2, 0] == 17 and got[1, 0] == 400


def test_histogram_formula():
    z = np.load(GOLDEN)
    w = bo.weights(z["frequencies"])
    words = np.random.RandomState(1).randint(0, len(w), 300)
    h = np.bincount(words, minlength=len(w)) * np.log(z["frequencies"].sum() / z["frequencies"])
    assert np.array_equal(bo.histogram(words, w), h / h.sum())
    got = bo.load_histograms({"a": np.zeros((8, 2), np.int32), "b": np.zeros((9, 2), np.int32)}, w)
    assert list(got) == ["b"]


def _brute_pairs(hist, candidates, exifs, k, enforce):
    out = {}
    for im, cands in candidates.items():
        if im not in hist:
            continue
        others = [c for c in cands if c != im and c in hist]
        rows = [(float(np.fabs(hist[im] - hist[c]).sum()), j, c) for j, c in enumerate(others)]
        rows.sort(key=lambda r: (math.isnan(r[0]), r[0] if not math.isnan(r[0]) else 0.0, r[1]))
        if enforce:
            same = [r for r in rows if exifs[r[2]]["camera"] == exifs[im]["camera"]][:k]
            diff = [r for r in rows if exifs[r[2]]["camera"] != exifs[im]["camera"]][:k]
            keep = same + diff
        else:
            keep = rows[:k]
        for d, _, c in keep:
            out[bo.sorted_pair(im, c)] = d
    return out


@pytest.mark.parametrize("enforce", [False, True])
@pytest.mark.parametrize("k", [0, 1, 3, 50])
def test_construct_pairs_matches_brute_force(k, enforce):
    rng = np.random.RandomState(k + 7 * enforce)
    names = ["im%02d" % i for i in range(30)]
    w = rng.uniform(0.1, 3.0, 40)
    hist = bo.load_histograms({n: rng.randint(0, 40, (rng.randint(5, 60), 3)) for n in names}, w)
    hist["im05"] = hist.get("im09", hist[next(iter(hist))]).copy()   # exact ties
    exifs = {n: {"camera": "cam%d" % (i % 3)} for i, n in enumerate(names)}
    refs, cands = names[::2], list(reversed(names[3:]))             # an unsorted candidate order
    got = bo.match_candidates_with_bow(hist, refs, cands, exifs, k, enforce)
    want = _brute_pairs(hist, {im: cands for im in refs}, exifs, k, enforce) if k > 0 else {}
    assert set(got) == set(want)
    for p in want:
        assert got[p] == want[p]


def test_candidates_none_and_empty():
    names = ["a", "b", "c", "d"]
    hist = {n: np.eye(4)[i] for i, n in enumerate(names)}
    exifs = {n: {"camera": "x"} for n in names}
    assert bo.match_candidates_with_bow(hist, names, names, exifs, 2, False, {}) == {}
    full = bo.match_candidates_with_bow(hist, names, names, exifs, 3, False, None)
    assert set(full) == {bo.sorted_pair(a, b) for a in names for b in names if a != b}
    one = bo.match_candidates_with_bow(hist, names, names, exifs, 3, False, {"a": ["c", "b"]})
    assert set(one) == {("a", "b"), ("a", "c")}
