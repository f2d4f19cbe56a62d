"""The matcher's per-set resident arrays (bearings, VLAD, BoW words and histograms), its shared VLAD / BoW selection
workspaces and the argument handling of the two selection entry points (csrc/select_common.cuh)."""
import ctypes
import os

import numpy as np
import pytest

from opensfm_b200 import _lib, bow, matching, synthetic as syn

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _bags(words):
    return bow.BagOfWords(words, np.arange(1, len(words) + 1))


def test_resident_arrays_go_back_on_remove_and_clear():
    centers = np.load(os.path.join(GOLDEN, "vlad_words_64.npz"))["words"]
    bags = _bags(np.load(os.path.join(GOLDEN, "bow_words_1024.npz"))["words"])
    desc = {i: syn.hahog_like_descriptors(200 + 40 * i, i, centers.shape[1]) for i in range(4)}
    rng = np.random.RandomState(0)
    pm = matching.PairMatcher()

    def fill(keys):
        for key in keys:
            pm.add(key, desc[key])
            b = rng.normal(size=(len(desc[key]), 3))
            pm.set_bearings(key, b / np.linalg.norm(b, axis=1)[:, None])
        assert pm.compute_vlad(keys, centers) == keys
        assert sorted(pm.compute_words(keys, bags, 3)) == keys
        assert sorted(pm.bow_histograms(keys, bags)) == keys

    def remove(key):
        _lib.check(pm._m.L.osfm_matcher_remove(pm._m.h, pm._ids.pop(key)))

    pm.add(0, desc[0])
    reserved0, in_use0 = pm.device_bytes()
    fill([1, 2, 3])
    reserved1, in_use1 = pm.device_bytes()
    assert in_use1 > in_use0
    for key in (1, 2, 3):
        remove(key)
    assert pm.device_bytes()[1] == in_use0
    fill([1, 2, 3])
    assert pm.device_bytes() == (reserved1, in_use1)
    pm.clear()
    assert pm.device_bytes() == (reserved1, 0)
    pm.add(0, desc[0])
    fill([1, 2, 3])
    assert pm.device_bytes() == (reserved1, in_use1)


def _selection_matcher(n):
    """n images of 12 integer-valued 2-D features, with VLAD descriptors and BoW histograms of a 4-word vocabulary:
    many exactly tied distances."""
    rng = np.random.RandomState(7)
    pm = matching.PairMatcher()
    pm.add_many([(i, rng.randint(0, 4, (12, 2)).astype(np.float32)) for i in range(n)])
    assert len(pm.compute_vlad(range(n), np.array([[0.5, 0.5], [2.5, 2.5]], np.float32))) == n
    bags = _bags(np.array([[0, 0], [0, 3], [3, 0], [3, 3]], np.float32))
    pm.compute_words(range(n), bags, 1)
    assert len(pm.bow_histograms(range(n), bags)) == n
    return pm


def test_alternating_vlad_and_bow_selection_equals_fresh_matchers():
    """6000 x 6000 distances need two 256 MB row blocks; the small calls need one."""
    n, k = 6000, 5
    rng = np.random.RandomState(3)
    cands = list(range(n))
    small = list(range(0, n, 97))
    labels = {len(r): np.array(r + cands) % 3 for r in (small, cands)}
    mask = {len(r): rng.rand(len(r), n) < 0.7 for r in (small, cands)}
    order = {}
    for r in (small, cands):
        o = np.full((len(r), n), -1, np.int32)
        for i in range(len(r)):
            cols = rng.permutation(n)[:n // 2]
            o[i, cols] = np.arange(len(cols))
        order[len(r)] = o
    calls = [("vlad", small), ("bow", cands), ("vlad", cands), ("bow", small), ("vlad", small)]

    def run(pm, kind, refs):
        if kind == "vlad":
            return pm.vlad_select(refs, cands, k, mask[len(refs)], labels[len(refs)])
        return pm.bow_select(refs, cands, k, order[len(refs)], labels[len(refs)])

    pm = _selection_matcher(n)
    shared = [run(pm, kind, refs) for kind, refs in calls]
    for (kind, refs), got in zip(calls, shared):
        want = run(_selection_matcher(n), kind, refs)
        assert len(got) == len(want) == len(refs)
        assert any(len(c) for c, _ in got)
        for r, ((c1, d1), (c2, d2)) in enumerate(zip(got, want)):
            assert np.array_equal(c1, c2) and np.array_equal(d1, d2), (kind, len(refs), r)


@pytest.mark.parametrize("kind", ["vlad", "bow"])
def test_selection_entry_points_arguments(kind):
    L = _lib.load()
    fn = L.osfm_matcher_vlad_select if kind == "vlad" else L.osfm_matcher_bow_select
    name = "VLAD" if kind == "vlad" else "BoW"
    rng = np.random.RandomState(1)
    pm = matching.PairMatcher()
    pm.add_many([(i, rng.randint(0, 4, (12, 2)).astype(np.float32)) for i in range(3)])
    pm.add(3, rng.randint(0, 4, (12, 3)).astype(np.float32))   # another length
    pm.add(4, rng.randint(0, 4, (12, 2)).astype(np.float32))   # no VLAD / histogram
    if kind == "vlad":
        pm.compute_vlad([0, 1, 2], np.array([[0.5, 0.5], [2.5, 2.5]], np.float32))
        pm.compute_vlad([3], np.array([[0.5, 0.5, 0.5]], np.float32))
    else:
        pm.compute_words([0, 1, 2], _bags(np.array([[0, 0], [3, 3]], np.float32)), 1)
        pm.bow_histograms([0, 1, 2], _bags(np.array([[0, 0], [3, 3]], np.float32)))
        pm.compute_words([3], _bags(np.array([[0, 0, 0], [3, 3, 3], [0, 3, 0]], np.float32)), 1)
        pm.bow_histograms([3], _bags(np.array([[0, 0, 0], [3, 3, 3], [0, 3, 0]], np.float32)))
    ids = {key: np.array([pm._ids[key]], np.int32) for key in range(5)}
    pair = np.array([pm._ids[0], pm._ids[1]], np.int32)

    def call(nref, refs, ncand, cand_ids, k, offs, cols=None, dist=None, m=pm._m.h):
        code = fn(m, nref, _ptr(refs), ncand, _ptr(cand_ids), None, None, k, _ptr(offs), _ptr(cols), _ptr(dist))
        return code, (L.osfm_last_error().decode() if code else "")

    offs = np.full(3, 7, np.int64)
    assert call(0, None, 2, pair, 1, None) == (0, "")
    # no candidates or k = 0: zero offsets, before the outputs or any set is looked at
    unknown = np.array([123456, 123457], np.int32)
    assert call(2, unknown, 0, None, 1, offs) == (0, "") and offs.tolist() == [0, 0, 0]
    offs[:] = 7
    assert call(2, unknown, 2, pair, 0, offs) == (0, "") and offs.tolist() == [0, 0, 0]
    cols, dist = np.empty(4, np.int32), np.empty(4)
    assert call(2, pair, 2, pair, 1, offs) == (2, "null output arrays")
    assert call(2, pair, 2, pair, 1, offs, cols, dist) == (0, "")
    assert offs.tolist() == [0, 1, 2] and cols[:2].tolist() == [1, 0]
    assert call(-1, pair, 2, pair, 1, offs) == (2, "bad %s selection sizes" % name)
    assert call(2, None, 2, pair, 1, offs) == (2, "null arrays")
    assert call(2, pair, 2, pair, 1, offs, m=None) == (2, "null matcher")
    assert call(1, ids[0], 1, unknown[:1], 1, offs, cols, dist) == (2, "unknown descriptor set id")
    assert call(1, ids[0], 1, ids[3], 1, offs, cols, dist) == (2, "%s of different lengths" % (
        "VLAD descriptors" if kind == "vlad" else "BoW histograms"))
    assert call(1, ids[4], 1, ids[0], 1, offs, cols, dist) == (2, (
        "descriptor set has no VLAD descriptor (osfm_matcher_vlad_compute)" if kind == "vlad"
        else "descriptor set has no BoW histogram (osfm_matcher_bow_histograms)"))
