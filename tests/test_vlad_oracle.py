"""CPU pins of the VLAD oracle (oracle/vlad_oracle.py): the reference's own known-answer tests
(opensfm/test/test_vlad.py, all three) and agreement with plain restatements on random inputs."""
import math
import os

import numpy as np
import pytest

from oracle import vlad_oracle as vo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vlad_words_64.npz")


# ---- opensfm/test/test_vlad.py, on the oracle ------------------------------------------------------------------
def test_vlad_distances_order():
    im = "im1"
    other_ims = ["im2", "im3"]
    histograms = {"im1": np.array([1, 0, 0]), "im2": np.array([0, 1, 0]),
                  "im3": np.array([1, 1, 0]) / np.linalg.norm([1, 1, 0])}
    distance_res, other_res = vo.compute_vlad_distances(histograms, im, other_ims)
    assert len(distance_res) == len(other_ims)
    assert other_res == other_ims
    order_res = np.argsort(distance_res)
    assert other_ims[order_res[0]] == "im3"
    assert other_ims[order_res[1]] == "im2"


def test_signed_square_root_normalize():
    v = np.array([1, 0.01])
    res = vo.signed_square_root_normalize(v)
    assert pytest.approx(np.linalg.norm(res), 1e-6) == 1
    assert pytest.approx(v[0] / v[1], 1e-6) == 10 * res[0] / res[1]


def test_unnormalized_vlad():
    features = np.array([[0, 1.1]])
    centers = np.array([[1.0, 0.0], [0.0, 1.0]])
    res = vo.unnormalized_vlad(features, centers)
    assert res is not None
    assert res[0] == res[1] == res[2] == 0
    assert pytest.approx(res[3], 1e-6) == 0.1


# ---- restatements ------------------------------------------------------------------------------------------------
def _sequential(features, centers):
    """compute_vlad_descriptor one float32 scalar operation at a time, as the reference's loops run."""
    F = np.asarray(features, np.float32)
    C = np.asarray(centers, np.float32)
    v = np.zeros(C.shape, np.float32)
    for f in F:
        best, bc = vo.FLT_MAX, -1
        for j, c in enumerate(C):
            t = np.float32(f[0] - c[0])
            s = np.float32(t * t)
            for k in range(1, len(f)):
                t = np.float32(f[k] - c[k])
                s = np.float32(s + np.float32(t * t))
            if s < best:
                best, bc = s, j
        for k in range(len(f)):
            v[bc, k] = np.float32(v[bc, k] + np.float32(f[k] - C[bc, k]))
    return v.reshape(-1)


@pytest.mark.parametrize("n,dim,nc", [(0, 3, 4), (1, 2, 2), (37, 3, 5), (60, 16, 7)])
def test_oracle_is_the_sequential_loop(n, dim, nc):
    rng = np.random.RandomState(n + dim)
    F = rng.normal(size=(n, dim)).astype(np.float32)
    C = rng.normal(size=(nc, dim)).astype(np.float32)
    C[-1] = C[0]   # an exact tie between two centres: the first wins
    got = vo.compute_vlad_descriptor(F, C)
    assert np.array_equal(got.view(np.uint32), _sequential(F, C).view(np.uint32))


def test_oracle_matches_fp64_brute_force():
    """Against an fp64 restatement: same assignment wherever the two best fp64 distances are further apart than the
    float32 rounding of the sums; residual sums within float32 accumulation error."""
    words = np.load(GOLDEN)["words"]
    rng = np.random.RandomState(3)
    F = np.round(rng.gamma(0.6, 30.0, (2000, 128))).clip(0, 255).astype(np.float32)
    d64 = ((F.astype(np.float64)[:, None, :] - words.astype(np.float64)[None]) ** 2).sum(axis=2)
    best64 = np.argmin(d64, axis=1)
    best32 = vo.nearest_centers(F, words)
    s = np.sort(d64, axis=1)
    clear = (s[:, 1] - s[:, 0]) > 1e-5 * s[:, 0]
    assert clear.mean() > 0.99
    assert np.array_equal(best32[clear], best64[clear])
    v64 = np.zeros(words.shape)
    np.add.at(v64, best32, F.astype(np.float64) - words[best32].astype(np.float64))
    got = vo.compute_vlad_descriptor(F, words).reshape(words.shape)
    scale = np.abs(F.astype(np.float64) - words[best32]).sum()
    assert np.abs(got - v64).max() <= 1e-6 * scale


def test_normalisation_fp64_sum_is_within_the_reference_rounding():
    rng = np.random.RandomState(5)
    v = rng.normal(0, 50, 8192).astype(np.float32)
    a = vo.signed_square_root_normalize(v.copy())
    b = vo.signed_square_root_normalize(v.copy(), fp64_sum=True)
    assert np.allclose(a, b, rtol=4e-7, atol=0)
    assert np.isnan(vo.signed_square_root_normalize(np.zeros(4, np.float32), fp64_sum=True)).all()


def _brute_pairs(hist, refs, cands, exifs, k, enforce):
    out = {}
    for im in refs:
        others = [c for c in sorted(set(cands)) if c != im and c in hist]
        rows = [(vo.vlad_distance(hist[im], hist[c]), j, c) for j, c in enumerate(others)]
        rows.sort(key=lambda r: (math.isnan(r[0]), r[0] if not math.isnan(r[0]) else 0.0, r[1]))
        if enforce:
            same = [r for r in rows if exifs[r[2]]["camera"] == exifs[im]["camera"]][:k]
            diff = [r for r in rows if exifs[r[2]]["camera"] != exifs[im]["camera"]][:k]
            keep = same + diff
        else:
            keep = rows[:k]
        for d, _, c in keep:
            out[vo.sorted_pair(im, c)] = d
    return out


@pytest.mark.parametrize("enforce", [False, True])
@pytest.mark.parametrize("k", [0, 1, 3, 50])
def test_construct_pairs_matches_brute_force(k, enforce):
    rng = np.random.RandomState(k + 7 * enforce)
    names = ["im%02d" % i for i in range(30)]
    hist = {n: rng.normal(size=12).astype(np.float32) for n in names}
    hist["im05"] = hist["im09"].copy()             # exact ties
    hist["im11"] = np.full(12, np.nan, np.float32)  # an empty image
    exifs = {n: {"camera": "cam%d" % (i % 3)} for i, n in enumerate(names)}
    refs, cands = names[::2], names[3:]
    got = vo.match_candidates_with_vlad(hist, refs, cands, exifs, k, enforce)
    want = _brute_pairs(hist, refs, cands, exifs, k, enforce) if k > 0 else {}
    assert set(got) == set(want)
    for p in want:
        assert (math.isnan(got[p]) and math.isnan(want[p])) or got[p] == want[p]
