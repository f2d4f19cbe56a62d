"""tracking.create_tracks_manager on the GPU against oracle/tracks_oracle.py (exact: tracks are connected components
and two integer rules, so there is no tolerance), the TracksManager accessors, and the hand-off into bundle adjustment."""
import ctypes
import dataclasses
import os
import re

import numpy as np
import pytest

from opensfm_b200 import _lib, bundle, synthetic as syn, tracking
from oracle import tracks_oracle as to

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def name(s):
    return "im%02d" % s


@pytest.fixture(scope="module")
def scene():
    return syn.cube_scene(20, 2000)


@pytest.fixture(scope="module")
def scene_rows(scene):
    """Observation rows of every shot: feature k of shot s is observation scene_rows[s][k]."""
    return [np.nonzero(scene.obs_shot == s)[0] for s in range(scene.num_shots)]


def scene_features(scene, rows):
    feats, colors = {}, {}
    for s, r in enumerate(rows):
        feats[name(s)] = np.column_stack([scene.obs_xy[r], scene.obs_sigma[r]])
        colors[name(s)] = (np.arange(3 * len(r)).reshape(-1, 3) % 256).astype(np.int32)
    return feats, colors


def true_matches(scene, rows, band=None, detected=None):
    """{(shot i, shot j): features of the two shots that observe the same point}, i < j <= i + band, over the
    features with detected[shot][feature] set."""
    out = {}
    for i in range(scene.num_shots):
        for j in range(i + 1, scene.num_shots if band is None else min(i + band + 1, scene.num_shots)):
            _, ki, kj = np.intersect1d(scene.obs_point[rows[i]], scene.obs_point[rows[j]], return_indices=True)
            if detected is not None:
                both = detected[i][ki] & detected[j][kj]
                ki, kj = ki[both], kj[both]
            if len(ki):
                out[name(i), name(j)] = np.column_stack([ki, kj]).astype(np.int32)
    return out


def noisy_matches(scene, rows, seed=5):
    """Every shot of this scene sees every point, so the matches are thinned first to make tracks of all lengths:
    half of the features take part, and a shot is matched with the next three.  Then 3 % of the rows are rewired to
    a wrong feature (merged tracks, two features of one image in a track) and 20 % dropped (tracks that only hold
    together through transitivity)."""
    rng = np.random.RandomState(seed)
    detected = [rng.rand(len(r)) < 0.5 for r in rows]
    out = {}
    for (a, b), m in true_matches(scene, rows, band=3, detected=detected).items():
        m = m.copy()
        wrong = rng.rand(len(m)) < 0.03
        m[wrong, 1] = rng.randint(0, len(rows[int(b[2:])]), wrong.sum())
        out[a, b] = m[rng.rand(len(m)) >= 0.2]
    return out


def build(feats, colors, matches, min_length, **kw):
    return tracking.create_tracks_manager(feats, colors, {}, {}, matches, min_length, **kw)


def partition_of(tm):
    a = tm.as_arrays()
    ts = a["track_start"]
    return {frozenset((a["images"][i], int(f)) for i, f in zip(a["obs_image"][ts[t]:ts[t + 1]].tolist(),
                                                                a["obs_feature"][ts[t]:ts[t + 1]].tolist()))
            for t in range(len(ts) - 1)}


def check_layout(tm, canonical_numbering=True):
    """Observations sorted by (track, image), one per image in a track, track_start consistent, tracks numbered by
    their smallest (image, feature)."""
    a = tm.as_arrays()
    trk, img, feat, ts = a["obs_track"], a["obs_image"].astype(np.int64), a["obs_feature"], a["track_start"]
    T = len(ts) - 1
    assert ts[0] == 0 and ts[-1] == len(trk)
    assert np.array_equal(ts, np.searchsorted(trk, np.arange(T + 1)))
    key = trk.astype(np.int64) * len(a["images"]) + img
    assert np.all(np.diff(key) > 0)
    if canonical_numbering and T:
        first = img[ts[:-1]] * (int(feat.max()) + 1) + feat[ts[:-1]]
        assert np.all(np.diff(first) > 0)


def check_against_oracle(tm, with_features, matches, min_length, with_common=True):
    part, common = to.tracks(with_features, matches, min_length, with_common=with_common)
    assert partition_of(tm) == part
    assert tm.num_tracks() == len(part)
    if not with_common:
        return
    assert tm.get_all_pairs_connectivity() == {k: len(v) for k, v in common.items()}
    pa, pb, ps, ca, cb = tm._common_arrays()
    assert len(ca) == sum(len(v) for v in common.values())
    for q in range(len(pa)):
        rows_a, rows_b = ca[ps[q]:ps[q + 1]], cb[ps[q]:ps[q + 1]]
        assert np.all(tm.obs_image[rows_a] == pa[q]) and np.all(tm.obs_image[rows_b] == pb[q])
        assert np.array_equal(tm.obs_track[rows_a], tm.obs_track[rows_b])
        assert np.all(np.diff(tm.obs_track[rows_a]) > 0)
        got = sorted(zip(tm.obs_feature[rows_a].tolist(), tm.obs_feature[rows_b].tolist()))
        assert got == sorted(common[tm.images[pa[q]], tm.images[pb[q]]])


# 1 ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("min_length", [2, 3, 5])
def test_exact_partition_parity(scene, scene_rows, min_length):
    feats, colors = scene_features(scene, scene_rows)
    matches = noisy_matches(scene, scene_rows)
    tm = build(feats, colors, matches, min_length)
    assert tm.num_tracks() > 500
    check_layout(tm)
    check_against_oracle(tm, feats, matches, min_length)
    # the noise did what it is there for: some surviving tracks join two points
    a = tm.as_arrays()
    point = scene.obs_point[np.concatenate(scene_rows)][np.cumsum([0] + [len(r) for r in scene_rows])[a["obs_image"]]
                                                        + a["obs_feature"]]
    assert np.any(point != point[a["track_start"][:-1]][a["obs_track"]])


# 2 ------------------------------------------------------------------------------------------------------------
def test_order_independence(scene, scene_rows):
    feats, colors = scene_features(scene, scene_rows)
    matches = noisy_matches(scene, scene_rows)
    ref = build(feats, colors, matches, 2)
    rng = np.random.RandomState(11)
    keys = list(matches)
    shuffled = {}
    for k in rng.permutation(len(keys)):
        (a, b), m = keys[k], matches[keys[k]]
        m = m[rng.permutation(len(m))]
        if rng.rand() < 0.5:
            shuffled[b, a] = m[:, ::-1]
        else:
            shuffled[a, b] = m
    got = build(feats, colors, shuffled, 2)
    for x, y in zip((ref.obs_track, ref.obs_image, ref.obs_feature, ref.track_start) + ref._common_arrays(),
                    (got.obs_track, got.obs_image, got.obs_feature, got.track_start) + got._common_arrays()):
        assert x.dtype == y.dtype and np.array_equal(x, y)


# 3 ------------------------------------------------------------------------------------------------------------
def hand_features(*names, n=12):
    return ({k: np.zeros((n, 3)) for k in names}, {k: np.zeros((n, 3), dtype=np.int32) for k in names})


@pytest.mark.parametrize("matches, with_features, min_length", [
    ({("a", "b"): [(0, 5)], ("b", "c"): [(5, 7)]}, "abc", 2),
    ({("a", "b"): [(0, 5), (1, 5), (2, 6)]}, "ab", 2),
    ({("a", "b"): [(0, 5), (1, 6)], ("b", "a"): [(5, 0), (7, 2)]}, "ab", 2),
    ({("a", "b"): [(0, 0), (1, 1)], ("b", "c"): [(1, 1)]}, "abc", 2),
    ({("a", "b"): [(0, 0), (1, 1)], ("b", "c"): [(1, 1)]}, "abc", 3),
    ({("a", "b"): [(0, 0), (1, 1)], ("b", "c"): [(1, 1)]}, "abc", 4),
    ({("a", "x"): [(0, 3), (1, 4), (2, 4)], ("x", "b"): [(3, 9)]}, "ab", 3),
    ({("a", "x"): [(0, 3)]}, "ab", 2),
    ({("x", "y"): [(0, 0)]}, "a", 2),
    ({("a", "a"): [(0, 1)], ("a", "b"): [(0, 0), (2, 2)]}, "ab", 2),
    ({}, "ab", 2),
    ({("a", "b"): []}, "ab", 2),
])
def test_hand_built_cases(matches, with_features, min_length):
    feats, colors = hand_features(*with_features)
    tm = build(feats, colors, matches, min_length)
    check_layout(tm, canonical_numbering=False)
    check_against_oracle(tm, feats, matches, min_length)


def test_chain_is_one_track():
    feats, colors = hand_features("a", "b", "c")
    tm = build(feats, colors, {("a", "b"): [(0, 5)], ("b", "c"): [(5, 7)]}, 2)
    assert partition_of(tm) == {frozenset({("a", 0), ("b", 5), ("c", 7)})}
    assert tm.get_all_pairs_connectivity() == {("a", "b"): 1, ("a", "c"): 1, ("b", "c"): 1}


# 4 ------------------------------------------------------------------------------------------------------------
def test_long_path_in_descending_order():
    n = 20000
    names = ["p%05d" % k for k in range(n)]
    feats = {k: np.zeros((1, 3)) for k in names}
    matches = {(names[k + 1], names[k]): np.zeros((1, 2), dtype=np.int32) for k in range(n - 2, -1, -1)}
    tm = build(feats, {}, matches, 2)
    assert tm.num_tracks() == 1 and np.array_equal(tm.track_start, [0, n])
    assert np.array_equal(tm.obs_image, np.arange(n)) and not tm.obs_feature.any()
    check_against_oracle(tm, feats, matches, 2, with_common=False)


def test_path_that_revisits_images_beside_a_clean_track():
    ni, nf = 50, 4000
    names = ["q%02d" % k for k in range(ni)]
    feats = {k: np.zeros((nf + 2, 3)) for k in names}
    f = np.arange(nf, dtype=np.int32)
    # node k of the path is feature k // ni of image k % ni, k = 0 .. ni * nf
    matches = {(names[i], names[i + 1]): np.column_stack([f, f]) for i in range(ni - 1)}
    matches[names[ni - 1], names[0]] = np.column_stack([f, f + 1])
    clean = np.array([[nf + 1, nf + 1]], dtype=np.int32)
    matches[names[0], names[1]] = np.concatenate([matches[names[0], names[1]], clean])
    matches[names[2], names[1]] = clean
    assert sum(len(m) for m in matches.values()) == ni * nf + 2
    tm = build(feats, {}, matches, 2)
    assert partition_of(tm) == {frozenset((names[i], nf + 1) for i in range(3))}
    check_against_oracle(tm, feats, matches, 2)


@pytest.mark.parametrize("min_length", [2, 402])
def test_star(min_length):
    names = ["s%03d" % k for k in range(400)]
    feats = {k: np.zeros((3, 3)) for k in names + ["hub"]}
    matches = {(k, "hub"): [(2, 1)] for k in names}
    tm = build(feats, {}, matches, min_length)
    assert tm.num_tracks() == (1 if min_length == 2 else 0)
    check_layout(tm)
    check_against_oracle(tm, feats, matches, min_length)


# 5 ------------------------------------------------------------------------------------------------------------
def test_index_errors_leave_the_handle_usable():
    feats, colors = hand_features("a", "b", n=4)
    good = {("a", "b"): [(0, 1), (2, 3)]}
    with pytest.raises(RuntimeError, match=r"feature index 4 is outside \[0, 4\) of image 1"):
        build(feats, colors, {("a", "b"): [(0, 1), (2, 4)]}, 2)
    with pytest.raises(RuntimeError, match=r"row 1 of pair 0.*feature index -1 is outside \[0, 4\) of image 0"):
        build(feats, colors, {("a", "b"): [(0, 1), (-1, 2)]}, 2)
    tm = build(feats, colors, good, 2)   # takes the pooled handle the failed calls used
    assert partition_of(tm) == {frozenset({("a", 0), ("b", 1)}), frozenset({("a", 2), ("b", 3)})}


def test_c_abi_rejects_bad_sizes_and_images():
    L = _lib.load()
    h = ctypes.c_void_p()
    _lib.check(L.osfm_tracks_create(0, ctypes.byref(h)))
    try:
        nt, no = ctypes.c_int64(0), ctypes.c_int64(0)

        def call(num_features, pair, rows):
            nf = np.asarray(num_features, dtype=np.int32)
            hf = np.ones(len(nf), dtype=np.uint8)
            pa, pb = np.array([pair[0]], dtype=np.int32), np.array([pair[1]], dtype=np.int32)
            m = np.asarray(rows, dtype=np.int32).reshape(-1, 2)
            ms = np.array([0, len(m)], dtype=np.int64)
            p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
            return L.osfm_tracks_build(h, len(nf), p(nf), p(hf), 1, p(pa), p(pb), p(ms), p(m), 2, ctypes.byref(nt),
                                       ctypes.byref(no))

        # more features than a 32-bit node id can name: refused from the counts alone, nothing is allocated
        with pytest.raises(ValueError, match=r"more than 2\^31 - 1 features"):
            _lib.check(call([2 ** 31 - 1, 1], (0, 1), [(0, 0)]))
        with pytest.raises(RuntimeError, match=r"pair 0 names images \(0, 2\), outside \[0, 2\)"):
            _lib.check(call([3, 3], (0, 2), [(0, 0)]))
        with pytest.raises(RuntimeError, match="needs a successful osfm_tracks_build"):
            _lib.check(L.osfm_tracks_common(h, ctypes.byref(nt), ctypes.byref(no)))
        _lib.check(call([3, 3], (0, 1), [(0, 0), (1, 2)]))
        assert (nt.value, no.value) == (2, 4)
    finally:
        L.osfm_tracks_destroy(h)


# 6 ------------------------------------------------------------------------------------------------------------
def test_tracks_manager_accessors(scene, scene_rows):
    feats, colors = scene_features(scene, scene_rows)
    matches = noisy_matches(scene, scene_rows)
    segm = {name(3): np.arange(len(scene_rows[3])) % 7}
    inst = {name(4): np.arange(len(scene_rows[4])) % 5}
    depths = {name(3): np.where(np.arange(len(scene_rows[3])) % 2, 0.5, np.nan), name(4): np.full(len(scene_rows[4]), 3.0)}
    tm = tracking.create_tracks_manager(feats, colors, segm, inst, matches, 3, depths, False, 2.0)
    part, common = to.tracks(feats, matches, 3)
    # dict of dicts from the oracle, keyed by the engine's track ids through each track's smallest observation
    by_first = {min((int(n[2:]), f) for n, f in tr): tr for tr in part}
    ids = tm.get_track_ids()
    assert ids == [str(k) for k in range(len(part))] and tm.num_tracks() == len(part)
    per_track = {ids[k]: dict(by_first[key]) for k, key in enumerate(sorted(by_first))}
    per_shot = {}
    for t, obs in per_track.items():
        for im, f in obs.items():
            per_shot.setdefault(im, {})[t] = f
    assert sorted(tm.get_shot_ids()) == sorted(per_shot) and tm.num_shots() == len(per_shot)
    for im in (name(0), name(3), name(4), name(19)):
        got = tm.get_shot_observations(im)
        assert {t: o.id for t, o in got.items()} == per_shot[im]
        for t, o in list(got.items())[:50]:
            assert np.array_equal(o.point, feats[im][o.id, :2]) and o.scale == feats[im][o.id, 2]
            assert np.array_equal(o.color, colors[im][o.id])
            assert o.segmentation == (o.id % 7 if im == name(3) else tracking.NO_SEMANTIC_VALUE)
            assert o.instance == (o.id % 5 if im == name(4) else tracking.NO_SEMANTIC_VALUE)
            if im == name(3) and o.id % 2:
                assert (o.depth_prior.value, o.depth_prior.std_deviation, o.depth_prior.is_radial) == (0.5, 2.0, False)
            elif im == name(4):
                assert (o.depth_prior.value, o.depth_prior.std_deviation) == (3.0, 6.0)
            else:
                assert o.depth_prior is None
            assert tm.get_observation(im, t).id == o.id
    for t in ids[:40] + ids[-40:]:
        assert {im: o.id for im, o in tm.get_track_observations(t).items()} == per_track[t]
    with pytest.raises(RuntimeError, match="Accessing invalid shot ID"):
        tm.get_all_common_observations(name(0), "nowhere")
    with pytest.raises(RuntimeError, match="Accessing invalid shot ID"):
        tm.get_shot_observations("nowhere")

    conn = tm.get_all_pairs_connectivity()
    assert conn == {k: len(v) for k, v in common.items()}
    pair = max(conn, key=conn.get)
    tuples = tm.get_all_common_observations(*pair)
    assert sorted((o1.id, o2.id) for _, o1, o2 in tuples) == sorted(common[pair])
    assert all(per_track[t][pair[0]] == o1.id and per_track[t][pair[1]] == o2.id for t, o1, o2 in tuples)
    flipped = tm.get_all_common_observations(pair[1], pair[0])
    assert [(t, o2.id, o1.id) for t, o1, o2 in flipped] == [(t, o1.id, o2.id) for t, o1, o2 in tuples]
    # the restricted form
    shots = [name(s) for s in (0, 3, 4, 7, 19)]
    some = ids[::3]
    want = {}
    for t in some:
        seen = sorted(im for im in per_track[t] if im in shots)
        for x in range(len(seen)):
            for y in range(x + 1, len(seen)):
                want[seen[x], seen[y]] = want.get((seen[x], seen[y]), 0) + 1
    assert tm.get_all_pairs_connectivity(shots, some) == want
    assert tm.get_all_pairs_connectivity(shots) == {k: v for k, v in conn.items() if k[0] in shots and k[1] in shots}

    # common tracks with features: [track ids], p1 (n x 2), p2 (n x 2), and the min_common cut
    cut = int(np.median(list(conn.values())))
    withf = tracking.all_common_tracks_with_features(tm, min_common=cut)
    assert set(withf) == {k for k, v in conn.items() if v >= cut} and 0 < len(withf) < len(conn)
    without = tracking.all_common_tracks_without_features(tm, min_common=cut)
    for k, (tr, p1, p2) in withf.items():
        assert p1.shape == p2.shape == (len(tr), 2) and len(tr) == conn[k] and without[k] == tr
        assert np.array_equal(p1, np.array([feats[k[0]][per_track[t][k[0]], :2] for t in tr]))
        assert np.array_equal(p2, np.array([feats[k[1]][per_track[t][k[1]], :2] for t in tr]))
    tr, p1, p2 = tracking.common_tracks(tm, *pair)
    assert (tr, p1.tolist(), p2.tolist()) == (withf[pair][0], withf[pair][1].tolist(), withf[pair][2].tolist())


# 7 ------------------------------------------------------------------------------------------------------------
def test_tracks_feed_bundle_adjustment(scene, scene_rows):
    feats, colors = scene_features(scene, scene_rows)
    tm = build(feats, colors, true_matches(scene, scene_rows), 2)
    a = tm.as_arrays()
    assert a["images"] == [name(s) for s in range(scene.num_shots)]
    # observation of the scene behind every track observation
    row = np.concatenate(scene_rows)[np.concatenate([[0], np.cumsum([len(r) for r in scene_rows])])[a["obs_image"]]
                                     + a["obs_feature"]]
    point = scene.obs_point[row]
    first = point[a["track_start"][:-1]]
    assert np.array_equal(point, first[a["obs_track"]])          # a track is one point ...
    assert len(np.unique(first)) == len(first)                   # ... and a point one track
    seen = np.bincount(scene.obs_point, minlength=len(scene.points))
    want = np.nonzero(seen[scene.obs_point] >= 2)[0]
    assert np.array_equal(np.sort(row), want)                    # every observation of a point seen twice, once
    assert np.array_equal(a["xy"], scene.obs_xy[row]) and np.array_equal(a["scale"], scene.obs_sigma[row])

    pb = syn.scene_to_problem(scene)
    own = bundle.solve(pb)
    pt = pb.obs_point[row][a["track_start"][:-1]]
    pb2 = dataclasses.replace(pb, points=pb.points[pt], point_const=pb.point_const[pt],
                              obs_shot=a["obs_image"], obs_point=a["obs_track"], obs_xy=a["xy"], obs_sigma=a["scale"])
    got = bundle.solve(pb2)

    def rms(e):
        return float(np.sqrt((e[:, :2] ** 2).sum(axis=1).mean()))

    # a point seen once fits its observation exactly; compare over the observations both problems have
    r_own, r_got = rms(own["reprojection_errors"][want]), rms(got["reprojection_errors"])
    assert abs(r_got - r_own) <= 0.01 * r_own, (r_got, r_own)
    assert r_got < 0.01


# 8 ------------------------------------------------------------------------------------------------------------
def test_c_abi_symbols():
    want = {"osfm_tracks_create", "osfm_tracks_destroy", "osfm_tracks_build", "osfm_tracks_get", "osfm_tracks_common",
            "osfm_tracks_get_common", "osfm_tracks_last_device_ms"}
    header = open(os.path.join(ROOT, "include", "opensfm_b200.h")).read()
    assert want <= set(re.findall(r"\b(osfm_tracks_[a-z_]+)\s*\(", header))
    L = _lib.load()
    for s in want:
        assert hasattr(L, s) and s in _lib.SIGNATURES
