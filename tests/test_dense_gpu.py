"""The dense engine on the GPU against the raster-order oracle (oracle/dense_oracle.cpp), bit for bit: estimation by
every method on several scenes, sizes, patch sizes and list lengths in one submission; cleaning and pruning; the
generator's independence of the batch; and argument errors."""
import numpy as np
import pytest

from opensfm_b200 import dense as D
from opensfm_b200 import synthetic as syn
from oracle import dense_oracle as do

pytestmark = pytest.mark.gpu

MIN_SCORE = 0.1


def _views(sc, masks=None):
    out = []
    for k in range(len(sc.K)):
        g = sc.gray[k]
        h, w = g.shape
        m = np.ones((h, w), np.uint8) if masks is None else masks[k]
        out.append(D.View(K=sc.K[k], R=sc.R[k], t=sc.t[k], width=w, height=h, gray=g, mask=m, color=sc.rgb[k],
                          labels=(np.arange(h * w) % 7).astype(np.uint8).reshape(h, w)))
    return out


def _oracle_estimate(views, ref, seed):
    vs = [views[v] for v in ref.views]
    return do.estimate([v.K for v in vs], [v.R for v in vs], [v.t for v in vs], [v.gray for v in vs], vs[0].mask,
                       ref.method, ref.patch_size, ref.num_depth_planes, ref.patchmatch_iterations,
                       np.float32(ref.min_patch_sd) * np.float32(ref.min_patch_sd), ref.min_depth, ref.max_depth,
                       seed=seed, key=ref.key)


def _gate(depth, score, max_depth):
    return np.where((score > np.float32(MIN_SCORE)) & (depth.astype(np.float64) < max_depth), depth, 0).astype(
        np.float32)


@pytest.fixture(scope="module")
def scenes():
    a = syn.textured_scene(4, 96, 72, seed=3)
    mixed = syn.textured_scene(3, sizes=[(96, 72), (80, 64), (112, 84)], seed=5, arc_degrees=30)
    wide = syn.textured_scene(8, 64, 48, seed=7, arc_degrees=60)
    masks = [np.ones(g.shape, np.uint8) for g in a.gray]
    masks[0][:12, :20] = 0
    return {"a": (a, _views(a, masks)), "mixed": (mixed, _views(mixed)), "wide": (wide, _views(wide))}


def _refs(method):
    """(scene, Reference) of one submission per scene: patch sizes 5 / 7 / 9, 2-view and 7-view lists."""
    return {
        "a": [D.Reference([0, 1, 2, 3], 3.0, 30.0, method, 7, 40, 2, key=0),
              D.Reference([1, 0], 3.0, 30.0, method, 5, 40, 2, key=1),
              D.Reference([2, 1, 3], 3.0, 30.0, method, 9, 40, 1, key=2)],
        "mixed": [D.Reference([0, 1, 2], 3.0, 30.0, method, 7, 30, 2, key=0),
                  D.Reference([2, 0, 1], 3.0, 30.0, method, 5, 30, 2, key=1)],
        "wide": [D.Reference([3, 0, 1, 2, 4, 5, 6], 3.0, 40.0, method, 5, 30, 2, key=3)],
    }


@pytest.mark.parametrize("method", ["BRUTE_FORCE", "PATCH_MATCH", "PATCH_MATCH_SAMPLE"])
def test_estimate_equals_oracle(scenes, method):
    for name, refs in _refs(method).items():
        sc, views = scenes[name]
        with D.Engine(views) as E:
            got = E.estimate(refs, seed=11, min_score=MIN_SCORE)
        for k, ref in enumerate(refs):
            want = _oracle_estimate(views, ref, 11)
            for g, w, what in zip((got.depth[k], got.plane[k], got.score[k], got.nghbr[k]), want,
                                  ("depth", "plane", "score", "nghbr")):
                assert np.array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                      w.view(np.uint32) if w.dtype == np.float32 else w), (
                    name, k, what, int((g != w).sum()))
            assert (want[0] > 0).mean() > 0.2, (name, k)


def test_determinism_alone_and_in_batch(scenes):
    sc, views = scenes["a"]
    refs = _refs("PATCH_MATCH_SAMPLE")["a"]
    with D.Engine(views) as E:
        batch = E.estimate(refs, seed=5)
        again = E.estimate(refs, seed=5)
        alone = E.estimate([refs[2]], seed=5)
        other = E.estimate([refs[2]], seed=6)
    for k in range(3):
        assert np.array_equal(batch.depth[k], again.depth[k]) and np.array_equal(batch.plane[k], again.plane[k])
    assert np.array_equal(batch.depth[2], alone.depth[0]) and np.array_equal(batch.nghbr[2], alone.nghbr[0])
    assert not np.array_equal(alone.depth[0], other.depth[0])


def test_pydense_mirror_equals_oracle(scenes):
    sc, views = scenes["mixed"]
    de = D.DepthmapEstimator(seed=4)
    de.set_depth_range(3.0, 30.0, 20)
    de.set_patchmatch_iterations(1)
    de.set_patch_size(5)
    de.set_min_patch_sd(2.0)
    for v in views:
        de.add_view(v.K, v.R, v.t, v.gray, v.mask)
    got = de.compute_patch_match()
    want = _oracle_estimate(views, D.Reference([0, 1, 2], 3.0, 30.0, "PATCH_MATCH", 5, 20, 1, 2.0), 4)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


@pytest.mark.parametrize("min_consistent", [1, 2, 3, 4])
def test_clean_and_prune_equal_oracle(scenes, min_consistent):
    sc, views = scenes["a"]
    refs = [D.Reference([k] + [v for v in range(4) if v != k], 3.0, 30.0, "PATCH_MATCH_SAMPLE", 7, 30, 2, key=k)
            for k in range(3)]                                 # view 3 gets no raw map: skipped by every cleaner
    est, clean, pruned, _ = D.depthmaps(views, refs, MIN_SCORE, 0.01, min_consistent, seed=2)
    raw = {k: _gate(est.depth[k], est.score[k], 30.0) for k in range(3)}
    lists = [[v for v in r.views if v in raw] for r in refs]
    want_clean = {}
    for k, lst in enumerate(lists):
        vs = [views[v] for v in lst]
        want_clean[k] = do.clean([v.K for v in vs], [v.R for v in vs], [v.t for v in vs], [raw[v] for v in lst], 0.01,
                                 min_consistent)
        assert np.array_equal(clean[k], want_clean[k]), (k, int((clean[k] != want_clean[k]).sum()))
    total = 0
    for k, lst in enumerate(lists):
        vs = [views[v] for v in lst]
        want = do.prune([v.K for v in vs], [v.R for v in vs], [v.t for v in vs], [want_clean[v] for v in lst],
                        [est.plane[v] for v in lst], vs[0].color, vs[0].labels, 0.01)
        for g, w in zip(pruned[k], want):
            assert np.array_equal(g, w), k
        total += len(want[0])
    assert total > 0 or min_consistent > len(lists[0])   # 3 raw maps: 4 consistent views keep nothing


def test_prune_edges_equal_oracle():
    """Points behind a neighbour and reprojections just outside its image, on hand-made clean maps."""
    rng = np.random.RandomState(1)
    sc = syn.textured_scene(3, 64, 48, seed=9, arc_degrees=50)
    views = _views(sc)
    depths = [sc.depth[k] * rng.uniform(0.97, 1.03, sc.depth[k].shape).astype(np.float32) for k in range(3)]
    depths[1][:, :8] = 0
    planes = [rng.normal(size=(48, 64, 3)).astype(np.float32) for _ in range(3)]
    for k in range(3):
        views[k].clean_depth, views[k].plane = depths[k], planes[k]
    # the second view turned around: every point is behind it
    views[2].R = -views[2].R
    views[2].t = -views[2].t
    with D.Engine(views) as E:
        got = E.prune([[0, 1, 2], [1, 0], [0, 2]], 0.02)
    for lst, g in zip([[0, 1, 2], [1, 0], [0, 2]], got):
        vs = [views[v] for v in lst]
        w = do.prune([v.K for v in vs], [v.R for v in vs], [v.t for v in vs], [depths[v] for v in lst],
                     [planes[v] for v in lst], vs[0].color, vs[0].labels, 0.02)
        for a, b in zip(g, w):
            assert np.array_equal(a, b), lst


def test_errors(scenes):
    sc, views = scenes["a"]
    with D.Engine(views) as E:
        for ref, msg in [(D.Reference([0, 1], 3, 30, "BRUTE_FORCE", 6), "patch size 6"),
                         (D.Reference([0, 1], 3, 30, "BRUTE_FORCE", 17), "patch size 17"),
                         (D.Reference([0, 9], 3, 30, "BRUTE_FORCE", 7), "view index 9"),
                         (D.Reference([0], 3, 30, "BRUTE_FORCE", 7), "views"),
                         (D.Reference([0, 1], -1, 30, "BRUTE_FORCE", 7), "depth range")]:
            with pytest.raises(ValueError, match=msg):
                E.estimate([ref])
        with pytest.raises(ValueError, match="expected"):
            E.set_maps(0, np.zeros((5, 5), np.float32))
        with pytest.raises(ValueError, match="no raw depthmap"):
            E.clean([[3, 0]])
