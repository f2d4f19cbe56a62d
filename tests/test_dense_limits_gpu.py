"""The dense engine at the limits of what it accepts, each case both bit for bit against the raster-order oracle
(oracle/dense_oracle.cpp) and through the fp64 postcondition checker (oracle/dense_fp64.py): patch sizes 1 to 15,
32-view lists, no PatchMatch iterations, one depth plane, min_patch_sd 0 and 40, a fully masked reference, tall
images and one-column / one-row interiors, the product's 640x480 with 100 planes, mixed submissions, a reused engine,
and cleaning and pruning of product-size maps.  The set-aside counts and the largest f32-versus-fp64 errors of every
case are printed (pytest -s)."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from opensfm_b200 import dense as D
from opensfm_b200 import synthetic as syn
from oracle import dense_fp64 as f
from oracle import dense_oracle as do

pytestmark = pytest.mark.gpu

MIN_SCORE = 0.1
METHODS = ["BRUTE_FORCE", "PATCH_MATCH", "PATCH_MATCH_SAMPLE"]


def _views(sc, masks=None):
    out = []
    for k in range(len(sc.K)):
        g = sc.gray[k]
        h, w = g.shape
        m = np.ones((h, w), np.uint8) if masks is None else masks[k]
        out.append(D.View(K=sc.K[k], R=sc.R[k], t=sc.t[k], width=w, height=h, gray=g, mask=m, color=sc.rgb[k],
                          labels=(np.arange(h * w) % 7).astype(np.uint8).reshape(h, w)))
    return out


def _oracle(views, ref, seed):
    vs = [views[v] for v in ref.views]
    return do.estimate([v.K for v in vs], [v.R for v in vs], [v.t for v in vs], [v.gray for v in vs], vs[0].mask,
                       ref.method, ref.patch_size, ref.num_depth_planes, ref.patchmatch_iterations,
                       np.float32(ref.min_patch_sd) * np.float32(ref.min_patch_sd), ref.min_depth, ref.max_depth,
                       seed=seed, key=ref.key)


def _problem(views, ref):
    vs = [views[v] for v in ref.views]
    return f.Problem([v.K for v in vs], [v.R for v in vs], [v.t for v in vs], [v.gray for v in vs], vs[0].mask,
                     ref.patch_size, ref.min_patch_sd, ref.min_depth, ref.max_depth, ref.num_depth_planes)


def _same(got, want, what):
    for g, w, name in zip(got, want, ("depth", "plane", "score", "nghbr")):
        assert np.array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                              w.view(np.uint32) if w.dtype == np.float32 else w), (what, name, int((g != w).sum()))


def _maps(est, k):
    return est.depth[k], est.plane[k], est.score[k], est.nghbr[k]


def _check(views, refs, est, seed, what, want=None):
    """Every reference bit for bit against the oracle (computed here unless given) and through the fp64 checker."""
    for k, ref in enumerate(refs):
        w = want[k] if want is not None and want[k] is not None else _oracle(views, ref, seed)
        _same(_maps(est, k), w, (what, k))
        rep = f.check_estimate(_problem(views, ref), ref.method, *_maps(est, k))
        f.assert_bounded(rep, (what, k))
        print("%s ref %d %s patch %d: assigned %d, sampled %d, checked %d, set aside %s, max |score err| %.3g "
              "(%.2f of tol), max depth rel err %.3g"
              % (what, k, ref.method, ref.patch_size, rep.assigned, rep.sampled, rep.checked, rep.set_aside,
                 rep.max_score_err, rep.max_score_err_rel_tol, rep.max_depth_rel_err))


@pytest.fixture(scope="module")
def small():
    sc = syn.textured_scene(4, 64, 48, seed=3)
    masks = [np.ones((48, 64), np.uint8) for _ in range(4)]
    masks[0][:8, :14] = 0
    return _views(sc, masks)


@pytest.mark.parametrize("method", METHODS)
def test_patch_sizes(small, method):
    refs = [D.Reference([k] + [v for v in range(4) if v != k], 3.0, 30.0, method, p, 20, 2, key=k)
            for k, p in enumerate([3, 11, 13, 15])]
    with D.Engine(small) as E:
        est = E.estimate(refs, seed=11)
    _check(small, refs, est, 11, "patch sizes")


def test_patch_one(small):
    """PatchMatch refuses patch size 1 before any launch, in the engine and the mirror; brute force returns zeros."""
    with D.Engine(small) as E:
        for method in ("PATCH_MATCH", "PATCH_MATCH_SAMPLE"):
            with pytest.raises(ValueError, match="patch size 1"):
                E.estimate([D.Reference([0, 1, 2], 3.0, 30.0, method, 1, 20, 2, min_patch_sd=0.0)])
        ref = D.Reference([0, 1, 2], 3.0, 30.0, "BRUTE_FORCE", 1, 20, 2, min_patch_sd=0.0)
        est = E.estimate([ref], seed=1)
    assert all((m == 0).all() for m in _maps(est, 0))
    _same(_maps(est, 0), _oracle(small, ref, 1), "patch 1")
    de = D.DepthmapEstimator()
    de.set_depth_range(3.0, 30.0, 20)
    de.set_patch_size(1)
    de.set_min_patch_sd(0)
    for v in small[:3]:
        de.add_view(v.K, v.R, v.t, v.gray, v.mask)
    for call in (de.compute_patch_match, de.compute_patch_match_sample):
        with pytest.raises(ValueError, match="patch size 1"):
            call()


@pytest.mark.parametrize("method", METHODS)
def test_32_views(method):
    sc = syn.textured_scene(6, 40, 30, seed=5, arc_degrees=50)
    views = _views(sc)
    lst = [0] + [1 + k % 5 for k in range(31)]
    refs = [D.Reference(lst, 3.0, 30.0, method, 5, 6, 1, key=3)]
    with D.Engine(views) as E:
        est = E.estimate(refs, seed=2)
        with pytest.raises(ValueError, match="33 views"):
            E.estimate([D.Reference(lst + [1], 3.0, 30.0, method, 5, 6, 1)])
    _check(views, refs, est, 2, "32 views")


@pytest.mark.parametrize("method", METHODS)
def test_limits(method):
    """No PatchMatch iterations, one depth plane, min_patch_sd 0 and 40, and a fully masked reference."""
    sc = syn.textured_scene(6, 40, 30, seed=5, arc_degrees=50)
    masks = [np.ones((30, 40), np.uint8) for _ in range(6)]
    masks[4][:] = 0
    views = _views(sc, masks)
    others = lambda k: [k] + [v for v in range(6) if v != k][:4]
    refs = [D.Reference(others(0), 3.0, 30.0, method, 5, 20, 0, key=0),
            D.Reference(others(1), 3.0, 30.0, method, 5, 1, 2, key=1),
            D.Reference(others(2), 3.0, 30.0, method, 5, 20, 2, 0.0, key=2),
            D.Reference(others(3), 3.0, 30.0, method, 5, 20, 2, 40.0, key=3),
            D.Reference(others(4), 3.0, 30.0, method, 5, 20, 2, key=4)]
    with D.Engine(views) as E:
        est = E.estimate(refs, seed=7)
    _check(views, refs, est, 7, "limits")
    if method != "BRUTE_FORCE":
        assert all((m == 0).all() for m in _maps(est, 4))


@pytest.mark.parametrize("method", METHODS)
def test_shapes(method):
    """A tall reference, one exactly patch-wide (its interior one column) and one exactly patch-high (one row)."""
    sc = syn.textured_scene(5, sizes=[(40, 120), (7, 40), (40, 7), (48, 40), (48, 40)], seed=6, arc_degrees=30)
    views = _views(sc)
    refs = [D.Reference([0, 3, 4], 3.0, 30.0, method, 5, 20, 2, key=0),
            D.Reference([1, 3, 4], 3.0, 30.0, method, 7, 20, 2, 2.0, key=1),
            D.Reference([2, 3, 4], 3.0, 30.0, method, 7, 20, 2, 2.0, key=2)]
    with D.Engine(views) as E:
        est = E.estimate(refs, seed=3)
    _check(views, refs, est, 3, "shapes")


# ---- the product's size: 640x480, 100 planes, 3 iterations -------------------------------------------------------------

SEED = 21


@pytest.fixture(scope="module")
def product():
    """Seven 640x480 views and one reference per method (brute force over a 3-view list, PatchMatch over 6), with
    their oracle outputs computed once, concurrently."""
    sc = syn.textured_scene(7, 640, 480, seed=11, arc_degrees=40)
    masks = [np.ones((480, 640), np.uint8) for _ in range(7)]
    masks[1][:60, :200] = 0
    views = _views(sc, masks)
    refs = [D.Reference([0, 1, 2], 3.0, 30.0, "BRUTE_FORCE", 7, 100, 3, key=10),
            D.Reference([1, 0, 2, 3, 4, 5], 3.0, 30.0, "PATCH_MATCH", 7, 100, 3, key=11),
            D.Reference([2, 0, 1, 3, 4, 5], 3.0, 30.0, "PATCH_MATCH_SAMPLE", 7, 100, 3, key=12)]
    with ThreadPoolExecutor(len(refs)) as ex:
        want = list(ex.map(lambda r: _oracle(views, r, SEED), refs))
    return views, refs, want


def test_product_size(product):
    views, refs, want = product
    with D.Engine(views) as E:
        est = E.estimate(refs, seed=SEED, min_score=MIN_SCORE)
        raw = E.clean([[0], [1], [2]], 0.01, 1)              # one consistent view keeps the whole raw map
    _check(views, refs, est, SEED, "640x480", want)
    for k, r in enumerate(refs):
        f.check_gate(est.depth[k], est.score[k], raw[k], MIN_SCORE, r.max_depth)


def test_mixed_submission_and_reused_engine(product):
    """A 640x480 reference with 24x24 ones of other methods and patches in one submission; then one engine reused
    across submissions of different shapes, against fresh engines."""
    views, refs, want = product
    tiny = syn.textured_scene(3, 24, 24, seed=2, arc_degrees=30)
    allv = views + _views(tiny)
    small = [D.Reference([7, 8, 9], 3.0, 30.0, "BRUTE_FORCE", 3, 20, 2, key=0),
             D.Reference([8, 7, 9], 3.0, 30.0, "PATCH_MATCH", 5, 20, 2, key=1),
             D.Reference([9, 7, 8], 3.0, 30.0, "PATCH_MATCH_SAMPLE", 7, 20, 2, key=2)]
    mixed = [small[0], refs[2], small[1], small[2]]
    subs = [mixed, small, [refs[1]], [D.Reference([8, 9, 7], 3.0, 30.0, "BRUTE_FORCE", 9, 10, 1, key=5)]]
    with D.Engine(allv) as E:
        got = [E.estimate(s, seed=SEED) for s in subs]
    _check(allv, mixed, got[0], SEED, "mixed", [None, want[2], None, None])
    for s, g in zip(subs[1:], got[1:]):
        with D.Engine(allv) as E:
            fresh = E.estimate(s, seed=SEED)
        for k in range(len(s)):
            _same(_maps(g, k), _maps(fresh, k), "reused engine")
    _same(_maps(got[2], 0), want[1], "reused engine, 640x480")


def test_clean_and_prune_product(product):
    """Cleaning and pruning of the product-size maps with min_consistent_views 1 to 4: bit for bit against the oracle
    and through the fp64 cleaner and pruner, whose set-asides are bounded."""
    views, refs, want = product
    lists = [[0, 1, 2], [1, 0, 2], [2, 0, 1]]
    raw = {k: np.where((want[k][2] > np.float32(MIN_SCORE)) & (want[k][0].astype(np.float64) < 30.0), want[k][0],
                       0).astype(np.float32) for k in range(3)}
    geo = lambda lst: ([views[v].K for v in lst], [views[v].R for v in lst], [views[v].t for v in lst])
    with D.Engine(views) as E:
        E.estimate(refs, seed=SEED, min_score=MIN_SCORE)
        for mc in (1, 2, 3, 4):
            clean = E.clean(lists, 0.01, mc)
            pruned = E.prune(lists, 0.01)
            for k, lst in enumerate(lists):
                assert np.array_equal(clean[k], do.clean(*geo(lst), [raw[v] for v in lst], 0.01, mc)), (mc, k)
                aside = f.check_clean(*geo(lst), [raw[v] for v in lst], clean[k], 0.01, mc)
                assert aside <= 0.01 * max(int((raw[k] > 0).sum()), 1) + 2, (mc, k, aside)
                print("clean mc %d ref %d: %d kept, %d set aside" % (mc, k, int((clean[k] > 0).sum()), aside))
            for k, lst in enumerate(lists):
                planes = [want[v][1] for v in lst]
                w = do.prune(*geo(lst), [clean[v] for v in lst], planes, views[lst[0]].color, views[lst[0]].labels,
                             0.01)
                for g, x in zip(pruned[k], w):
                    assert np.array_equal(g, x), (mc, k)
                aside = f.check_prune(*geo(lst), [clean[v] for v in lst], planes, pruned[k], 0.01)
                assert aside <= 0.01 * max(int((clean[k] > 0).sum()), 1) + 2, (mc, k, aside)
                print("prune mc %d ref %d: %d points, %d set aside" % (mc, k, len(pruned[k][0]), aside))
            if mc <= 2:
                assert all(len(p[0]) > 1000 for p in pruned), mc
