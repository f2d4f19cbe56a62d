"""The fp64 restatement of depthmap.cc (oracle/dense_fp64.py) on the CPU: its pieces against the C++ oracle's, its
postcondition checker on the oracle's outputs for the cases the GPU limits file runs (at reduced size), the f32 error
its tolerances allow for, and mutation tests: the checker must reject each deliberately broken output."""
import numpy as np
import pytest

from opensfm_b200 import synthetic as syn
from oracle import dense_fp64 as f
from oracle import dense_oracle as do

METHODS = ["BRUTE_FORCE", "PATCH_MATCH", "PATCH_MATCH_SAMPLE"]
def _rot(ax, ang):
    return syn.angle_axis_to_rotation(np.asarray(ax, float) * ang)


def _run(sc, views, mask, method, patch, planes=30, iters=2, sd=5.0, dmin=3.0, dmax=30.0, seed=11, key=0, imgs=None):
    imgs = imgs if imgs is not None else [sc.gray[v] for v in views]
    Ks, Rs, ts = [sc.K[v] for v in views], [sc.R[v] for v in views], [sc.t[v] for v in views]
    sd2 = np.float32(sd) * np.float32(sd)
    out = do.estimate(Ks, Rs, ts, imgs, mask, method, patch, planes, iters, sd2, dmin, dmax, seed=seed, key=key)
    prob = f.Problem(Ks, Rs, ts, imgs, mask, patch, sd, dmin, dmax, planes)
    return prob, out


# ---- the pieces against the C++ oracle ----------------------------------------------------------------------------


def test_pieces_agree_with_oracle():
    rng = np.random.RandomState(0)
    for _ in range(50):
        K = np.array([[rng.uniform(300, 900), 0, rng.uniform(100, 400)], [0, rng.uniform(300, 900),
                      rng.uniform(100, 300)], [0, 0, 1]])
        K2 = K * np.array([[rng.uniform(0.8, 1.2)], [rng.uniform(0.8, 1.2)], [1.0]])
        R1, R2 = _rot(rng.normal(size=3), rng.uniform(0, 0.3)), _rot(rng.normal(size=3), rng.uniform(0, 0.3))
        t1, t2 = rng.normal(size=3), rng.normal(size=3)
        Kall, Kinv0, Q, a = f.view_terms([K, K2], [R1, R2], [t1, t2])
        pl = np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), -rng.uniform(0.03, 0.3)], np.float32)
        prob = f.Problem([K, K2], [R1, R2], [t1, t2], [np.zeros((9, 9), np.uint8)] * 2, np.ones((9, 9), np.uint8), 3)
        H = prob.homography(pl.astype(np.float64), 1)[0]
        Ho = do.homography(Kinv0, Q[1], a[1], K2, pl)
        assert np.allclose(Ho, H, rtol=2e-7, atol=1e-6 * np.abs(H).max())
        x, y = rng.uniform(0, 600), rng.uniform(0, 400)
        assert abs(do.depth_of_plane(x, y, Kinv0, pl) - f.depth_of_plane(x, y, Kinv0, pl)) <= \
            3e-7 * f.depth_of_plane(x, y, Kinv0, pl)
        dep = rng.uniform(1, 50)
        assert np.allclose(do.backproject(x, y, dep, Kinv0, R1, t1), f.backproject(x, y, dep, K, R1, t1),
                           rtol=1e-12, atol=1e-12)
        nrm = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), -1], np.float32)
        assert np.allclose(do.plane_from_depth_normal(x, y, Kinv0, dep, nrm),
                           f.plane_from_depth_and_normal(x, y, Kinv0, dep, nrm), rtol=1e-5)
        xs = rng.randint(0, 256, 49).astype(np.float64)
        ys = np.clip(128 + (xs - 128) * rng.uniform(-1, 1) + rng.normal(0, 20, 49), 0, 255)
        ws = f.bilateral_weight(xs - xs[24], np.tile(np.arange(-3, 4), 7), np.repeat(np.arange(-3, 4), 7))
        sw = ws.sum()
        mx, my = (ws * xs).sum() / sw, (ws * ys).sum() / sw
        ncc = ((ws * xs * ys).sum() / sw - mx * my) / np.sqrt(((ws * xs * xs).sum() / sw - mx * mx) *
                                                              ((ws * ys * ys).sum() / sw - my * my))
        assert abs(do.ncc(xs, ys, ws) - ncc) < 1e-4


def test_score_of_a_known_warp():
    """A view that is the reference shifted by half a pixel sees, through any plane, the reference sampled at
    x + 0.5: the fp64 score is the NCC of the patch with its bilinear shift, and -1 where a sample leaves the image."""
    rng = np.random.RandomState(2)
    im = rng.randint(0, 256, (20, 30)).astype(np.uint8)
    K = np.array([[50.0, 0, 15], [0, 50, 10], [0, 0, 1]])
    K1 = K.copy()
    K1[0, 2] += 0.5
    prob = f.Problem([K, K1], [np.eye(3)] * 2, [np.zeros(3)] * 2, [im, im], np.ones_like(im), 5)
    s = prob.plane_image_score([10], [12], [[0.1, 0.0, -0.2]], 1)
    f64 = im.astype(float)
    patch = f64[8:13, 10:15]
    shifted = 0.5 * (f64[8:13, 10:15] + f64[8:13, 11:16])
    w = f.bilateral_weight(patch - f64[10, 12], np.arange(-2, 3)[None], np.arange(-2, 3)[:, None])
    mx, my = (w * patch).sum() / w.sum(), (w * shifted).sum() / w.sum()
    cov = (w * patch * shifted).sum() / w.sum() - mx * my
    vx, vy = (w * patch ** 2).sum() / w.sum() - mx * mx, (w * shifted ** 2).sum() / w.sum() - my * my
    assert abs(s.score[0] - cov / np.sqrt(vx * vy)) < 1e-12
    assert abs(s.coord_margin[0] - 7.0) < 1e-9                # the patch's last row, 12, against rows - 1 = 19
    # the last interior column samples at x = 29.5 >= cols - 1: zero, and the variance gate does not reject it
    edge = prob.plane_image_score([10], [27], [[0.1, 0.0, -0.2]], 1)
    assert edge.score[0] > -1 and abs(edge.coord_margin[0] - 0.5) < 1e-9


def test_f32_warp_coordinates_within_tolerance():
    """The first-order warp's sample coordinates evaluated in f32 as the reference does (homography rounded to f32)
    stay within a quarter of the set-aside distance of their fp64 values, at 640x480 and patch 15."""
    sc = syn.textured_scene(4, 640, 480, seed=3)
    prob = f.Problem(sc.K, sc.R, sc.t, list(sc.gray), np.ones((480, 640), np.uint8), 15, 5.0, 3.0, 30.0, 30)
    rng = np.random.RandomState(0)
    N = 2000
    i, j = rng.randint(7, 473, N), rng.randint(7, 633, N)
    dep = np.exp(rng.uniform(np.log(3), np.log(30), N))
    nrm = np.stack([rng.uniform(-1, 1, N), rng.uniform(-1, 1, N), -np.ones(N)], 1)
    pl = f.plane_from_depth_and_normal(j, i, prob.Kinv0, dep, nrm).astype(np.float32).astype(np.float64)

    def coords(H, fj, fi, dt):
        u = H[:, 0, 0] * fj + H[:, 0, 1] * fi + H[:, 0, 2]
        v = H[:, 1, 0] * fj + H[:, 1, 1] * fi + H[:, 1, 2]
        w = H[:, 2, 0] * fj + H[:, 2, 1] * fi + H[:, 2, 2]
        ww = w * w
        a, b = (H[:, 0, 0] * w - H[:, 2, 0] * u) / ww, (H[:, 1, 0] * w - H[:, 2, 0] * v) / ww
        c, d = (H[:, 0, 1] * w - H[:, 2, 1] * u) / ww, (H[:, 1, 1] * w - H[:, 2, 1] * v) / ww
        dx, dy = prob.off_dx.astype(dt)[None], prob.off_dy.astype(dt)[None]
        return ((u / w)[:, None] + a[:, None] * dx + c[:, None] * dy,
                (v / w)[:, None] + b[:, None] * dx + d[:, None] * dy)

    worst = 0.0
    for e in range(1, 4):
        H = prob.homography(pl, e)
        x32, y32 = coords(H.astype(np.float32), j.astype(np.float32), i.astype(np.float32), np.float32)
        x64, y64 = coords(H, j.astype(np.float64), i.astype(np.float64), np.float64)
        near = (np.abs(x64) < 1280) & (np.abs(y64) < 960)
        worst = max(worst, float(np.maximum(np.abs(x32 - x64), np.abs(y32 - y64))[near].max()))
    assert worst <= prob.coord_tol / 4, (worst, prob.coord_tol)


# ---- the checker on the oracle's outputs ----------------------------------------------------------------------------


@pytest.fixture(scope="module")
def small():
    sc = syn.textured_scene(4, 64, 48, seed=3)
    mask = np.ones((48, 64), np.uint8)
    mask[:8, :14] = 0
    return sc, mask


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("patch", [3, 11, 13, 15])
def test_checker_passes_oracle_patch_sizes(small, method, patch):
    sc, mask = small
    prob, out = _run(sc, [0, 1, 2, 3], mask, method, patch, planes=20)
    f.assert_bounded(f.check_estimate(prob, method, *out), (method, patch))


@pytest.mark.parametrize("method", METHODS)
def test_checker_passes_oracle_limits(method):
    sc = syn.textured_scene(6, 40, 30, seed=5, arc_degrees=50)
    ones = np.ones((30, 40), np.uint8)
    for what, kw in [("iterations 0", dict(iters=0)), ("one depth plane", dict(planes=1)),
                     ("min_patch_sd 0", dict(sd=0.0)), ("min_patch_sd 40", dict(sd=40.0))]:
        prob, out = _run(sc, [0, 1, 2, 3, 4, 5], ones, method, 5, **kw)
        f.assert_bounded(f.check_estimate(prob, method, *out), (method, what))
    prob, out = _run(sc, [0, 1, 2], np.zeros_like(ones), method, 5)        # a fully masked reference
    f.check_estimate(prob, method, *out)
    if method != "BRUTE_FORCE":
        assert all((m == 0).all() for m in out)
    # a 32-view list: the reference and 31 views (repeats of the 5 others)
    views = [0] + [1 + k % 5 for k in range(31)]
    prob, out = _run(sc, views, ones, method, 5, planes=6, iters=1)
    f.assert_bounded(f.check_estimate(prob, method, *out), (method, "32 views"))


@pytest.mark.parametrize("method", METHODS)
def test_checker_passes_oracle_shapes(method):
    tall = syn.textured_scene(3, sizes=[(24, 60), (30, 64), (24, 60)], seed=4, arc_degrees=30)
    prob, out = _run(tall, [0, 1, 2], np.ones((60, 24), np.uint8), method, 5)
    f.assert_bounded(f.check_estimate(prob, method, *out), (method, "tall"))
    # a reference exactly patch-wide, then patch-high: its interior is one column, then one row
    for size in [(7, 40), (40, 7)]:
        sc = syn.textured_scene(3, sizes=[size, (48, 40), (48, 40)], seed=6, arc_degrees=30)
        prob, out = _run(sc, [0, 1, 2], np.ones(size[::-1], np.uint8), method, 7, sd=2.0)
        rep = f.check_estimate(prob, method, *out)
        f.assert_bounded(rep, (method, size))


def test_patch_one():
    sc = syn.textured_scene(3, 32, 24, seed=3)
    ones = np.ones((24, 32), np.uint8)
    for method in ("PATCH_MATCH", "PATCH_MATCH_SAMPLE"):
        with pytest.raises(ValueError, match="patch size 1"):
            _run(sc, [0, 1, 2], ones, method, 1, sd=0.0)
    prob, out = _run(sc, [0, 1, 2], ones, "BRUTE_FORCE", 1, sd=0.0)
    assert all((m == 0).all() for m in out)                 # one sample: every NCC is -1, nothing beats 0
    f.check_estimate(prob, "BRUTE_FORCE", *out)


# ---- mutations: the checker has teeth ---------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def outputs(small):
    sc, mask = small
    res = {}
    for method in METHODS:
        prob, out = _run(sc, [0, 1, 2, 3], mask, method, 7, planes=20)
        res[method] = (prob, [np.array(m) for m in out])
    return res


def _decided_pixel(prob, method, out, rng, need_depth=True):
    """A pixel whose score check is decided and far from every margin."""
    depth, plane, score, nghbr = out
    ok = (plane != 0).any(-1) & ((depth != 0) if need_depth else True)
    ii, jj = np.nonzero(ok)
    k = rng.permutation(len(ii))[:200]
    vs = prob.view_scores(ii[k], jj[k], plane[ii[k], jj[k]].astype(np.float64))
    _, nb, gap = f.plane_score(vs)
    good = (gap > 0.05) & np.all([(v.coord_margin > 1) & (v.var_margin > 1e3) for v in vs], 0) & (nb >= 1)
    good &= score[ii[k], jj[k]] > 0.2
    p = np.nonzero(good)[0][0]
    return ii[k][p], jj[k][p]


def _expect_fail(prob, method, out, match):
    with pytest.raises(AssertionError, match=match):
        f.check_estimate(prob, method, *out)


@pytest.mark.parametrize("method", ["BRUTE_FORCE", "PATCH_MATCH"])
def test_mutation_nghbr_swapped(outputs, method):
    prob, out = outputs[method]
    i, j = _decided_pixel(prob, method, out, np.random.RandomState(1))
    bad = [m.copy() for m in out]
    bad[3][i, j] = 1 + bad[3][i, j] % (prob.n - 1)
    _expect_fail(prob, method, bad, "nghbr|score")


@pytest.mark.parametrize("method", METHODS)
def test_mutation_plane_perturbed(outputs, method):
    prob, out = outputs[method]
    i, j = _decided_pixel(prob, method, out, np.random.RandomState(2))
    bad = [m.copy() for m in out]
    bad[1][i, j, 2] *= np.float32(1 + 1e-3)
    _expect_fail(prob, method, bad, "plane|depth|score")


@pytest.mark.parametrize("method", METHODS)
def test_mutation_score_shifted(outputs, method):
    prob, out = outputs[method]
    i, j = _decided_pixel(prob, method, out, np.random.RandomState(3))
    bad = [m.copy() for m in out]
    bad[2][i, j] += np.float32(1e-3)
    _expect_fail(prob, method, bad, "score")


def test_mutation_ignored_pixel_given_a_plane(outputs):
    for method in ("PATCH_MATCH", "PATCH_MATCH_SAMPLE"):
        prob, out = outputs[method]
        bad = [m.copy() for m in out]
        i, j = 4, 6                                                # inside the masked corner
        assert prob.mask[i, j] == 0 and (bad[1][i, j] == 0).all()
        i2, j2 = _decided_pixel(prob, method, out, np.random.RandomState(4))
        for m in bad:
            m[i, j] = m[i2, j2]
        _expect_fail(prob, method, bad, "ignored")


def test_mutation_brute_force_tie_to_later_plane():
    """Views that see the reference through a plane-independent warp (same pose, principal point shifted by half a
    pixel in x and y, the same image) score every depth plane identically, and identical copies tie every view: the first plane
    and the lowest view must win.  Resolving either tie the other way must fail."""
    sc = syn.textured_scene(2, 40, 30, seed=8)
    K1 = sc.K[0].copy()
    K1[:2, 2] += 0.5
    # R = I and one centre: Q = I and a = 0 exactly, so the homography does not depend on the plane
    Ks, Rs, ts = [sc.K[0], K1, K1], [np.eye(3)] * 3, [np.array([0.2, -0.1, 0.3])] * 3
    im = sc.gray[0]
    mask = np.ones_like(im)
    out = do.estimate(Ks, Rs, ts, [im, im, im], mask, "BRUTE_FORCE", 5, 10, 1, 25.0, 3.0, 30.0)
    prob = f.Problem(Ks, Rs, ts, [im, im, im], mask, 5, 5.0, 3.0, 30.0, 10)
    rep = f.check_estimate(prob, "BRUTE_FORCE", *out)
    assert rep.total_set_aside == 0 and rep.assigned > 500
    ii, jj = np.nonzero((out[1] != 0).any(-1))
    assert (out[1][ii, jj, 2] == out[1][ii[0], jj[0], 2]).all() and (out[3][ii, jj] == 1).all()
    later = [m.copy() for m in out]
    dep = np.float32(prob.depth_planes()[4])
    later[1][ii[7], jj[7], 2] = -(np.float32(1) / dep)
    later[0][ii[7], jj[7]] = dep
    _expect_fail(prob, "BRUTE_FORCE", later, "first depth plane")
    swapped = [m.copy() for m in out]
    swapped[3][ii[7], jj[7]] = 2
    _expect_fail(prob, "BRUTE_FORCE", swapped, "nghbr")


# ---- cleaning and pruning -----------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def maps():
    sc = syn.textured_scene(3, 64, 48, seed=9, arc_degrees=40)
    raw, planes = [], []
    for k in range(3):
        views = [k] + [v for v in range(3) if v != k]
        d, p, s, _ = do.estimate([sc.K[v] for v in views], [sc.R[v] for v in views], [sc.t[v] for v in views],
                                 [sc.gray[v] for v in views], np.ones((48, 64), np.uint8), "PATCH_MATCH_SAMPLE", 7, 30,
                                 2, 25.0, 3.0, 30.0, seed=2, key=k)
        raw.append(np.where((s > np.float32(0.1)) & (d < 30.0), d, 0).astype(np.float32))
        planes.append(p)
    return sc, raw, planes


@pytest.mark.parametrize("min_consistent", [1, 2, 3, 4])
def test_clean_and_prune_checkers_pass_oracle(maps, min_consistent):
    sc, raw, planes = maps
    cleaned = []
    for k in range(3):
        lst = [k] + [v for v in range(3) if v != k]
        args = ([sc.K[v] for v in lst], [sc.R[v] for v in lst], [sc.t[v] for v in lst])
        got = do.clean(*args, [raw[v] for v in lst], 0.01, min_consistent)
        aside = f.check_clean(*args, [raw[v] for v in lst], got, 0.01, min_consistent)
        assert aside <= 0.01 * max((raw[k] > 0).sum(), 1) + 2
        cleaned.append(got)
    for k in range(3):
        lst = [k] + [v for v in range(3) if v != k]
        args = ([sc.K[v] for v in lst], [sc.R[v] for v in lst], [sc.t[v] for v in lst])
        got = do.prune(*args, [cleaned[v] for v in lst], [planes[v] for v in lst], sc.rgb[k],
                       np.zeros((48, 64), np.uint8), 0.01)
        aside = f.check_prune(*args, [cleaned[v] for v in lst], [planes[v] for v in lst], got, 0.01)
        assert aside <= 0.01 * max((cleaned[k] > 0).sum(), 1) + 2
        if min_consistent <= 2:
            assert len(got[0]) > 100


def test_mutation_prune_point_dropped(maps):
    sc, raw, planes = maps
    lst = [0, 1, 2]
    args = ([sc.K[v] for v in lst], [sc.R[v] for v in lst], [sc.t[v] for v in lst])
    got = do.prune(*args, raw, planes, sc.rgb[0], np.zeros((48, 64), np.uint8), 0.01)
    keep, unsure, _, _ = f.prune(*args, raw, planes, 0.01)
    assert keep.sum() > 100
    f.check_prune(*args, raw, planes, got, 0.01)
    # drop the first point whose keep is decided
    r = f.project(got[0].astype(np.float64), sc.K[0], sc.R[0], sc.t[0])
    pj, pi = np.rint(r[:, 0] / r[:, 2]).astype(int), np.rint(r[:, 1] / r[:, 2]).astype(int)
    k = np.nonzero(~unsure[pi, pj])[0][0]
    dropped = tuple(np.delete(a, k, 0) for a in got)
    with pytest.raises(AssertionError, match="keeps is missing"):
        f.check_prune(*args, raw, planes, dropped, 0.01)
    # a clean map that keeps an inconsistent depth
    cl = do.clean(*args, raw, 0.01, 3)
    want, undecided = f.clean(*args, raw, 0.01, 3)
    i, j = np.argwhere((raw[0] > 0) & (cl == 0) & ~undecided)[0]
    bad = cl.copy()
    bad[i, j] = raw[0][i, j]
    with pytest.raises(AssertionError, match="clean map differs"):
        f.check_clean(*args, raw, bad, 0.01, 3)
