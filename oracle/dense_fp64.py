"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product.

fp64 numpy restatement of pydense's DepthmapEstimator, DepthmapCleaner and DepthmapPruner
(opensfm/src/dense/src/depthmap.cc), written from the reference alone: it shares no code with oracle/dense_oracle.cpp
or the engine, and it does not reproduce their f32 arithmetic.  It answers "what should this output be" for maps that
come from anywhere (the C++ oracle on the CPU, the engine on the GPU), with a postcondition checker per method.

Every decided quantity comes with a margin: its distance to the nearest decision boundary of the reference (a sample
coordinate against 0 or cols - 1, a variance against 0.1 or the minimum patch variance, the top two scores against
each other, the 5 % post-process ratio, the clean and prune depth tests).  f32 arithmetic may land on either side of
a boundary it sits within its rounding of, so such a check is set aside and counted in the report, never skipped
silently; the caller bounds the count.

The tolerances below were calibrated on the C++ oracle's outputs, which the engine equals bit for bit
(tests/test_dense_fp64_cpu.py, tests/test_dense_limits_gpu.py); beside each is the largest value observed over those
cases, or the analytic bound it rests on.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

METHODS = ("BRUTE_FORCE", "PATCH_MATCH", "PATCH_MATCH_SAMPLE")
EPS32 = 2.0 ** -24

# |f32 score - fp64 score| <= SCORE_K * EPS32 * cond + 2 * (the samples' movement, see plane_image_score), with
# cond = mxx / varx + myy / vary (>= 2) the NCC's sensitivity to a relative error in its sums.  Observed: at most 0.31
# of this tolerance (patch 1 to 15, 40x30 to 640x480).
SCORE_K = 64.0
# A sample coordinate within COORD_K * EPS32 * (larger image side) pixels of 0 or cols - 1 (rows - 1) may be read on
# the other side of the bilinear bounds rule.  Observed f32-vs-fp64 sample coordinate difference: 11.5 in these units
# (4.4e-4 px at 640x480, 5.2e-5 px at 96x72).
COORD_K = 48.0
# The f32 coordinate error the score tolerance allows for, in the same units (the observed 11.5, rounded up).
COORD_ERR_K = 12.0
# A weighted NCC variance within VAR_K * EPS32 * (mean of squares) of 0.1 may fall on the other side of the gate.
VAR_K = 64.0
# Patch variance against min_patch_sd^2, relative: the f32 two-pass variance of at most 225 integers is within
# 225 * EPS32 (1.3e-5) of the exact one; this fp64 one is exact.
PATCH_VAR_RTOL = 4e-5
# depth against DepthOfPlaneBackprojection(plane), relative.  Observed: 8.8e-8 (a random initialisation that was never
# improved keeps the drawn depth, one f32 plane construction away from its plane).
DEPTH_RTOL = 1e-5
# The 5 % rule |d - m| / d against 0.05, absolute: d and m carry f32 rounding and the depth of the plane restated here
# differs from the f32 one by at most DEPTH_RTOL.
RATIO_TOL = 4e-5
# Clean / prune: a reprojected coordinate (px) within REPROJ_K * EPS32 * (larger image side) of the bounds rule or of
# a rounding boundary, and the depth tests within DEPTH_TEST_RTOL of the depth of the point, are set aside.  The
# reference rounds the point to f32 (relative 2^-24), which moves its reprojection by about f |X| / z * 2^-24, a few
# EPS32 * side for these scenes.
REPROJ_K = 16.0
DEPTH_TEST_RTOL = 1e-5


def view_terms(Ks, Rs, ts):
    """AddView's K^-1 of the reference, and Q_e = R_e R_0^T, a_e = Q_e t_0 - t_e of every view, in fp64."""
    K = np.asarray(Ks, np.float64).reshape(-1, 3, 3)
    R = np.asarray(Rs, np.float64).reshape(-1, 3, 3)
    t = np.asarray(ts, np.float64).reshape(-1, 3)
    Q = R @ R[0].T
    a = np.einsum("nij,j->ni", Q, t[0]) - t
    return K, np.linalg.inv(K[0]), Q, a


def plane_from_depth_and_normal(x, y, Kinv, depth, normal):
    """PlaneFromDepthAndNormal over arrays: normal / max(1e-6, -normal . (depth K^-1 (x, y, 1)))."""
    x, y, depth = (np.asarray(v, np.float64) for v in (x, y, depth))
    normal = np.asarray(normal, np.float64)
    X = np.stack([x, y, np.ones_like(x)], -1)
    p = depth[..., None] * (X @ np.asarray(Kinv, np.float64).T)
    denom = -(normal * p).sum(-1)
    return normal / np.maximum(1e-6, denom)[..., None]


def depth_of_plane(x, y, Kinv, plane):
    """DepthOfPlaneBackprojection over arrays: 1 / max(1e-6, -plane^T K^-1 (x, y, 1))."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    X = np.stack([x, y, np.ones_like(x)], -1)
    denom = -(np.asarray(plane, np.float64) * (X @ np.asarray(Kinv, np.float64).T)).sum(-1)
    return 1.0 / np.maximum(1e-6, denom)


def backproject(x, y, depth, K, R, t):
    """Backproject over arrays: R^T (depth K^-1 (x, y, 1) - t)."""
    x, y, depth = (np.asarray(v, np.float64) for v in (x, y, depth))
    X = np.stack([x, y, np.ones_like(x)], -1)
    q = depth[..., None] * (X @ np.linalg.inv(np.asarray(K, np.float64)).T) - np.asarray(t, np.float64)
    return q @ np.asarray(R, np.float64)


def project(X, K, R, t):
    return (np.asarray(X, np.float64) @ np.asarray(R, np.float64).T + np.asarray(t, np.float64)) @ \
        np.asarray(K, np.float64).T


def bilateral_weight(dcolor, dx, dy):
    """BilateralWeight, from its formula: exp(-dcolor^2 / (2 50^2) - (dx^2 + dy^2) / (2 5^2))."""
    return np.exp(-dcolor * dcolor / (2 * 50.0 ** 2) - (dx * dx + dy * dy) / (2 * 5.0 ** 2))


def _bounds_margin(x, y, cols, rows):
    """Inside [0, cols - 1) x [0, rows - 1): the distance by which the inside / outside decision could flip."""
    dx = np.minimum(np.abs(x), np.abs(x - (cols - 1)))
    dy = np.minimum(np.abs(y), np.abs(y - (rows - 1)))
    ox = (x < 0) | (x >= cols - 1)
    oy = (y < 0) | (y >= rows - 1)
    inside = ~ox & ~oy
    # outside: every violated side has to move back in for the decision to flip
    out_m = np.maximum(np.where(ox, dx, 0.0), np.where(oy, dy, 0.0))
    return np.where(inside, np.minimum(dx, dy), out_m), inside


def linear_interpolation(im, y, x):
    """LinearInterpolation in fp64: 0 outside [0, cols - 1) x [0, rows - 1); also the decision margin."""
    rows, cols = im.shape
    margin, inside = _bounds_margin(x, y, cols, rows)
    xs, ys = np.where(inside, x, 0.0), np.where(inside, y, 0.0)
    ix, iy = xs.astype(np.int64), ys.astype(np.int64)
    ix1, iy1 = np.minimum(ix + 1, cols - 1), np.minimum(iy + 1, rows - 1)
    dx, dy = xs - ix, ys - iy
    f = np.asarray(im, np.float64)
    im0 = (1 - dx) * f[iy, ix] + dx * f[iy, ix1]
    im1 = (1 - dx) * f[iy1, ix] + dx * f[iy1, ix1]
    return np.where(inside, (1 - dy) * im0 + dy * im1, 0.0), margin


def interpolation_slope(im, y, x):
    """|d/dx| + |d/dy| of LinearInterpolation inside its bounds (0 outside): how fast a sample moves with its
    coordinates."""
    rows, cols = im.shape
    _, inside = _bounds_margin(x, y, cols, rows)
    xs, ys = np.where(inside, x, 0.0), np.where(inside, y, 0.0)
    ix, iy = xs.astype(np.int64), ys.astype(np.int64)
    ix1, iy1 = np.minimum(ix + 1, cols - 1), np.minimum(iy + 1, rows - 1)
    dx, dy = xs - ix, ys - iy
    f = np.asarray(im, np.float64)
    gx = (1 - dy) * (f[iy, ix1] - f[iy, ix]) + dy * (f[iy1, ix1] - f[iy1, ix])
    gy = (1 - dx) * (f[iy1, ix] - f[iy, ix]) + dx * (f[iy1, ix1] - f[iy, ix1])
    return np.where(inside, np.abs(gx) + np.abs(gy), 0.0)


@dataclass
class Score:
    """ComputePlaneImageScore of N pixels, with what decides how far f32 may be from it."""
    score: np.ndarray          # fp64 NCC, or -1 where a gate rejects
    tol: np.ndarray            # how far an f32 evaluation may be from score where no margin is small
    coord_margin: np.ndarray   # px, smallest over the patch's samples
    var_margin: np.ndarray     # distance of the weighted variances to 0.1, in units of their f32 error


class Problem:
    """One reference (view 0) and its views, as DepthmapEstimator holds them after AddView and the setters."""

    def __init__(self, Ks, Rs, ts, images, mask, patch_size=7, min_patch_sd=5.0, min_depth=0.0, max_depth=0.0,
                 num_depth_planes=50):
        self.K, self.Kinv0, self.Q, self.a = view_terms(Ks, Rs, ts)
        self.Ks, self.Rs, self.ts = (np.asarray(v, np.float64) for v in (Ks, Rs, ts))
        self.images = [np.asarray(im, np.uint8) for im in images]
        self.mask = np.asarray(mask, np.uint8)
        self.n = len(self.images)
        self.patch = int(patch_size)
        self.hpz = (self.patch - 1) // 2
        sd = np.float32(min_patch_sd)
        self.min_var = float(sd * sd)          # SetMinPatchSD stores sd * sd as a float
        self.min_depth, self.max_depth, self.planes = float(min_depth), float(max_depth), int(num_depth_planes)
        self.h, self.w = self.images[0].shape
        self.side = max(max(im.shape) for im in self.images)
        self.coord_tol = COORD_K * EPS32 * self.side
        d = np.arange(-self.hpz, self.hpz + 1, dtype=np.float64)
        self.off_dy, self.off_dx = [g.ravel() for g in np.meshgrid(d, d, indexing="ij")]   # dy outer, dx inner

    # -- the score --------------------------------------------------------------------------------------------------

    def homography(self, planes, e):
        """K_e (Q_e + a_e v^T) K_0^-1 per plane v, (N, 3, 3)."""
        planes = np.asarray(planes, np.float64).reshape(-1, 3)
        M = self.Q[e][None] + self.a[e][None, :, None] * planes[:, None, :]
        return self.K[e][None] @ M @ self.Kinv0[None]

    def plane_image_score(self, i, j, planes, e, chunk=4096) -> Score:
        """ComputePlaneImageScore of plane (N, 3) at pixels (i, j) against view e (scalar or per pixel)."""
        i, j = np.asarray(i, np.int64).ravel(), np.asarray(j, np.int64).ravel()
        planes = np.asarray(planes, np.float64).reshape(-1, 3)
        N = len(i)
        e = np.broadcast_to(np.asarray(e, np.int64), (N,))
        if N > chunk:
            parts = [self.plane_image_score(i[k:k + chunk], j[k:k + chunk], planes[k:k + chunk], e[k:k + chunk])
                     for k in range(0, N, chunk)]
            return Score(*[np.concatenate([getattr(p, f) for p in parts])
                           for f in ("score", "tol", "coord_margin", "var_margin")])
        out = Score(np.full(N, -1.0), np.zeros(N), np.full(N, np.inf), np.full(N, np.inf))
        fi, fj = i.astype(np.float64), j.astype(np.float64)
        ref = self.images[0].astype(np.float64)
        im1 = ref[i[:, None] + self.off_dy[None].astype(np.int64), j[:, None] + self.off_dx[None].astype(np.int64)]
        center = ref[i, j]
        wgt = bilateral_weight(im1 - center[:, None], self.off_dx[None], self.off_dy[None])
        for view in np.unique(e):
            s = np.nonzero(e == view)[0]
            H = self.homography(planes[s], view)
            u = H[:, 0, 0] * fj[s] + H[:, 0, 1] * fi[s] + H[:, 0, 2]
            v = H[:, 1, 0] * fj[s] + H[:, 1, 1] * fi[s] + H[:, 1, 2]
            w = H[:, 2, 0] * fj[s] + H[:, 2, 1] * fi[s] + H[:, 2, 2]
            ok = w != 0
            with np.errstate(divide="ignore", invalid="ignore"):
                ww = w * w
                dfdx_x = (H[:, 0, 0] * w - H[:, 2, 0] * u) / ww
                dfdx_y = (H[:, 1, 0] * w - H[:, 2, 0] * v) / ww
                dfdy_x = (H[:, 0, 1] * w - H[:, 2, 1] * u) / ww
                dfdy_y = (H[:, 1, 1] * w - H[:, 2, 1] * v) / ww
                x2 = (u / w)[:, None] + dfdx_x[:, None] * self.off_dx[None] + dfdy_x[:, None] * self.off_dy[None]
                y2 = (v / w)[:, None] + dfdx_y[:, None] * self.off_dx[None] + dfdy_y[:, None] * self.off_dy[None]
            x2 = np.where(ok[:, None], x2, -1.0)
            y2 = np.where(ok[:, None], y2, -1.0)
            im2, cm = linear_interpolation(self.images[view], y2, x2)
            slope = interpolation_slope(self.images[view], y2, x2)
            x1, wt = im1[s], wgt[s]
            sw = wt.sum(1)
            mx, my = (wt * x1).sum(1) / sw, (wt * im2).sum(1) / sw
            mxx, myy, mxy = (wt * x1 * x1).sum(1) / sw, (wt * im2 * im2).sum(1) / sw, (wt * x1 * im2).sum(1) / sw
            varx, vary = mxx - mx * mx, myy - my * my
            gate = (varx < 0.1) | (vary < 0.1) | ~ok
            with np.errstate(divide="ignore", invalid="ignore"):
                ncc = (mxy - mx * my) / np.sqrt(varx * vary)
                cond = np.where(gate, 0.0, mxx / varx + myy / vary)
                # f32 sample coordinates are off by up to coord_err: the samples move by slope * coord_err, which
                # moves the NCC by about their weighted rms over the other variance's root
                moved = COORD_ERR_K * EPS32 * self.side * np.sqrt((wt * slope * slope).sum(1) / sw) / np.sqrt(vary)
                moved = np.where(gate, 0.0, moved)
            out.score[s] = np.where(gate, -1.0, ncc)
            out.tol[s] = SCORE_K * EPS32 * cond + 2 * moved
            out.coord_margin[s] = np.where(ok, cm.min(1), np.inf)
            vm = np.minimum(np.abs(varx - 0.1) / (EPS32 * np.maximum(mxx, 1.0)),
                            np.abs(vary - 0.1) / (EPS32 * np.maximum(myy, 1.0)))
            out.var_margin[s] = np.where(ok, vm, np.inf)
        return out

    def view_scores(self, i, j, planes) -> List[Score]:
        return [self.plane_image_score(i, j, planes, e) for e in range(1, self.n)]

    # -- pieces of the estimator -------------------------------------------------------------------------------------

    def depth_planes(self):
        """ComputeBruteForce's depths: 1 / (1 / min + d (1 / max - 1 / min) / (planes - 1)), or min for one plane."""
        if self.planes <= 1:
            return np.array([self.min_depth])
        d = np.arange(self.planes, dtype=np.float64)
        return 1.0 / (1.0 / self.min_depth + d * (1.0 / self.max_depth - 1.0 / self.min_depth) / (self.planes - 1))

    def patch_variance(self):
        """PatchVariance of every pixel whose patch lies inside the image (NaN elsewhere), exact for u8 images."""
        P, h, w = self.patch, self.h, self.w
        f = self.images[0].astype(np.float64)
        S = np.zeros((h + 1, w + 1))
        S2 = np.zeros((h + 1, w + 1))
        S[1:, 1:] = f.cumsum(0).cumsum(1)
        S2[1:, 1:] = (f * f).cumsum(0).cumsum(1)
        out = np.full((h, w), np.nan)
        if P > h or P > w:
            return out
        box = lambda T: T[P:, P:] - T[:-P, P:] - T[P:, :-P] + T[:-P, :-P]
        n = float(P * P)
        s, s2 = box(S), box(S2)
        out[self.hpz:h - self.hpz, self.hpz:w - self.hpz] = (s2 - s * s / n) / n
        return out

    def interior(self):
        m = np.zeros((self.h, self.w), bool)
        m[self.hpz:self.h - self.hpz, self.hpz:self.w - self.hpz] = True
        return m


def plane_score(view_scores: Sequence[Score]):
    """ComputePlaneScore over precomputed per-view scores: strictly greater wins, starting from (-1, 0).  Returns the
    score, the local view index, and the decision margin: the gap between the winner and the best loser (the start
    value -1 included) minus both tolerances; exact ties count as decided (the lowest index wins them)."""
    S = np.stack([s.score for s in view_scores], 1)                       # (N, n - 1)
    T = np.stack([s.tol for s in view_scores], 1)
    best = np.full(S.shape[0], -1.0)
    nb = np.zeros(S.shape[0], np.int64)
    for e in range(S.shape[1]):
        win = S[:, e] > best
        best = np.where(win, S[:, e], best)
        nb = np.where(win, e + 1, nb)
    Sx = np.concatenate([np.full((S.shape[0], 1), -1.0), S], 1)
    Tx = np.concatenate([np.zeros((S.shape[0], 1)), T], 1)
    tw = np.take_along_axis(Tx, nb[:, None], 1)[:, 0]
    gap = best[:, None] - Sx
    gap = np.where(gap == 0, np.inf, np.abs(gap) - Tx - tw[:, None])   # an exact tie is decided by the index
    gap[np.arange(len(nb)), nb] = np.inf
    return best, nb, gap.min(1)


def median5(depth):
    """cv::medianBlur(depth, 5) with replicated borders, in fp64."""
    p = np.pad(np.asarray(depth, np.float64), 2, mode="edge")
    win = np.lib.stride_tricks.sliding_window_view(p, (5, 5))
    return np.median(win.reshape(depth.shape + (25,)), -1)


# ---- the checker ------------------------------------------------------------------------------------------------------


@dataclass
class Report:
    """What a check decided and what it set aside, with the largest f32-versus-fp64 errors seen."""
    sampled: int = 0                      # sampled pixels with a plane
    checked: int = 0                      # of those, pixels whose score was compared
    assigned: int = 0                     # pixels with a plane
    set_aside: Dict[str, int] = field(default_factory=dict)
    max_score_err: float = 0.0            # |score - fp64 score| where decided
    max_score_err_rel_tol: float = 0.0    # the same in units of the tolerance (must stay <= 1)
    max_depth_rel_err: float = 0.0        # |depth - DepthOfPlaneBackprojection(plane)| / depth

    def aside(self, what, count):
        if count:
            self.set_aside[what] = self.set_aside.get(what, 0) + int(count)

    @property
    def total_set_aside(self):
        return sum(self.set_aside.values())


# Set-aside bounds.  Map-wide rules (patch variance, the 5 % rule): a fraction of the assigned pixels.  Per-pixel score
# rules (bounds, gates, top two views, top two depth planes): a fraction of the sampled pixels, which at 640x480 lean
# towards the border band where warps leave the image; observed up to 6.3 % there (brute force, 3 views), up to
# 2.6 % on the smaller scenes.
ASIDE_FRACTION = 0.01
SAMPLE_ASIDE_FRACTION = 0.08
_MAP_WIDE = ("patch variance at min_patch_sd^2", "post-process ratio at 5 %")


def assert_bounded(rep: Report, what=""):
    wide = sum(rep.set_aside.get(k, 0) for k in _MAP_WIDE)
    assert wide <= ASIDE_FRACTION * max(rep.assigned, 1) + 2, (what, rep)
    assert rep.total_set_aside - wide <= SAMPLE_ASIDE_FRACTION * max(rep.sampled, 1) + 2, (what, rep)
    assert rep.max_score_err_rel_tol <= 1.0, (what, rep)


def sample_pixels(prob: Problem, count=4096, seed=0, full_below=160 * 120):
    """Pixels the score checks run on: every interior pixel of an image up to full_below pixels; otherwise a fixed
    random sample of count interior pixels, plus every interior pixel within two pixels of the interior's border or
    of a mask edge."""
    inner = prob.interior()
    if prob.h * prob.w <= full_below:
        return np.nonzero(inner)
    rng = np.random.RandomState(seed)
    pick = np.zeros_like(inner)
    ii, jj = np.nonzero(inner)
    k = rng.choice(len(ii), min(count, len(ii)), replace=False)
    pick[ii[k], jj[k]] = True
    h, w, b = prob.h, prob.w, prob.hpz + 2
    edge = np.zeros_like(inner)
    edge[:b + 1] = edge[-b - 1:] = True
    edge[:, :b + 1] = edge[:, -b - 1:] = True
    m = prob.mask > 0
    near = np.zeros_like(m)
    for di in range(-2, 3):
        for dj in range(-2, 3):
            near |= np.roll(np.roll(m, di, 0), dj, 1) != m
    return np.nonzero(inner & (pick | edge | near))


def _fail(what, where):
    idx = np.argwhere(where)
    raise AssertionError("%s at %d pixels, first (i, j) = %s" % (what, len(idx), tuple(idx[0]) if len(idx) else None))


def check_estimate(prob: Problem, method: str, depth, plane, score, nghbr, pixels=None,
                   brute_force_optimality: Optional[bool] = None) -> Report:
    """The postconditions of DepthmapEstimator's output (ungated depth, plane, score, nghbr as a list-local view
    index) for method, from any source.  Raises AssertionError naming the first violated rule."""
    assert method in METHODS, method
    depth, score = np.asarray(depth, np.float32), np.asarray(score, np.float32)
    plane, nghbr = np.asarray(plane, np.float32), np.asarray(nghbr)
    h, w, hpz = prob.h, prob.w, prob.hpz
    rep = Report()
    inner = prob.interior()
    has_plane = (plane != 0).any(-1)
    rep.assigned = int(has_plane.sum())

    # the border band is never written
    band = ~inner
    if (depth[band] != 0).any() or (plane[band] != 0).any() or (score[band] != 0).any() or (nghbr[band] != 0).any():
        _fail("the border band of width %d is not zero" % hpz, band & ((depth != 0) | has_plane | (score != 0) |
                                                                        (nghbr != 0)))
    # the four maps agree on which pixels were assigned
    bad = ~has_plane & ((depth != 0) | (score != 0) | (nghbr != 0))
    if bad.any():
        _fail("a pixel without a plane has a depth, score or view", bad)
    # nghbr: a list-local view in [1, n); PatchMatch's best-of-views keeps view 0 only when every view scored -1
    low = 0 if method == "PATCH_MATCH" else 1
    bad = has_plane & ((nghbr < low) | (nghbr >= prob.n))
    if method == "PATCH_MATCH":
        bad |= has_plane & (nghbr == 0) & (score != -1)
    if bad.any():
        _fail("nghbr out of range", bad)

    pv = prob.patch_variance()
    if method != "BRUTE_FORCE":
        # masked and low-variance pixels are ignored: all zero; every other interior pixel has a plane
        low_var = pv < prob.min_var
        near = np.abs(pv - prob.min_var) <= PATCH_VAR_RTOL * max(1.0, prob.min_var)
        ignored = inner & ((prob.mask == 0) | low_var) & ~(near & (prob.mask != 0))
        live = inner & (prob.mask != 0) & ~low_var & ~near
        if has_plane[ignored].any():
            _fail("an ignored (masked or low-variance) pixel has a plane", ignored & has_plane)
        if (~has_plane[live]).any():
            _fail("a live pixel has no plane", live & ~has_plane)
        rep.aside("patch variance at min_patch_sd^2", (inner & near & (prob.mask != 0)).sum())
        # depth is 0 or DepthOfPlaneBackprojection(plane) to f32 rounding
        ii, jj = np.nonzero(has_plane)
        dop = np.zeros((h, w))
        dop[ii, jj] = depth_of_plane(jj, ii, prob.Kinv0, plane[ii, jj])
        d = depth.astype(np.float64)
        kept = has_plane & (depth != 0)
        rel = np.abs(d - dop) / np.maximum(dop, 1e-30)
        rep.max_depth_rel_err = float(rel[kept].max()) if kept.any() else 0.0
        if (rel[kept] > DEPTH_RTOL).any():
            _fail("depth differs from the depth of its plane", kept & (rel > DEPTH_RTOL))
        # PostProcess: zeroed exactly where the 5 % median rule says, on the maps before it (depth of the plane)
        m = median5(dop)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(dop > 0, np.abs(dop - m) / dop, np.inf)
        drop = (dop == 0) | (ratio > 0.05)
        near = (dop > 0) & (np.abs(ratio - 0.05) <= RATIO_TOL)
        rep.aside("post-process ratio at 5 %", near.sum())
        if ((depth != 0) & drop & ~near).any():
            _fail("a depth the 5 % rule removes was kept", (depth != 0) & drop & ~near)
        if ((depth == 0) & ~drop & ~near).any():
            _fail("a depth the 5 % rule keeps was removed", (depth == 0) & ~drop & ~near)

    # scores at the sampled pixels: the engine's own (plane, nghbr), and for BF / PM the best view
    if pixels is None:
        pixels = sample_pixels(prob)
    pi, pj = pixels
    sel = has_plane[pi, pj]
    pi, pj = pi[sel], pj[sel]
    rep.sampled = len(pi)
    if len(pi):
        pl = plane[pi, pj].astype(np.float64)
        nb = nghbr[pi, pj].astype(np.int64)
        sc = score[pi, pj].astype(np.float64)
        if method == "PATCH_MATCH_SAMPLE":
            own = prob.plane_image_score(pi, pj, pl, nb)
            s64, tol = own.score, own.tol
            unsure = (own.coord_margin < prob.coord_tol) | (own.var_margin < VAR_K)
        else:
            vs = prob.view_scores(pi, pj, pl)
            s64, nb64, gap = plane_score(vs)
            tol = np.stack([v.tol for v in vs], 1)[np.arange(len(pi)), np.maximum(nb - 1, 0)]
            unsure = np.zeros(len(pi), bool)
            for v in vs:
                unsure |= (v.coord_margin < prob.coord_tol) | (v.var_margin < VAR_K)
            undecided = ~unsure & (gap <= 0)
            rep.aside("top two views within tolerance", undecided.sum())
            dec = ~unsure & ~undecided
            if (nb[dec] != nb64[dec]).any():
                bad = np.zeros((h, w), bool)
                bad[pi[dec][nb[dec] != nb64[dec]], pj[dec][nb[dec] != nb64[dec]]] = True
                _fail("nghbr is not the best view (lowest index on ties)", bad)
            s64 = np.where(nb == nb64, s64, np.stack([v.score for v in vs], 1)[np.arange(len(pi)),
                                                                                 np.maximum(nb - 1, 0)])
        rep.aside("sample coordinate or variance at a gate", unsure.sum())
        ok = ~unsure
        err = np.abs(sc - s64)
        rep.checked = int(ok.sum())
        if ok.any():
            rep.max_score_err = float(err[ok].max())
            rep.max_score_err_rel_tol = float((err[ok] / np.maximum(tol[ok], 1e-300)).max())
        if (err[ok] > tol[ok]).any():
            bad = np.zeros((h, w), bool)
            bad[pi[ok][err[ok] > tol[ok]], pj[ok][err[ok] > tol[ok]]] = True
            _fail("score differs from the fp64 score of its plane and view", bad)

    if method == "BRUTE_FORCE":
        _check_brute_force(prob, depth, plane, score, has_plane, rep, pixels, brute_force_optimality)
    return rep


def _check_brute_force(prob, depth, plane, score, has_plane, rep, pixels, optimality):
    """Brute force: the plane is fronto-parallel, of one of the depth planes; with optimality, it is the first depth
    plane that maximises the score, and pixels whose best score is <= 0 stay zero.  The ignore mask is not applied."""
    deps = prob.depth_planes()
    pz = -1.0 / deps                                   # the fronto-parallel plane (0, 0, -1 / depth)
    ii, jj = np.nonzero(has_plane)
    p = plane[ii, jj].astype(np.float64)
    if (p[:, :2] != 0).any():
        _fail("a brute-force plane is not fronto-parallel", has_plane & (plane[..., :2] != 0).any(-1))
    idx = np.abs(p[:, 2:3] - pz[None]).argmin(1)
    rel = np.abs(p[:, 2] - pz[idx]) / np.abs(pz[idx])
    if (rel > DEPTH_RTOL).any():
        bad = np.zeros(has_plane.shape, bool)
        bad[ii[rel > DEPTH_RTOL], jj[rel > DEPTH_RTOL]] = True
        _fail("a brute-force plane is none of the depth planes", bad)
    d_of = np.full(has_plane.shape, -1, np.int64)
    d_of[ii, jj] = idx
    dop = depth_of_plane(jj, ii, prob.Kinv0, p)
    rel = np.abs(depth[ii, jj] - dop) / dop
    rep.max_depth_rel_err = max(rep.max_depth_rel_err, float(rel.max()) if len(rel) else 0.0)
    if (rel > DEPTH_RTOL).any():
        bad = np.zeros(has_plane.shape, bool)
        bad[ii[rel > DEPTH_RTOL], jj[rel > DEPTH_RTOL]] = True
        _fail("depth differs from the depth of its plane", bad)
    if (score[has_plane] <= 0).any():
        _fail("a brute-force pixel was assigned a score <= 0", has_plane & (score <= 0))
    if optimality is None:
        optimality = prob.h * prob.w <= 160 * 120
    if not optimality:
        return
    pi, pj = pixels
    n = len(pi)
    S = np.empty((n, len(deps)))
    T = np.empty((n, len(deps)))
    unsure = np.zeros(n, bool)
    for d, dep in enumerate(deps):
        pl = np.broadcast_to(np.array([0.0, 0.0, -1.0 / dep]), (n, 3))
        vs = prob.view_scores(pi, pj, pl)
        S[:, d], nb, _ = plane_score(vs)
        T[:, d] = np.stack([np.zeros(n)] + [v.tol for v in vs], 1)[np.arange(n), nb]
        for v in vs:
            unsure |= (v.coord_margin < prob.coord_tol) | (v.var_margin < VAR_K)
    best = S.max(1)
    first = S.argmax(1)                                # the first index among exact ties
    # zero: the best fp64 score is <= 0, away from 0
    zero_ok = ~unsure & (best <= -T.max(1))
    got = d_of[pi, pj]
    if (got[zero_ok] >= 0).any():
        bad = np.zeros(has_plane.shape, bool)
        bad[pi[zero_ok & (got >= 0)], pj[zero_ok & (got >= 0)]] = True
        _fail("a brute-force pixel whose best score is <= 0 was assigned", bad)
    pos_ok = ~unsure & (best > T.max(1))
    if (got[pos_ok] < 0).any():
        bad = np.zeros(has_plane.shape, bool)
        bad[pi[pos_ok & (got < 0)], pj[pos_ok & (got < 0)]] = True
        _fail("a brute-force pixel with a positive best score was left empty", bad)
    rep.aside("brute-force best score at 0", (~unsure & ~zero_ok & ~pos_ok).sum())
    # the first maximum: any other plane within both tolerances of the winner, not an exact tie, is undecided
    k = np.nonzero(pos_ok & (got >= 0))[0]
    Sk, Tk, gk, fk = S[k], T[k], got[k], first[k]
    sw = Sk[np.arange(len(k)), gk]
    tw = Tk[np.arange(len(k)), gk]
    diff = Sk - sw[:, None]
    near = (np.abs(diff) <= Tk + tw[:, None]) & (diff != 0)
    near[np.arange(len(k)), gk] = False
    undecided = near.any(1)
    rep.aside("brute-force top two planes within tolerance", undecided.sum())
    worse = diff > Tk + tw[:, None]                  # a plane clearly better than the one chosen
    bad = worse.any(1) | (~undecided & (gk != fk))
    if bad.any():
        m = np.zeros(has_plane.shape, bool)
        m[pi[k[bad]], pj[k[bad]]] = True
        _fail("a brute-force plane is not the first depth plane maximising the score", m)


def check_gate(depth, score, raw, min_score, max_depth):
    """compute_depthmap's gate: raw is depth where score > min_score and depth < max_depth, else 0 (exactly)."""
    want = np.where((np.asarray(score, np.float32) > np.float32(min_score)) &
                    (np.asarray(depth, np.float64) < max_depth), depth, 0).astype(np.float32)
    if not np.array_equal(np.asarray(raw, np.float32), want):
        _fail("the raw map is not the gated depth", np.asarray(raw) != want)


# ---- cleaning and pruning ---------------------------------------------------------------------------------------------


def clean(Ks, Rs, ts, depths, same_depth_threshold=0.01, min_consistent_views=2):
    """DepthmapCleaner::Clean of view 0 in fp64.  Returns the clean depth and the pixels whose decision sits within
    the tolerances of a boundary (a reprojection against the bounds rule, |d_at - d| against d * threshold, or the
    count of consistent views against the minimum)."""
    d0 = np.asarray(depths[0], np.float32)
    h, w = d0.shape
    ii, jj = np.mgrid[:h, :w]
    X = backproject(jj.ravel(), ii.ravel(), d0.ravel().astype(np.float64), Ks[0], Rs[0], ts[0])
    rt = REPROJ_K * EPS32 * max(max(np.shape(d)) for d in depths)
    sure = np.zeros(h * w, np.int64)
    maybe = np.zeros(h * w, np.int64)
    for o in range(1, len(depths)):
        r = project(X, Ks[o], Rs[o], ts[o])
        z = r[:, 2]
        front = z >= 1e-8
        with np.errstate(divide="ignore", invalid="ignore"):
            u, v = r[:, 0] / z, r[:, 1] / z
        u, v = np.where(front, u, -1.0), np.where(front, v, -1.0)
        do = np.asarray(depths[o], np.float32)
        da, cm = linear_interpolation(do, v, u)
        lhs, rhs = np.abs(da - z), z * same_depth_threshold
        ok = front & (lhs < rhs)
        # the interpolated depth moves with the reprojection's rounding, steeply across a depth edge
        near = np.abs(lhs - rhs) <= DEPTH_TEST_RTOL * np.abs(z) + interpolation_slope(do, v, u) * rt
        unsure = front & ((cm < rt) | near)
        sure += ok & ~unsure
        maybe += unsure
    cons_lo, cons_hi = 1 + sure, 1 + sure + maybe
    keep = cons_lo >= min_consistent_views
    undecided = (cons_lo < min_consistent_views) & (cons_hi >= min_consistent_views)
    out = np.where(keep, d0.ravel(), 0).astype(np.float32).reshape(h, w)
    return out, (undecided & (d0.ravel() != 0)).reshape(h, w)


def _normalize(v):
    n = np.linalg.norm(v, axis=-1, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(n > 0, v / n, 0.0)


def prune(Ks, Rs, ts, depths, planes, same_depth_threshold=0.01):
    """DepthmapPruner::Prune of view 0 in fp64: per pixel whether it is kept, whether that sits within the tolerances
    of a boundary (rounding of the reprojection to a pixel, the depth test, the area test), and its point and
    world-frame normal."""
    d0 = np.asarray(depths[0], np.float32).astype(np.float64)
    h, w = d0.shape
    ii, jj = np.mgrid[:h, :w]
    pos = d0.ravel() > 0
    nrm = _normalize(np.asarray(planes[0], np.float64).reshape(-1, 3))
    with np.errstate(divide="ignore", invalid="ignore"):
        area = -nrm[:, 2] / d0.ravel() * Ks[0][0][0]
    X = backproject(jj.ravel(), ii.ravel(), d0.ravel(), Ks[0], Rs[0], ts[0])
    rt = REPROJ_K * EPS32 * max(max(np.shape(d)) for d in depths)
    hides_any = np.zeros(h * w, bool)     # some view hides the point: the reference drops it
    drop_sure = np.zeros(h * w, bool)     # some view hides it away from every boundary
    unsure = np.zeros(h * w, bool)
    for o in range(1, len(depths)):
        r = project(X, Ks[o], Rs[o], ts[o])
        z = r[:, 2]
        front = z >= 1e-8
        with np.errstate(divide="ignore", invalid="ignore"):
            fu, fv = r[:, 0] / z + 0.5, r[:, 1] / z + 0.5
        fu, fv = np.where(front, fu, -1e9), np.where(front, fv, -1e9)
        iu, iv = np.trunc(fu), np.trunc(fv)            # static_cast<int64_t> truncates toward zero
        near_int = (np.abs(fu - np.round(fu)) < rt) | (np.abs(fv - np.round(fv)) < rt)
        do, po = np.asarray(depths[o], np.float32), np.asarray(planes[o], np.float64)
        ho, wo = do.shape
        inside = front & (iu >= 0) & (iu < wo) & (iv >= 0) & (iv < ho)
        q_i, q_j = np.where(inside, iv, 0).astype(np.int64), np.where(inside, iu, 0).astype(np.int64)
        da = do[q_i, q_j].astype(np.float64)
        thr = (1 - same_depth_threshold) * z
        closer = inside & (da > thr)
        no = _normalize(po[q_i, q_j])
        with np.errstate(divide="ignore", invalid="ignore"):
            ao = -no[:, 2] / da * Ks[o][0][0]
        hides = closer & ((da == 0) | (ao > area))
        u_here = front & pos & (near_int | (inside & ((np.abs(da - thr) <= DEPTH_TEST_RTOL * np.abs(z)) |
                                                     (closer & (np.abs(ao - area) <= DEPTH_TEST_RTOL * np.abs(area))))))
        unsure |= u_here
        hides_any |= hides
        drop_sure |= hides & ~u_here
    keep = pos & ~hides_any
    normals = nrm @ np.asarray(Rs[0], np.float64)        # R^T n, as rows
    return (keep.reshape(h, w), (unsure & pos & ~drop_sure).reshape(h, w), X.reshape(h, w, 3),
            normals.reshape(h, w, 3))


def check_clean(Ks, Rs, ts, depths, got, same_depth_threshold, min_consistent_views):
    """The clean map from any source against the fp64 cleaner; returns the number of pixels set aside."""
    want, undecided = clean(Ks, Rs, ts, depths, same_depth_threshold, min_consistent_views)
    got = np.asarray(got, np.float32)
    bad = (got != want) & ~undecided
    if bad.any():
        _fail("the clean map differs from the fp64 cleaner", bad)
    # an undecided pixel still either keeps its raw depth or is zero
    d0 = np.asarray(depths[0], np.float32)
    if ((got != d0) & (got != 0)).any():
        _fail("a clean depth is neither its raw depth nor zero", (got != d0) & (got != 0))
    return int(undecided.sum())


def check_prune(Ks, Rs, ts, depths, planes, got, same_depth_threshold):
    """Pruned (points, normals, colours, labels) from any source against the fp64 pruner: each point is recovered to
    its pixel by projecting it into view 0; the kept pixels come in raster order, every decided keep is present and
    every decided drop absent.  Returns the number of pixels set aside."""
    keep, unsure, X, N = prune(Ks, Rs, ts, depths, planes, same_depth_threshold)
    pts, nrm = np.asarray(got[0], np.float64), np.asarray(got[1], np.float64)
    h, w = keep.shape
    if len(pts):
        r = project(pts, Ks[0], Rs[0], ts[0])
        pj, pi = np.rint(r[:, 0] / r[:, 2]).astype(np.int64), np.rint(r[:, 1] / r[:, 2]).astype(np.int64)
        if not ((pi >= 0) & (pi < h) & (pj >= 0) & (pj < w)).all():
            raise AssertionError("a pruned point does not project into the reference")
        flat = pi * w + pj
        if (np.diff(flat) <= 0).any():
            raise AssertionError("pruned points are not in raster order, or repeat a pixel")
        scale = np.abs(X[pi, pj]).max(1) + 1.0
        if (np.abs(pts - X[pi, pj]).max(1) > 1e-5 * scale).any():
            raise AssertionError("a pruned point is not the backprojection of its pixel")
        if (np.abs(nrm - N[pi, pj]).max(1) > 1e-5).any():
            raise AssertionError("a pruned normal is not R^T normalize(plane) of its pixel")
    else:
        flat = np.zeros(0, np.int64)
    present = np.zeros(h * w, bool)
    present[flat] = True
    present = present.reshape(h, w)
    if (keep & ~unsure & ~present).any():
        _fail("a point the fp64 pruner keeps is missing", keep & ~unsure & ~present)
    if (~keep & ~unsure & present).any():
        _fail("a point the fp64 pruner drops is present", ~keep & ~unsure & present)
    return int(unsure.sum())
