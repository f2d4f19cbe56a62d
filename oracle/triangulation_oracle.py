"""Triangulation of tracks in numpy: the CPU restatement that opensfm_b200/csrc/triangulate.cu is checked against.

What it restates:

  * `AngleBetweenVectors` (geometry/src/triangulation.cc): acos of u.v / sqrt(u.u v.v), 0 when that is at least 1 in
    absolute value (and NaN, which passes no comparison, for a zero vector);
  * `TriangulateBearingsMidpoint` (triangulation.cc:137-177): the angle test (some pair of world-frame bearings at an
    angle in [min_angle, pi - min_angle]), the closed-form midpoint of `TriangulateBearingsMidpointSolve`
    (geometry/triangulation.h:58-82) with the 3x3 inverse taken as Eigen takes it (cofactors times 1 / det), then per
    observation the reprojection test (angle of X - c_i to b_i above the threshold fails) and the depth test
    ((X - c_i) . b_i below min_depth fails);
  * `PointRefinement` (triangulation.cc:221-233): Ceres' TinySolver on the residuals normalize(X - c_i) - b_i with
    `Normalize::ForwardDerivatives` as the Jacobian.  TinySolver itself (ceres/tiny_solver.h) is not available to
    read here; `refine` follows its published algorithm with its default options:
      - Jacobi scaling s = 1 / (1 + column norms of J), fixed at the first evaluation; the normal equations are
        those of J diag(s): jtj = (J S)^T (J S), g = (J S)^T (-f); cost = |f|^2 / 2;
      - stop before any step if max |g| < 1e-10;
      - u = 1 / 1e4 (the initial trust-region radius), v = 2; iterations 1 .. max_num_iterations - 1:
        jtj + diag(u clamp(jtj_kk, 1e-6, 1e32)) by Cholesky, step = its solution for g, dx = s * step;
        stop if |dx| < 1e-8 (|x| + 1e-8);
        rho = (2 cost - |f(x + dx)|^2) / (step . (2 g - jtj step));
        rho > 0: accept, re-evaluate, stop if max |g| < 1e-10 or cost < machine epsilon, else
        u *= max(1/3, 1 - (2 rho - 1)^3), v = 2;  otherwise u *= v, v *= 2.
    The tests pin where it ends, not its path: from a valid midpoint the point it returns has a gradient of the
    bearing cost at round-off and equals an independent least-squares solve.
  * `TrackTriangulator.triangulate` (opensfm/reconstruction.py:1032-1073): keep a track's observations in shots of
    the reconstruction, stop below 2, rotate the camera-frame bearings to the world frame (R^T b), midpoint, and
    refine what passes; and `triangulate_shot_features` / `retriangulate` (:1143-1226), the loops over tracks that
    call it, with the "FULL" triangulation type.

`triangulate_tracks` runs the per-track restatement over the structure-of-arrays the engine takes, and also returns,
per track, how far the quantity that decided its status lay from its threshold (`margin`), so that a comparison can
set aside the tracks whose status a different summation order could flip.
"""
from __future__ import annotations

import math
from typing import Any, Dict, Tuple

import numpy as np

NOT_SELECTED, TOO_FEW, BAD_ANGLE, BAD_REPROJECTION, OK = range(5)

GRADIENT_TOLERANCE = 1e-10
PARAMETER_TOLERANCE = 1e-8
COST_THRESHOLD = np.finfo(np.float64).eps
INITIAL_TRUST_REGION = 1e4
MIN_DIAGONAL, MAX_DIAGONAL = 1e-6, 1e32


def angle_between_vectors(u: np.ndarray, v: np.ndarray) -> float:
    with np.errstate(invalid="ignore", divide="ignore"):
        c = float(np.dot(u, v) / math.sqrt(float(np.dot(u, u) * np.dot(v, v))))
    if abs(c) >= 1.0:
        return 0.0
    return math.acos(c) if c == c else float("nan")


def _inverse3(m: np.ndarray) -> np.ndarray:
    """Eigen's 3x3 inverse: cofactor (c, r) / det, det along the first column."""
    def cof(i, j):
        i1, i2, j1, j2 = (i + 1) % 3, (i + 2) % 3, (j + 1) % 3, (j + 2) % 3
        return m[i1, j1] * m[i2, j2] - m[i1, j2] * m[i2, j1]

    with np.errstate(divide="ignore", invalid="ignore"):
        invdet = 1.0 / (cof(0, 0) * m[0, 0] + cof(1, 0) * m[1, 0] + cof(2, 0) * m[2, 0])
        return np.array([[cof(c, r) * invdet for c in range(3)] for r in range(3)])


def midpoint_solve(centers: np.ndarray, bearings: np.ndarray) -> np.ndarray:
    """TriangulateBearingsMidpointSolve: the point closest to all rays, (I + BBt Cinv) A / n - Cinv BBtA."""
    n = len(centers)
    BBt = bearings.T @ bearings
    BBtA = np.einsum("ik,il,il->k", bearings, bearings, centers)
    A = centers.sum(axis=0)
    Cinv = _inverse3(n * np.eye(3) - BBt)
    with np.errstate(invalid="ignore", over="ignore"):
        return (np.eye(3) + BBt @ Cinv) @ A / n - Cinv @ BBtA


def _distance(q: float, threshold: float) -> float:
    return abs(q - threshold) if q == q else math.inf


def triangulate_bearings_midpoint(centers: np.ndarray, bearings: np.ndarray, thresholds, min_angle: float,
                                  min_depth: float) -> Tuple[int, np.ndarray, float]:
    """(status, midpoint, margin) of world-frame rays: OK, BAD_ANGLE or BAD_REPROJECTION; the midpoint is NaN unless
    OK.  margin: how far the deciding quantity lay from its threshold (inf when no comparison decided)."""
    n = len(centers)
    nan = np.full(3, np.nan)
    if len(thresholds) < n:
        return BAD_REPROJECTION, nan, math.inf
    passing, failing = [], []
    for i in range(n):
        for j in range(i):
            a = angle_between_vectors(bearings[i], bearings[j])
            d = min(_distance(a, min_angle), _distance(a, math.pi - min_angle))
            (passing if min_angle <= a <= math.pi - min_angle else failing).append(d)
    if not passing:
        return BAD_ANGLE, nan, min(failing, default=math.inf)
    # the pass is decided by its clearest pair; a status flips only if every passing pair flips
    margin = max(passing)
    X = midpoint_solve(centers, bearings)
    bad, good = [], []
    for i in range(n):
        p = X - centers[i]
        a = angle_between_vectors(p, bearings[i])
        depth = float(np.dot(p, bearings[i]))
        fails = [_distance(a, thresholds[i])] if a > thresholds[i] else []
        fails += [_distance(depth, min_depth)] if depth < min_depth else []
        if fails:
            bad.append(max(fails))
        else:
            good.append(min(_distance(a, thresholds[i]), _distance(depth, min_depth)))
    if bad:
        return BAD_REPROJECTION, nan, min(margin, max(bad))
    return OK, X, min(margin, min(good))


def bearing_cost(x: np.ndarray, centers: np.ndarray, bearings: np.ndarray, jacobian: bool = False):
    """f = normalize(x - c_i) - b_i stacked, and optionally the 3n x 3 Jacobian (Normalize::ForwardDerivatives)."""
    p = x[None, :] - centers
    n2 = (p * p).sum(axis=1)
    f = p / np.sqrt(n2)[:, None] - bearings
    if not jacobian:
        return f.ravel()
    J = (n2[:, None, None] * np.eye(3)[None] - p[:, :, None] * p[:, None, :]) / (np.sqrt(n2) * n2)[:, None, None]
    return f.ravel(), J.reshape(-1, 3)


def refine(centers: np.ndarray, bearings: np.ndarray, point: np.ndarray, iterations: int) -> np.ndarray:
    """PointRefinement: TinySolver's Levenberg-Marquardt (rules in the module docstring)."""
    x = np.array(point, dtype=np.float64)

    def update(x, s):
        f, J = bearing_cost(x, centers, bearings, jacobian=True)
        if s is None:
            s = 1.0 / (1.0 + np.linalg.norm(J, axis=0))
        Js = J * s[None, :]
        g = Js.T @ -f
        return 0.5 * float(f @ f), Js.T @ Js, g, s

    cost, jtj, g, s = update(x, None)
    if np.abs(g).max() < GRADIENT_TOLERANCE:
        return x
    u, v = 1.0 / INITIAL_TRUST_REGION, 2.0
    for _ in range(1, iterations):
        reg = jtj + np.diag(u * np.clip(np.diag(jtj), MIN_DIAGONAL, MAX_DIAGONAL))
        L = np.linalg.cholesky(reg)
        step = np.linalg.solve(L.T, np.linalg.solve(L, g))
        dx = s * step
        if np.linalg.norm(dx) < PARAMETER_TOLERANCE * (np.linalg.norm(x) + PARAMETER_TOLERANCE):
            break
        f_new = bearing_cost(x + dx, centers, bearings)
        cost_change = 2.0 * cost - float(f_new @ f_new)
        rho = cost_change / float(step @ (2.0 * g - jtj @ step))
        if rho > 0:
            x = x + dx
            cost, jtj, g, _ = update(x, s)
            if np.abs(g).max() < GRADIENT_TOLERANCE or cost < COST_THRESHOLD:
                break
            t = 2.0 * rho - 1.0
            u *= max(1.0 / 3.0, 1.0 - t * t * t)
            v = 2.0
        else:
            u *= v
            v *= 2.0
    return x


def triangulate_rays(centers: np.ndarray, bearings: np.ndarray, threshold: float, min_angle: float, min_depth: float,
                     iterations: int) -> Tuple[int, np.ndarray, float]:
    """TrackTriangulator.triangulate after the bearings are in the world frame: (status, X, margin)."""
    if len(centers) < 2:
        return TOO_FEW, np.full(3, np.nan), math.inf
    status, X, margin = triangulate_bearings_midpoint(centers, bearings, [threshold] * len(centers), min_angle,
                                                      min_depth)
    if status == OK:
        X = refine(centers, bearings, X, iterations)
    return status, X, margin


def triangulate_tracks(track_start: np.ndarray, obs_image: np.ndarray, image_rt: np.ndarray, image_origin: np.ndarray,
                       image_in: np.ndarray, bearings: np.ndarray, selected: np.ndarray, threshold: float,
                       min_angle: float, min_depth: float, iterations: int
                       ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(status[T], X[T, 3], margin[T]) over the engine's arrays (osfm_tracks_triangulate's inputs)."""
    T = len(track_start) - 1
    status = np.zeros(T, dtype=np.int8)
    X = np.full((T, 3), np.nan)
    margin = np.full(T, np.inf)
    rt = np.asarray(image_rt, dtype=np.float64).reshape(-1, 3, 3)
    for t in range(T):
        if not selected[t]:
            continue
        rows = np.arange(track_start[t], track_start[t + 1])
        rows = rows[np.asarray(image_in, dtype=bool)[obs_image[rows]]]
        im = obs_image[rows]
        w = np.einsum("nij,nj->ni", rt[im], bearings[rows])
        status[t], X[t], margin[t] = triangulate_rays(image_origin[im], w, threshold, min_angle, min_depth, iterations)
    return status, X, margin


# ---------------------------------------------------------------------------------------------------------------
# the reference's loops (reconstruction.py:1032-1073, 1143-1226) over a tracks manager and a reconstruction
# ---------------------------------------------------------------------------------------------------------------
def triangulate_track(tracks_manager, reconstruction, track: str, threshold: float, min_ray_angle_degrees: float,
                      min_depth: float, iterations: int) -> None:
    """TrackTriangulator.triangulate with TrackHandlerTrackManager: bearings from each shot's camera.pixel_bearing."""
    os_, bs, ids = [], [], []
    for shot_id, obs in tracks_manager.get_track_observations(track).items():
        if shot_id not in reconstruction.shots:
            continue
        shot = reconstruction.shots[shot_id]
        os_.append(shot.pose.get_origin())
        b = shot.camera.pixel_bearing(np.array(obs.point))
        bs.append(shot.pose.get_rotation_matrix().T.dot(b))
        ids.append(shot_id)
    status, X, _ = triangulate_rays(np.array(os_).reshape(-1, 3), np.array(bs).reshape(-1, 3), threshold,
                                    np.radians(min_ray_angle_degrees), min_depth, iterations)
    if status == OK:
        reconstruction.create_point(track, X.tolist())
        for shot_id in ids:
            reconstruction.add_observation(shot_id, track, tracks_manager.get_observation(shot_id, track))


def _options(config: Dict[str, Any]):
    return (config["triangulation_threshold"], config["triangulation_min_ray_angle"],
            config["triangulation_min_depth"], config["triangulation_refinement_iterations"])


def triangulate_shot_features(tracks_manager, reconstruction, shot_ids, config: Dict[str, Any]) -> None:
    all_shots_ids = set(tracks_manager.get_shot_ids())
    tracks_ids = {t for s in shot_ids if s in all_shots_ids for t in tracks_manager.get_shot_observations(s)}
    for track in tracks_ids:
        if track not in reconstruction.points and config["triangulation_type"] == "FULL":
            triangulate_track(tracks_manager, reconstruction, track, *_options(config))


def retriangulate(tracks_manager, reconstruction, config: Dict[str, Any]) -> Dict[str, Any]:
    report = {"num_points_before": len(reconstruction.points)}
    reconstruction.points = {}
    all_shots_ids = set(tracks_manager.get_shot_ids())
    tracks = set()
    for image in reconstruction.shots.keys():
        if image in all_shots_ids:
            tracks.update(tracks_manager.get_shot_observations(image).keys())
    for track in tracks:
        if config["triangulation_type"] == "FULL":
            triangulate_track(tracks_manager, reconstruction, track, *_options(config))
    report["num_points_after"] = len(reconstruction.points)
    return report
