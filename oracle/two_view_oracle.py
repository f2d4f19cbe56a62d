"""The two-view stage of `two_view_reconstruction_general` after its RANSAC, in numpy, one pair at a time: the
restatement that rp_two_view (opensfm_b200/csrc/relpose.cu) is checked against.  It starts from a given lo_model
(RANSAC is oracle/relative_pose_oracle.py's) and a given plane motion (the host's, opensfm_b200.relative_pose).

What it restates (opensfm/reconstruction.py:298-560, matching.py:805-844, multiview.py:541-553,
geometry/relative_pose.h:86-183):

  * poses are [R | t] in compute_inliers_bearings' convention: the second camera sits at t and sees the world
    direction R y.  RANSAC's configuration is [R_l^T | -R_l^T t_l] of lo_model = [R_l | t_l]; the transposed one,
    checked when check_reversal, is (R^T, -R^T t) of that;
  * bearing inliers: the midpoint X of the rays (0, x) and (t, R y) (TriangulateTwoBearingsMidpointSolve, no result
    when |det| < 1e-10), an inlier when |X / |X| - x| < threshold and |R^T (X - t) / |.| - y| < threshold;
  * with more than 5 inliers, RelativePoseRefinement on them: the parameters are the angle-axis of R^T
    (RotationMatrixToAngleAxis through the quaternion) and t; RelativePoseCost has 100 rows picked from the inliers
    (ascending) by index = int(float32(rand_k) / float32(RAND_MAX) * count), rand_k the k-th glibc rand() after
    srand(42), and 101 residuals: 1 - (px . x + py . y) / 2 with both rotations by AngleAxisRotatePoint (first-order
    branch when |aa|^2 <= DBL_EPSILON), exactly 1 with no derivative when the midpoint fails, and 1 - |t|; then
    TinySolver with max_num_iterations = iterations (`tiny_solver` below), AngleAxisToRotationMatrix back, and the
    inliers again;
  * a configuration with at most 5 final inliers is dropped; of two, none is kept when min / max > reversal_ratio,
    else the larger, the transposed one on a tie;
  * the 5-point result when it exists and has strictly more inliers than the plane result, else the plane result
    when there is a plane motion, else none.  The plane result is always motion 0 (see
    opensfm_b200.relative_pose.plane_motion for the reference's argmax).

TinySolver (ceres/tiny_solver.h) follows the rules oracle/triangulation_oracle.py's docstring states for `refine`;
`tiny_solver` is that loop over any residual function, and tests/test_two_view_oracle.py checks that it returns
`triangulation_oracle.refine`'s points bit for bit on the bearing cost.

Deliberate differences from the reference, all at rounding level:
  * the Jacobian comes from a forward-mode dual number with plain division (Ceres' Jet divides through the
    reciprocal) and the residual values from the same expressions;
  * the 2 x 2 midpoint solve is relpose::midpoint's (adjugate over det), not Eigen's inverse times b;
  * the engine sums J^T J, J^T f and f . f in a warp's tree order, and solves its 6 x 6 system by its own Cholesky.

Every thresholded decision's margin is recorded (`TwoView.margins`): the smallest distance of a chord that decided a
row to the threshold, the smallest distance of a midpoint |det| to 1e-10, and the count gaps behind the Necker ratio,
the "> 5" rule and the 5-point / plane choice.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np

from oracle.relative_pose_oracle import MIDPOINT_DET_EPS, normalize_rows
from oracle.triangulation_oracle import (COST_THRESHOLD, GRADIENT_TOLERANCE, INITIAL_TRUST_REGION, MAX_DIAGONAL,
                                         MIN_DIAGONAL, PARAMETER_TOLERANCE)

PICKED = 100
RAND_MAX = 2147483647
MIN_INLIERS = 6
DBL_EPSILON = float(np.finfo(np.float64).eps)


# ---------------------------------------------------------------------------------------------------------------
# glibc rand() and the picked rows
# ---------------------------------------------------------------------------------------------------------------
def glibc_rand(seed: int, count: int) -> List[int]:
    """The first `count` outputs of rand() after srand(seed): random_r's TYPE_3 additive generator (degree 31,
    separation 3), seeded by 16807 * r mod (2^31 - 1), 310 outputs discarded."""
    r = [seed & 0xffffffff]
    for i in range(1, 31):
        r.append((16807 * r[i - 1]) % 2147483647)
    r += r[:3]
    for i in range(34, 344 + count):
        r.append((r[i - 31] + r[i - 3]) & 0xffffffff)
    return [v >> 1 for v in r[344:]]


def pick_fractions() -> np.ndarray:
    """float(rand_k) / float(RAND_MAX), k < 100, in float32."""
    return np.array(glibc_rand(42, PICKED), dtype=np.int64).astype(np.float32) / np.float32(RAND_MAX)


def picked_positions(count: int) -> np.ndarray:
    """RelativePoseCost's positions in the inlier list of `count` rows: int(fraction * count) in float32."""
    return (pick_fractions() * np.float32(count)).astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------
# forward-mode dual numbers over the 6 parameters
# ---------------------------------------------------------------------------------------------------------------
class Dual:
    """Values v (any shape) with their derivatives d (shape + (6,))."""

    def __init__(self, v, d=None):
        self.v = np.asarray(v, dtype=np.float64)
        self.d = np.zeros(self.v.shape + (6,)) if d is None else d

    @staticmethod
    def lift(a) -> "Dual":
        return a if isinstance(a, Dual) else Dual(a)

    def __add__(self, o):
        o = Dual.lift(o)
        return Dual(self.v + o.v, self.d + o.d)

    __radd__ = __add__

    def __sub__(self, o):
        o = Dual.lift(o)
        return Dual(self.v - o.v, self.d - o.d)

    def __rsub__(self, o):
        return Dual.lift(o) - self

    def __neg__(self):
        return Dual(-self.v, -self.d)

    def __mul__(self, o):
        o = Dual.lift(o)
        return Dual(self.v * o.v, self.d * o.v[..., None] + self.v[..., None] * o.d)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = Dual.lift(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = self.v / o.v
            return Dual(v, (self.d - v[..., None] * o.d) / o.v[..., None])

    def __rtruediv__(self, o):
        return Dual.lift(o) / self

    def sqrt(self):
        with np.errstate(divide="ignore", invalid="ignore"):
            v = np.sqrt(self.v)
            return Dual(v, self.d / (2.0 * v)[..., None])

    def sin(self):
        return Dual(np.sin(self.v), np.cos(self.v)[..., None] * self.d)

    def cos(self):
        return Dual(np.cos(self.v), -np.sin(self.v)[..., None] * self.d)


def parameters(p: np.ndarray) -> List[Dual]:
    """The 6 parameters as duals seeded with the unit directions."""
    return [Dual(p[i], np.eye(6)[i].copy()) for i in range(6)]


def angle_axis_rotate(aa: List[Dual], pt: List[Dual]) -> List[Dual]:
    """ceres::AngleAxisRotatePoint; the branch is decided by the value of |aa|^2."""
    theta2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2]
    if float(theta2.v) > DBL_EPSILON:
        theta = theta2.sqrt()
        c, s = theta.cos(), theta.sin()
        inv = 1.0 / theta
        w = [aa[0] * inv, aa[1] * inv, aa[2] * inv]
        wxp = [w[1] * pt[2] - w[2] * pt[1], w[2] * pt[0] - w[0] * pt[2], w[0] * pt[1] - w[1] * pt[0]]
        tmp = (w[0] * pt[0] + w[1] * pt[1] + w[2] * pt[2]) * (1.0 - c)
        return [pt[i] * c + wxp[i] * s + w[i] * tmp for i in range(3)]
    wxp = [aa[1] * pt[2] - aa[2] * pt[1], aa[2] * pt[0] - aa[0] * pt[2], aa[0] * pt[1] - aa[1] * pt[0]]
    return [pt[i] + wxp[i] for i in range(3)]


def relative_pose_cost(p: np.ndarray, x: np.ndarray, y: np.ndarray) -> Dual:
    """RelativePoseCost's residuals at p over the picked rows (x, y) (k x 3 each), then 1 - |t|: a Dual of k + 1
    values and their 6 derivatives."""
    P = parameters(p)
    X_ = [Dual(x[:, c]) for c in range(3)]
    Y_ = [Dual(y[:, c]) for c in range(3)]
    t = P[3:]
    by = angle_axis_rotate([-P[0], -P[1], -P[2]], Y_)
    r0 = t[0] * X_[0] + t[1] * X_[1] + t[2] * X_[2]
    r1 = t[0] * by[0] + t[1] * by[1] + t[2] * by[2]
    a00 = X_[0] * X_[0] + X_[1] * X_[1] + X_[2] * X_[2]
    a10 = X_[0] * by[0] + X_[1] * by[1] + X_[2] * by[2]
    a01 = -a10
    a11 = -(by[0] * by[0] + by[1] * by[1] + by[2] * by[2])
    det = a00 * a11 - a01 * a10
    ok = ~((-MIDPOINT_DET_EPS < det.v) & (det.v < MIDPOINT_DET_EPS))
    l0 = (a11 * r0 - a01 * r1) / det
    l1 = (a00 * r1 - a10 * r0) / det
    X = [0.5 * (l0 * X_[c] + (t[c] + l1 * by[c])) for c in range(3)]
    q = angle_axis_rotate(P[:3], [X[c] - t[c] for c in range(3)])
    nx = (X[0] * X[0] + X[1] * X[1] + X[2] * X[2]).sqrt()
    nq = (q[0] * q[0] + q[1] * q[1] + q[2] * q[2]).sqrt()
    ax = (X[0] / nx) * X_[0] + (X[1] / nx) * X_[1] + (X[2] / nx) * X_[2]
    ay = (q[0] / nq) * Y_[0] + (q[1] / nq) * Y_[1] + (q[2] / nq) * Y_[2]
    f = 1.0 - (ax + ay) * 0.5
    v = np.where(ok, f.v, 1.0)
    d = np.where(ok[:, None], f.d, 0.0)
    last = 1.0 - (t[0] * t[0] + t[1] * t[1] + t[2] * t[2]).sqrt()
    return Dual(np.append(v, last.v), np.vstack([d, last.d[None, :]]))


# ---------------------------------------------------------------------------------------------------------------
# TinySolver over a residual function
# ---------------------------------------------------------------------------------------------------------------
def tiny_solver(residuals: Callable[[np.ndarray, bool], Tuple[np.ndarray, Optional[np.ndarray]]], x0: np.ndarray,
                iterations: int) -> np.ndarray:
    """Ceres' TinySolver from x0 with max_num_iterations = iterations, the rules of triangulation_oracle.refine:
    residuals(x, jacobian) returns (f, J or None)."""
    x = np.array(x0, dtype=np.float64)

    def update(x, s):
        f, J = residuals(x, True)
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
        f_new, _ = residuals(x + dx, False)
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


# ---------------------------------------------------------------------------------------------------------------
# rotations (ceres/rotation.h) and the refinement's parametrisation
# ---------------------------------------------------------------------------------------------------------------
def rotation_to_angle_axis(R: np.ndarray) -> np.ndarray:
    """ceres::RotationMatrixToAngleAxis: the quaternion (trace branch, else the largest diagonal), then the angle
    by atan2 with the sign of the scalar part folded in."""
    q = np.zeros(4)
    trace = R[0, 0] + R[1, 1] + R[2, 2]
    if trace >= 0.0:
        t = math.sqrt(trace + 1.0)
        q[0] = 0.5 * t
        t = 0.5 / t
        q[1] = (R[2, 1] - R[1, 2]) * t
        q[2] = (R[0, 2] - R[2, 0]) * t
        q[3] = (R[1, 0] - R[0, 1]) * t
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = math.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        q[i + 1] = 0.5 * t
        t = 0.5 / t
        q[0] = (R[k, j] - R[j, k]) * t
        q[j + 1] = (R[j, i] + R[i, j]) * t
        q[k + 1] = (R[k, i] + R[i, k]) * t
    s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    k = 2.0
    if s2 > 0.0:
        s, c = math.sqrt(s2), q[0]
        k = 2.0 * (math.atan2(-s, -c) if c < 0.0 else math.atan2(s, c)) / s
    return q[1:] * k


def angle_axis_to_rotation(aa: np.ndarray) -> np.ndarray:
    """ceres::AngleAxisToRotationMatrix, first-order when |aa|^2 <= DBL_EPSILON."""
    theta2 = float(aa @ aa)
    if theta2 > DBL_EPSILON:
        theta = math.sqrt(theta2)
        w = aa / theta
        c, s = math.cos(theta), math.sin(theta)
        return c * np.eye(3) + (1.0 - c) * np.outer(w, w) + s * np.array(
            [[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    return np.array([[1.0, -aa[2], aa[1]], [aa[2], 1.0, -aa[0]], [-aa[1], aa[0], 1.0]])


def refine_parameters(B: np.ndarray) -> np.ndarray:
    """relative_pose_optimize_nonlinear's [R^T | -R^T t] of B = [R | t], as RelativePoseRefinement parametrises it."""
    R, t = B[:, :3], B[:, 3]
    Rt, tc = R.T, -(R.T @ t)
    return np.concatenate([rotation_to_angle_axis(Rt), -(R @ tc)])


def refine_pose(p: np.ndarray) -> np.ndarray:
    """... and back: R' = AngleAxisToRotationMatrix(p), t' = -R' p_t, B = [R'^T | -R'^T t']."""
    R = angle_axis_to_rotation(p[:3])
    tr = -(R @ p[3:])
    return np.column_stack([R.T, -(R.T @ tr)])


def refine(B: np.ndarray, x: np.ndarray, y: np.ndarray, inliers: np.ndarray, iterations: int) -> np.ndarray:
    """RelativePoseRefinement of B on the inlier rows (ascending indices into x, y)."""
    rows = inliers[picked_positions(len(inliers))]
    xs, ys = x[rows], y[rows]

    def residuals(p, jacobian):
        f = relative_pose_cost(p, xs, ys)
        return f.v, (f.d if jacobian else None)

    return refine_pose(tiny_solver(residuals, refine_parameters(B), iterations))


# ---------------------------------------------------------------------------------------------------------------
# bearing inliers and the decisions
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class Margins:
    chord: float = math.inf     # min distance to the threshold of a chord that decided a row
    det: float = math.inf       # min distance of a midpoint |det| to 1e-10
    necker: float = math.inf    # min |count - max count| gap behind the Necker ratio (two configurations kept)
    min_inliers: float = math.inf   # min |count - 5.5| behind a "> 5" rule
    method: float = math.inf    # |5-point count - plane count| when both results exist


def bearing_inliers(B: np.ndarray, x: np.ndarray, y: np.ndarray, threshold: float,
                    margins: Optional[Margins] = None) -> np.ndarray:
    """matching.compute_inliers_bearings of every row under B = [R | t]: a boolean mask."""
    R, t = B[:, :3], B[:, 3]
    by = y @ R.T
    r0, r1 = x @ t, by @ t
    a00 = np.einsum("ij,ij->i", x, x)
    a10 = np.einsum("ij,ij->i", x, by)
    a01, a11 = -a10, -np.einsum("ij,ij->i", by, by)
    det = a00 * a11 - a01 * a10
    ok = ~((-MIDPOINT_DET_EPS < det) & (det < MIDPOINT_DET_EPS))
    with np.errstate(divide="ignore", invalid="ignore"):
        l0 = (a11 * r0 - a01 * r1) / det
        l1 = (a00 * r1 - a10 * r0) / det
        X = 0.5 * (l0[:, None] * x + (t[None, :] + l1[:, None] * by))
        br1 = X / np.linalg.norm(X, axis=1)[:, None]
        br2 = (X - t) @ R
        br2 = br2 / np.linalg.norm(br2, axis=1)[:, None]
        d1 = np.linalg.norm(br1 - x, axis=1)
        d2 = np.linalg.norm(br2 - y, axis=1)
        inl = ok & (d1 < threshold) & (d2 < threshold)
    if margins is not None and np.isfinite(B).all():
        margins.det = min(margins.det, float(np.min(np.abs(np.abs(det) - MIDPOINT_DET_EPS))))
        e1, e2 = np.abs(d1 - threshold), np.abs(d2 - threshold)
        with np.errstate(invalid="ignore"):
            # an inlier flips when either chord does; an outlier only when every failing chord does
            m_in = np.minimum(e1, e2)
            m_out = np.maximum(np.where(d1 >= threshold, e1, 0.0), np.where(d2 >= threshold, e2, 0.0))
            m = np.where(inl, m_in, m_out)[ok]
        m = m[np.isfinite(m)]
        if len(m):
            margins.chord = min(margins.chord, float(m.min()))
    return inl


def necker(counts: List[int], reversal_ratio: float) -> int:
    """two_view_reconstruction_5pt's choice among the configurations' final counts (one or two, the given pose
    first): the index kept, or -1."""
    kept = [c for c, n in enumerate(counts) if n >= MIN_INLIERS]
    if len(kept) == 1:
        return kept[0]
    if len(kept) == 2:
        n1, n2 = counts
        if min(n1, n2) / max(n1, n2) > reversal_ratio:
            return -1
        return 0 if n1 > n2 else 1
    return -1


def decide(five_point_count: Optional[int], plane_count: Optional[int]) -> Optional[str]:
    """two_view_reconstruction_general's choice: "5_point", "plane_based" or None.  A count is None when that
    method has no result."""
    if five_point_count is not None and five_point_count > (plane_count or 0):
        return "5_point"
    if plane_count is not None:
        return "plane_based"
    return None


@dataclass
class TwoView:
    pose: np.ndarray              # (2, 3, 4) final pose of each configuration, NaN when not run
    counts: np.ndarray            # (3,) final inliers of each configuration, then of the plane motion
    chosen: int
    mask_5pt: np.ndarray
    mask_plane: np.ndarray
    method: Optional[str]
    margins: Margins = field(default_factory=Margins)


def two_view(b1: np.ndarray, b2: np.ndarray, lo_model: np.ndarray, plane_pose: np.ndarray, threshold: float,
             iterations: int, check_reversal: bool = False, reversal_ratio: float = 1.0) -> TwoView:
    """The two-view stage of one pair from RANSAC's lo_model [R_l | t_l] and the plane motion [R_p | t_p] (NaN when
    there is none)."""
    x, y = normalize_rows(b1), normalize_rows(b2)
    mg = Margins()
    Rl, tl = lo_model[:, :3], lo_model[:, 3]
    B0 = np.column_stack([Rl.T, -(Rl.T @ tl)])
    configs = [B0, np.column_stack([B0[:, :3].T, -(B0[:, :3].T @ B0[:, 3])])] if check_reversal else [B0]
    pose = np.full((2, 3, 4), np.nan)
    counts = np.zeros(3, dtype=np.int64)
    finals = []
    for c, B in enumerate(configs):
        inl = np.nonzero(bearing_inliers(B, x, y, threshold, mg))[0]
        mg.min_inliers = min(mg.min_inliers, abs(len(inl) - (MIN_INLIERS - 0.5)))
        if len(inl) >= MIN_INLIERS:
            B = refine(B, x, y, inl, iterations)
        mask = bearing_inliers(B, x, y, threshold, mg)
        pose[c], counts[c] = B, mask.sum()
        mg.min_inliers = min(mg.min_inliers, abs(counts[c] - (MIN_INLIERS - 0.5)))
        finals.append(mask)
    chosen = necker([int(n) for n in counts[:len(configs)]], reversal_ratio)
    if len(configs) == 2 and min(counts[:2]) >= MIN_INLIERS:
        mg.necker = float(abs(counts[0] - counts[1]))
    Rp, tp = plane_pose[:, :3], plane_pose[:, 3]
    has_plane = bool(np.isfinite(plane_pose).all())
    mask_plane = (bearing_inliers(np.column_stack([Rp.T, -(Rp.T @ tp)]), x, y, threshold, mg) if has_plane
                  else np.zeros(len(x), bool))
    counts[2] = mask_plane.sum()
    mask_5pt = finals[chosen] if chosen >= 0 else np.zeros(len(x), bool)
    if chosen >= 0 and has_plane:
        mg.method = float(abs(int(counts[chosen]) - int(counts[2])))
    method = decide(int(counts[chosen]) if chosen >= 0 else None, int(counts[2]) if has_plane else None)
    return TwoView(pose, counts, chosen, mask_5pt, mask_plane, method, mg)
