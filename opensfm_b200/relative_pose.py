"""Five-point relative-pose RANSAC of many image pairs at once on the GPU (opensfm_b200/csrc/relpose.cu, C ABI
osfm_relpose_*): the estimator `two_view_reconstruction_general` starts the two-view bootstrap with.  The rules, and
the deliberate differences from pyrobust, are stated in oracle/relative_pose_oracle.py.  There is no CPU path.

The input is one bearing table and, per row, the index of the first image's bearing and of the second image's;
pairs own consecutive rows (`pair_start`).  `ransac_lists` builds that from per-pair (b1, b2) arrays
(`pack_lists`, the shared `ransac.pack_pairs`), and
`relative_pose_ransac` is the drop-in of `opensfm.multiview.relative_pose_ransac` for one pair.  `robust_match_pairs`
and `robust_match_lists` run the geometric verification of `matching.robust_match_calibrated` on the same batches.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Any, Dict, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import ptr
from .ransac import Engine, batch_rows, pack_pairs

ITERATIONS = 1000   # what two_view_reconstruction_general passes

_last_device_ms = 0.0


@dataclass
class PairsResult:
    lo_model: np.ndarray          # (P, 3, 4): pyrobust's result.lo_model, [R | t] with x2 = R x1 + t
    ransac_inliers: np.ndarray    # (P,) int32
    inlier_mask: np.ndarray       # (R,) bool: the rows lo_model keeps (result.inliers_indices)
    pair_start: np.ndarray        # (P + 1,) int64
    device_ms: float

    def poses(self) -> np.ndarray:
        """(P, 3, 4) [R^T | -R^T t]: what multiview.relative_pose_ransac returns."""
        R = self.lo_model[:, :, :3]
        t = self.lo_model[:, :, 3]
        Rt = R.transpose(0, 2, 1)
        return np.concatenate([Rt, -np.einsum("pij,pj->pi", Rt, t)[:, :, None]], axis=2)

    def inliers(self, p: int) -> np.ndarray:
        """Inlier mask of pair p's rows."""
        return self.inlier_mask[self.pair_start[p]:self.pair_start[p + 1]]


class RelativePose(Engine):
    """osfm_relpose (ransac.Engine): the problems are image pairs."""

    kind = "relpose"

    def run(self, bearings: np.ndarray, pair_start: np.ndarray, row_a: np.ndarray, row_b: np.ndarray,
            threshold: float, iterations: int = ITERATIONS) -> PairsResult:
        bearings = np.ascontiguousarray(bearings, dtype=np.float64).reshape(-1, 3)
        pair_start, row_a, row_b = batch_rows(pair_start, row_a, row_b)
        P = len(pair_start) - 1
        lo = np.zeros((P, 3, 4), dtype=np.float64)
        ransac = np.zeros(P, dtype=np.int32)
        mask = np.zeros(len(row_a), dtype=np.uint8)
        _lib.check(self.L.osfm_relpose_run(self.h, len(bearings), ptr(bearings), P, ptr(pair_start), ptr(row_a),
                                           ptr(row_b), float(threshold), int(iterations), ptr(lo), ptr(ransac),
                                           ptr(mask)))
        self._num_problems = P
        return PairsResult(lo, ransac, mask.view(bool), pair_start, self._device_ms())


def ransac_pairs(bearings: np.ndarray, pair_start: np.ndarray, row_a: np.ndarray, row_b: np.ndarray,
                 threshold: float, iterations: int = ITERATIONS, device: int = 0) -> PairsResult:
    """Every pair's five-point relative-pose RANSAC; rows index one bearing table."""
    global _last_device_ms
    with _lib.pooled("relpose", device) as h:
        res = RelativePose(handle=h).run(bearings, pair_start, row_a, row_b, threshold, iterations)
    _last_device_ms = res.device_ms
    return res


def last_device_ms() -> float:
    """Device time of the last ransac_pairs / ransac_lists call."""
    return _last_device_ms


pack_lists = pack_pairs   # (bearing table, pair_start, row_a, row_b) of per-pair (b1, b2) arrays


def ransac_lists(b1_list: Sequence[np.ndarray], b2_list: Sequence[np.ndarray], threshold: float,
                 iterations: int = ITERATIONS, device: int = 0) -> PairsResult:
    return ransac_pairs(*pack_lists(b1_list, b2_list), threshold, iterations, device)


def relative_pose_ransac(b1: np.ndarray, b2: np.ndarray, threshold: float, iterations: int,
                         probability: float) -> np.ndarray:
    """multiview.relative_pose_ransac: [R^T | -R^T t] (3 x 4) of pyrobust's lo_model [R | t].  `probability` is
    accepted and, as in the reference, not used: pyrobust's stopping rule keeps its default of 0.99."""
    return ransac_lists([b1], [b2], threshold, iterations).poses()[0]


# ---------------------------------------------------------------------------------------------------------------
# two_view_reconstruction_general after the RANSAC: refinement, bearing inliers, Necker check, plane motion
# ---------------------------------------------------------------------------------------------------------------
REFINE_ITERATIONS = 1000      # five_point_refine_rec_iterations
PLANE_SINGULAR_RATIO = 1.0001  # no motion when two singular values of H are closer than this ratio
MIN_INLIERS = 6               # a configuration is refined, and kept, with more than 5 inliers

_last_stage_ms = (0.0, 0.0)


def plane_motions(H: Optional[np.ndarray]):
    """The up to 8 motions (R, t, n, d) of the plane homography H in normalised coordinates, by Faugeras and
    Lustman's decomposition ("Motion and structure from motion in a piecewise planar environment", INRIA report
    856, 1988), with H = d R + t n^T; None when H is None or two of its singular values d1 >= d2 >= d3 are within a
    ratio of 1.0001.

    With H = U diag(d1, d2, d3) V^T and s = det U det V, a motion of the diagonal problem (R', t', n') gives R =
    s U R' V^T, t = U t', n = V n', d = s d'.  For e1, e3 in {+1, -1}, x1 = e1 sqrt((d1^2 - d2^2) / (d1^2 - d3^2)),
    x3 = e3 sqrt((d2^2 - d3^2) / (d1^2 - d3^2)) and n' = (x1, 0, x3):
      d' = d2:  R' = rotation about y by theta, sin theta = (d1 - d3) x1 x3 / d2, cos theta = (d3 x1^2 + d1 x3^2) / d2,
                t' = (d1 - d3) (x1, 0, -x3);
      d' = -d2: R' = reflection-rotation with sin phi = (d1 + d3) x1 x3 / d2, cos phi = (d3 x1^2 - d1 x3^2) / d2,
                t' = (d1 + d3) (x1, 0, x3).
    The order is (e1, e3) = (+, +), (+, -), (-, +), (-, -), each with d' > 0 first."""
    if H is None:
        return None
    U, sv, Vt = np.linalg.svd(np.asarray(H, dtype=np.float64))
    d1, d2, d3 = sv
    if d1 / d2 < PLANE_SINGULAR_RATIO or d2 / d3 < PLANE_SINGULAR_RATIO:
        return None
    s = np.linalg.det(U) * np.linalg.det(Vt)
    denominator = d1 * d1 - d3 * d3
    a1 = np.sqrt((d1 * d1 - d2 * d2) / denominator)
    a3 = np.sqrt((d2 * d2 - d3 * d3) / denominator)
    motions = []
    for x1, x3 in ((a1, a3), (a1, -a3), (-a1, a3), (-a1, -a3)):
        n = Vt.T @ np.array([x1, 0.0, x3])
        sin_theta = (d1 - d3) * x1 * x3 / d2
        cos_theta = (d3 * x1 * x1 + d1 * x3 * x3) / d2
        Rp = np.array([[cos_theta, 0.0, -sin_theta], [0.0, 1.0, 0.0], [sin_theta, 0.0, cos_theta]])
        motions.append((s * (U @ Rp @ Vt), U @ ((d1 - d3) * np.array([x1, 0.0, -x3])), n, s * d2))
        sin_phi = (d1 + d3) * x1 * x3 / d2
        cos_phi = (d3 * x1 * x1 - d1 * x3 * x3) / d2
        Rn = np.array([[cos_phi, 0.0, sin_phi], [0.0, -1.0, 0.0], [sin_phi, 0.0, -cos_phi]])
        motions.append((s * (U @ Rn @ Vt), U @ ((d1 + d3) * np.array([x1, 0.0, x3])), n, -s * d2))
    return motions


def plane_motion(b1: np.ndarray, b2: np.ndarray, threshold: float) -> np.ndarray:
    """two_view_reconstruction_plane_based's motion [R_p | t_p] (3 x 4) of one pair, NaN when there is none:
    cv2.findHomography(RANSAC, threshold) of the bearings' image-plane points, then the first of plane_motions.

    The reference picks `motions[np.argmax(map(len, motion_inliers))]`.  numpy turns a map object into a 0-d object
    array, whose argmax is 0 whatever the inlier counts, so its plane result is always the first motion; this keeps
    that behaviour (and computes the inliers of that motion only, on the device)."""
    import cv2

    b1 = np.asarray(b1, dtype=np.float64)
    b2 = np.asarray(b2, dtype=np.float64)
    H, _ = cv2.findHomography(b1[:, :2] / b1[:, 2:], b2[:, :2] / b2[:, 2:], cv2.RANSAC, threshold)
    motions = plane_motions(H)
    if not motions:
        return np.full((3, 4), np.nan)
    R, t, _, _ = motions[0]
    return np.column_stack([R, t])


@dataclass
class TwoViewResult:
    lo_model: np.ndarray          # (P, 3, 4) as PairsResult.lo_model
    ransac_inliers: np.ndarray    # (P,) int32
    pose: np.ndarray              # (P, 2, 3, 4): each configuration's final [R | t], second image to first (NaN: not run)
    counts: np.ndarray            # (P, 3) int32: final inliers of each configuration, then of the plane motion
    chosen: np.ndarray            # (P,) int32: the configuration the 5-point result keeps (1: transposed), -1: none
    mask_5pt: np.ndarray          # (R,) bool
    mask_plane: np.ndarray        # (R,) bool
    plane: np.ndarray             # (P, 3, 4): the plane motion [R_p | t_p], NaN when there is none
    pair_start: np.ndarray
    ransac_ms: float
    two_view_ms: float

    def rows(self, p: int) -> slice:
        return slice(int(self.pair_start[p]), int(self.pair_start[p + 1]))

    def method(self, p: int) -> Optional[str]:
        """"5_point", "plane_based" or None (no initial motion)."""
        c = int(self.chosen[p])
        if c >= 0 and self.counts[p, c] > self.mask_plane[self.rows(p)].sum():
            return "5_point"
        return None if np.isnan(self.plane[p]).any() else "plane_based"

    def result(self, p: int):
        """two_view_reconstruction_general's (R, t, inliers, report) of pair p: R an angle-axis vector, t the
        translation, inliers the row indices."""
        import cv2

        c = int(self.chosen[p])
        inliers_5p = np.nonzero(self.mask_5pt[self.rows(p)])[0]
        inliers_plane = np.nonzero(self.mask_plane[self.rows(p)])[0]
        report: Dict[str, Any] = {"5_point_inliers": len(inliers_5p), "plane_based_inliers": len(inliers_plane)}
        method = self.method(p)
        if method == "5_point":
            report["method"] = method
            R, t = self.pose[p, c, :, :3], self.pose[p, c, :, 3]
            return cv2.Rodrigues(R.T)[0].ravel(), -R.T.dot(t), inliers_5p, report
        if method == "plane_based":
            report["method"] = method
            return cv2.Rodrigues(self.plane[p, :, :3].copy())[0].ravel(), self.plane[p, :, 3].copy(), inliers_plane, report
        report["decision"] = "Could not find initial motion"
        return None, None, [], report


def two_view_pairs(bearings: np.ndarray, pair_start: np.ndarray, row_a: np.ndarray, row_b: np.ndarray,
                   threshold: float, iterations: int = REFINE_ITERATIONS, check_reversal: bool = False,
                   reversal_ratio: float = 1.0, device: int = 0) -> TwoViewResult:
    """two_view_reconstruction_general of every pair (rows index one bearing table, as ransac_pairs): the plane
    motions on the host, then RANSAC and the two-view stage on the device in one call.  `iterations` is the
    refinement's (five_point_refine_rec_iterations); RANSAC runs its 1000."""
    global _last_device_ms, _last_stage_ms
    bearings = np.ascontiguousarray(bearings, dtype=np.float64).reshape(-1, 3)
    pair_start, row_a, row_b = batch_rows(pair_start, row_a, row_b)
    P = len(pair_start) - 1
    plane = np.full((P, 3, 4), np.nan)
    for p in range(P):
        a, b = row_a[pair_start[p]:pair_start[p + 1]], row_b[pair_start[p]:pair_start[p + 1]]
        # pairs the device rejects (fewer than 5 rows, rows outside the table) fail there with their message
        if len(a) >= 5 and a.min() >= 0 and b.min() >= 0 and max(a.max(), b.max()) < len(bearings):
            plane[p] = plane_motion(bearings[a], bearings[b], threshold)
    R = len(row_a)
    lo = np.zeros((P, 3, 4))
    ransac = np.zeros(P, dtype=np.int32)
    pose = np.zeros((P, 2, 3, 4))
    counts = np.zeros((P, 3), dtype=np.int32)
    chosen = np.zeros(P, dtype=np.int32)
    m5 = np.zeros(R, dtype=np.uint8)
    mp = np.zeros(R, dtype=np.uint8)
    with _lib.pooled("relpose", device) as h:
        _lib.check(h.L.osfm_relpose_two_view(
            h.h, len(bearings), ptr(bearings), P, ptr(pair_start), ptr(row_a), ptr(row_b), float(threshold),
            ITERATIONS, int(iterations), int(bool(check_reversal)), float(reversal_ratio), ptr(plane), ptr(lo),
            ptr(ransac), ptr(pose), ptr(counts), ptr(chosen), ptr(m5), ptr(mp)))
        a_ms, b_ms, total = ctypes.c_float(0), ctypes.c_float(0), ctypes.c_float(0)
        _lib.check(h.L.osfm_relpose_last_stage_ms(h.h, ctypes.byref(a_ms), ctypes.byref(b_ms)))
        _lib.check(h.L.osfm_relpose_last_device_ms(h.h, ctypes.byref(total)))
    _last_device_ms = float(total.value)
    _last_stage_ms = (float(a_ms.value), float(b_ms.value))
    return TwoViewResult(lo, ransac, pose, counts, chosen, m5.view(bool), mp.view(bool), plane, pair_start,
                         _last_stage_ms[0], _last_stage_ms[1])


def two_view_lists(b1_list: Sequence[np.ndarray], b2_list: Sequence[np.ndarray], threshold: float,
                   iterations: int = REFINE_ITERATIONS, check_reversal: bool = False, reversal_ratio: float = 1.0,
                   device: int = 0) -> TwoViewResult:
    return two_view_pairs(*pack_lists(b1_list, b2_list), threshold, iterations, check_reversal, reversal_ratio, device)


def last_stage_ms():
    """(RANSAC kernels, two-view kernel or match filter) device time of the last two_view_pairs / two_view_lists /
    robust_match_pairs / robust_match_lists call."""
    return _last_stage_ms


# ---------------------------------------------------------------------------------------------------------------
# robust_match_calibrated after the RANSAC: bearing inliers at 4, 2 and 1 times the threshold, each refined
# ---------------------------------------------------------------------------------------------------------------
MATCH_REFINE_ITERATIONS = 10   # five_point_refine_match_iterations
MATCH_MIN_INLIERS = 8          # a relax round with fewer inliers empties the pair


@dataclass
class RobustMatchResult:
    lo_model: np.ndarray          # (P, 3, 4) as PairsResult.lo_model
    ransac_inliers: np.ndarray    # (P,) int32
    pose: np.ndarray              # (P, 3, 4): the refined [R | t], second image to first; NaN for an empty pair
    counts: np.ndarray            # (P, 4) int32: inliers of the 4x, 2x and 1x rounds, then of the final pass; -1: not run
    inlier_mask: np.ndarray       # (R,) bool: the final inliers
    pair_start: np.ndarray
    ransac_ms: float
    filter_ms: float

    def mask(self, p: int) -> np.ndarray:
        """Final inlier mask of pair p's rows (all False when the pair ended empty)."""
        return self.inlier_mask[self.pair_start[p]:self.pair_start[p + 1]]

    def empty_round(self, p: int) -> Optional[int]:
        """The relax round (0: 4x, 1: 2x, 2: 1x) whose fewer than 8 inliers emptied pair p, None if none did."""
        low = np.flatnonzero((self.counts[p, :3] >= 0) & (self.counts[p, :3] < MATCH_MIN_INLIERS))
        return int(low[0]) if len(low) else None


def robust_match_pairs(bearings: np.ndarray, pair_start: np.ndarray, row_a: np.ndarray, row_b: np.ndarray,
                       threshold: float, ransac_iterations: int = ITERATIONS,
                       refine_iterations: int = MATCH_REFINE_ITERATIONS, device: int = 0) -> RobustMatchResult:
    """robust_match_calibrated's verification of every pair (rows index one bearing table, as ransac_pairs), RANSAC
    and the relax rounds in one device call: `threshold` (robust_matching_calib_threshold) is RANSAC's angle and the
    rounds' chord bound.  Every pair needs at least 8 rows."""
    global _last_device_ms, _last_stage_ms
    bearings = np.ascontiguousarray(bearings, dtype=np.float64).reshape(-1, 3)
    pair_start, row_a, row_b = batch_rows(pair_start, row_a, row_b)
    P = len(pair_start) - 1
    lo = np.zeros((P, 3, 4))
    ransac = np.zeros(P, dtype=np.int32)
    pose = np.zeros((P, 3, 4))
    counts = np.zeros((P, 4), dtype=np.int32)
    mask = np.zeros(len(row_a), dtype=np.uint8)
    with _lib.pooled("relpose", device) as h:
        _lib.check(h.L.osfm_relpose_robust_match(
            h.h, len(bearings), ptr(bearings), P, ptr(pair_start), ptr(row_a), ptr(row_b), float(threshold),
            int(ransac_iterations), int(refine_iterations), ptr(lo), ptr(ransac), ptr(pose), ptr(counts), ptr(mask)))
        a_ms, b_ms, total = ctypes.c_float(0), ctypes.c_float(0), ctypes.c_float(0)
        _lib.check(h.L.osfm_relpose_last_stage_ms(h.h, ctypes.byref(a_ms), ctypes.byref(b_ms)))
        _lib.check(h.L.osfm_relpose_last_device_ms(h.h, ctypes.byref(total)))
    _last_device_ms = float(total.value)
    _last_stage_ms = (float(a_ms.value), float(b_ms.value))
    return RobustMatchResult(lo, ransac, pose, counts, mask.view(bool), pair_start, *_last_stage_ms)


def robust_match_lists(b1_list: Sequence[np.ndarray], b2_list: Sequence[np.ndarray], threshold: float,
                       ransac_iterations: int = ITERATIONS, refine_iterations: int = MATCH_REFINE_ITERATIONS,
                       device: int = 0) -> RobustMatchResult:
    return robust_match_pairs(*pack_lists(b1_list, b2_list), threshold, ransac_iterations, refine_iterations, device)
