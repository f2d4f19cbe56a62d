"""The geometric verification of calibrated image pairs, `matching.robust_match_calibrated` after the descriptor
matches, in numpy, one pair at a time: the restatement that rp_match_filter (opensfm_b200/csrc/relpose.cu,
osfm_relpose_robust_match) is checked against.

What it restates (opensfm/matching.py:871-903, multiview.py:494-517, 541-553):

  * RANSAC: multiview.relative_pose_ransac(b1, b2, threshold, 1000, 0.999), that is pyrobust's five-point RANSAC
    with `threshold` as an angle (oracle/relative_pose_oracle.py's `ransac_relative_pose`), and its pose
    T = [R^T | -R^T t] of lo_model = [R | t];
  * for relax in 4, 2, 1: the bearing inliers of T with the chord bound relax * threshold
    (compute_inliers_bearings, oracle/two_view_oracle.py's `bearing_inliers`); fewer than 8 empty the pair;
    otherwise T becomes relative_pose_optimize_nonlinear of T on those inliers (RelativePoseRefinement with
    TinySolver, max_num_iterations = five_point_refine_match_iterations: two_view_oracle's `refine`);
  * the result is the bearing inliers of the last T at threshold.

`robust_match` starts from a given lo_model, as two_view_oracle.two_view does, so that a test can compare the stage
after RANSAC on the engine's own RANSAC result; `robust_match_calibrated` runs the oracle's RANSAC first.

Deliberate differences from the reference, those of two_view_oracle: the bearings are normalised once, before
RANSAC, and the rows come in the caller's order (the reference's come in its match list's order, which the caller
keeps).  The rounding-level differences of the refinement are stated there.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from oracle.relative_pose_oracle import normalize_rows, ransac_relative_pose
from oracle.two_view_oracle import Margins, bearing_inliers, refine

RELAX = (4, 2, 1)
MIN_INLIERS = 8
RANSAC_ITERATIONS = 1000
REFINE_ITERATIONS = 10       # five_point_refine_match_iterations


@dataclass
class RobustMatch:
    pose: np.ndarray              # 3 x 4: the last T, NaN when the pair ended empty
    counts: List[int]             # inliers of the 4x, 2x and 1x rounds, then of the final pass; -1: not run
    mask: np.ndarray              # bool per row: the final inliers (none when empty)
    empty_round: Optional[int]    # the round whose fewer than 8 inliers emptied the pair, None if none did
    margins: Margins = field(default_factory=Margins)


def robust_match(b1: np.ndarray, b2: np.ndarray, lo_model: np.ndarray, threshold: float,
                 iterations: int = REFINE_ITERATIONS) -> RobustMatch:
    """The relax rounds and the final inliers of one pair from RANSAC's lo_model [R_l | t_l]."""
    x, y = normalize_rows(b1), normalize_rows(b2)
    mg = Margins()
    Rl, tl = lo_model[:, :3], lo_model[:, 3]
    T = np.column_stack([Rl.T, -(Rl.T @ tl)])
    counts = [-1] * (len(RELAX) + 1)
    for r, relax in enumerate(RELAX):
        inliers = np.nonzero(bearing_inliers(T, x, y, relax * threshold, mg))[0]
        counts[r] = len(inliers)
        if len(inliers) < MIN_INLIERS:
            return RobustMatch(np.full((3, 4), np.nan), counts, np.zeros(len(x), bool), r, mg)
        T = refine(T, x, y, inliers, iterations)
    mask = bearing_inliers(T, x, y, threshold, mg)
    counts[-1] = int(mask.sum())
    return RobustMatch(T, counts, mask, None, mg)


def robust_match_calibrated(b1: np.ndarray, b2: np.ndarray, threshold: float,
                            ransac_iterations: int = RANSAC_ITERATIONS,
                            refine_iterations: int = REFINE_ITERATIONS) -> RobustMatch:
    """RANSAC, then `robust_match`; the caller handles pairs of fewer than 8 rows (the reference returns no matches
    for them before any estimation)."""
    if len(b1) < MIN_INLIERS:
        raise ValueError("robust_match_calibrated needs at least 8 rows, got %d" % len(b1))
    lo = ransac_relative_pose(b1, b2, threshold, ransac_iterations).lo_model
    return robust_match(b1, b2, lo, threshold, refine_iterations)
