"""Absolute-pose RANSAC of many shots at once on the GPU (opensfm_b200/csrc/resect.cu, C ABI osfm_resect_*): the
estimator `resect` runs on every candidate image of the incremental reconstruction.  The rules, and the deliberate
differences from pyrobust, are stated in oracle/absolute_pose_oracle.py.  There is no CPU path.

The input is one bearing table, one world-point table and, per row, the index of its bearing and of its point;
shots own consecutive rows (`shot_start`).  `ransac_lists` builds that from per-shot (bs, Xs) arrays, and
`absolute_pose_ransac` is the drop-in of `opensfm.multiview.absolute_pose_ransac` for one shot.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Sequence

import numpy as np

from . import _lib
from ._lib import ptr
from .ransac import Engine, batch_rows

ITERATIONS = 1000   # what resect passes

_last_device_ms = 0.0


@dataclass
class ShotsResult:
    lo_model: np.ndarray          # (S, 3, 4): pyrobust's result.lo_model, [R | t] world to camera
    ransac_inliers: np.ndarray    # (S,) int32
    chord_inliers: np.ndarray     # (S,) int32: resect's inlier count
    chord_mask: np.ndarray        # (R,) bool
    shot_start: np.ndarray        # (S + 1,) int64
    device_ms: float

    def poses(self) -> np.ndarray:
        """(S, 3, 4) [R_c2w | origin]: what multiview.absolute_pose_ransac returns."""
        R = self.lo_model[:, :, :3]
        t = self.lo_model[:, :, 3]
        Rt = R.transpose(0, 2, 1)
        return np.concatenate([Rt, -np.einsum("sij,sj->si", Rt, t)[:, :, None]], axis=2)

    def inliers(self, s: int) -> np.ndarray:
        """Chord inlier mask of shot s's rows."""
        return self.chord_mask[self.shot_start[s]:self.shot_start[s + 1]]


class Resection(Engine):
    """osfm_resect (ransac.Engine): the problems are shots."""

    kind = "resect"

    def run(self, bearings: np.ndarray, points: np.ndarray, shot_start: np.ndarray, row_bearing: np.ndarray,
            row_point: np.ndarray, threshold: float, iterations: int = ITERATIONS) -> ShotsResult:
        bearings = np.ascontiguousarray(bearings, dtype=np.float64).reshape(-1, 3)
        points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        shot_start, row_bearing, row_point = batch_rows(shot_start, row_bearing, row_point,
                                                        ("shot_start", "row_bearing", "row_point"))
        S = len(shot_start) - 1
        lo = np.zeros((S, 3, 4), dtype=np.float64)
        ransac = np.zeros(S, dtype=np.int32)
        chord = np.zeros(S, dtype=np.int32)
        mask = np.zeros(len(row_bearing), dtype=np.uint8)
        _lib.check(self.L.osfm_resect_run(self.h, len(bearings), ptr(bearings), len(points), ptr(points), S,
                                          ptr(shot_start), ptr(row_bearing), ptr(row_point), float(threshold),
                                          int(iterations), ptr(lo), ptr(ransac), ptr(chord), ptr(mask)))
        self._num_problems = S
        return ShotsResult(lo, ransac, chord, mask.view(bool), shot_start, self._device_ms())


def ransac_shots(bearings: np.ndarray, points: np.ndarray, shot_start: np.ndarray, row_bearing: np.ndarray,
                 row_point: np.ndarray, threshold: float, iterations: int = ITERATIONS, device: int = 0) -> ShotsResult:
    """Every shot's absolute-pose RANSAC and chord inliers; rows index one bearing and one point table."""
    global _last_device_ms
    with _lib.pooled("resect", device) as h:
        res = Resection(handle=h).run(bearings, points, shot_start, row_bearing, row_point, threshold, iterations)
    _last_device_ms = res.device_ms
    return res


def last_device_ms() -> float:
    """Device time of the last ransac_shots / ransac_lists call (and so of the resect* calls)."""
    return _last_device_ms


def pack_lists(bs_list: Sequence[np.ndarray], Xs_list: Sequence[np.ndarray]):
    """(bearing table, point table, shot_start, row_bearing, row_point) of per-shot arrays: row r of the tables is
    row r of the concatenated shots."""
    n = np.array([len(b) for b in bs_list], dtype=np.int64)
    if any(len(b) != len(X) for b, X in zip(bs_list, Xs_list)) or len(bs_list) != len(Xs_list):
        raise ValueError("every shot needs as many points as bearings")
    shot_start = np.zeros(len(n) + 1, dtype=np.int64)
    np.cumsum(n, out=shot_start[1:])
    if not len(n) or shot_start[-1] == 0:
        return np.zeros((0, 3)), np.zeros((0, 3)), shot_start, np.zeros(0, np.int64), np.zeros(0, np.int64)
    bearings = np.concatenate([np.asarray(b, np.float64).reshape(-1, 3) for b in bs_list])
    points = np.concatenate([np.asarray(X, np.float64).reshape(-1, 3) for X in Xs_list])
    rows = np.arange(shot_start[-1], dtype=np.int64)
    return bearings, points, shot_start, rows, rows.copy()


def ransac_lists(bs_list: Sequence[np.ndarray], Xs_list: Sequence[np.ndarray], threshold: float,
                 iterations: int = ITERATIONS, device: int = 0) -> ShotsResult:
    return ransac_shots(*pack_lists(bs_list, Xs_list), threshold, iterations, device)


def absolute_pose_ransac(bs: np.ndarray, Xs: np.ndarray, threshold: float, iterations: int,
                         probability: float) -> np.ndarray:
    """multiview.absolute_pose_ransac: [R_c2w | origin] (3 x 4).  `probability` is accepted and, as in the reference,
    not used: pyrobust's stopping rule keeps its default of 0.99."""
    return ransac_lists([bs], [Xs], threshold, iterations).poses()[0]
