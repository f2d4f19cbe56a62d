"""Absolute-pose RANSAC of many shots at once on the GPU (opensfm_b200/csrc/resect.cu, C ABI osfm_resect_*): the
estimator `resect` runs on every candidate image of the incremental reconstruction.  The rules, and the deliberate
differences from pyrobust, are stated in oracle/absolute_pose_oracle.py.  There is no CPU path.

The input is one bearing table, one world-point table and, per row, the index of its bearing and of its point;
shots own consecutive rows (`shot_start`).  `ransac_lists` builds that from per-shot (bs, Xs) arrays, and
`absolute_pose_ransac` is the drop-in of `opensfm.multiview.absolute_pose_ransac` for one shot.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import ptr

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


class Resection:
    """osfm_resect: one stream, its workspaces and the sample stream kept on the device; a new handle, or `handle`
    when given."""

    def __init__(self, device: int = 0, handle: Optional[_lib.Handle] = None):
        self.handle = handle if handle is not None else _lib.Handle("resect", device)
        self.h, self.L, self.device = self.handle.h, self.handle.L, self.handle.device
        self._trace_cap = 0
        self._num_shots = 0

    def set_stream_prefix(self, length: int) -> None:
        """How many generator outputs the device keeps (a test hook: shots that use them all continue from the saved
        generator state)."""
        _lib.check(self.L.osfm_resect_set_stream_prefix(self.h, int(length)))

    def set_trace(self, capacity: int) -> None:
        """Record up to `capacity` drawn sample indices per shot in the following runs (0: off)."""
        _lib.check(self.L.osfm_resect_set_trace(self.h, int(capacity)))
        self._trace_cap = int(capacity)

    def trace(self):
        """(drawn indices per shot as a list of arrays, how many were drawn, generator outputs consumed per shot) of
        the last run."""
        S, cap = self._num_shots, self._trace_cap
        count = np.zeros(S, dtype=np.int32)
        used = np.zeros(S, dtype=np.int64)
        idx = np.zeros(S * cap, dtype=np.int32)
        _lib.check(self.L.osfm_resect_get_trace(self.h, ptr(count), ptr(used), ptr(idx)))
        idx = idx.reshape(S, cap)
        return [idx[s, :min(int(count[s]), cap)] for s in range(S)], count, used

    def run(self, bearings: np.ndarray, points: np.ndarray, shot_start: np.ndarray, row_bearing: np.ndarray,
            row_point: np.ndarray, threshold: float, iterations: int = ITERATIONS) -> ShotsResult:
        bearings = np.ascontiguousarray(bearings, dtype=np.float64).reshape(-1, 3)
        points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        shot_start = np.ascontiguousarray(shot_start, dtype=np.int64)
        row_bearing = np.ascontiguousarray(row_bearing, dtype=np.int64)
        row_point = np.ascontiguousarray(row_point, dtype=np.int64)
        S = len(shot_start) - 1
        if S < 0 or shot_start[-1] != len(row_bearing) or len(row_bearing) != len(row_point):
            raise ValueError("shot_start must end at the number of rows, and row_bearing / row_point must match in "
                             "length")
        lo = np.zeros((S, 3, 4), dtype=np.float64)
        ransac = np.zeros(S, dtype=np.int32)
        chord = np.zeros(S, dtype=np.int32)
        mask = np.zeros(len(row_bearing), dtype=np.uint8)
        _lib.check(self.L.osfm_resect_run(self.h, len(bearings), ptr(bearings), len(points), ptr(points), S,
                                          ptr(shot_start), ptr(row_bearing), ptr(row_point), float(threshold),
                                          int(iterations), ptr(lo), ptr(ransac), ptr(chord), ptr(mask)))
        self._num_shots = S
        ms = ctypes.c_float(0)
        _lib.check(self.L.osfm_resect_last_device_ms(self.h, ctypes.byref(ms)))
        return ShotsResult(lo, ransac, chord, mask.view(bool), shot_start, float(ms.value))


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
