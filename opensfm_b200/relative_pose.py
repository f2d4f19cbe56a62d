"""Five-point relative-pose RANSAC of many image pairs at once on the GPU (opensfm_b200/csrc/relpose.cu, C ABI
osfm_relpose_*): the estimator `two_view_reconstruction_general` starts the two-view bootstrap with.  The rules, and
the deliberate differences from pyrobust, are stated in oracle/relative_pose_oracle.py.  There is no CPU path.

The input is one bearing table and, per row, the index of the first image's bearing and of the second image's;
pairs own consecutive rows (`pair_start`).  `ransac_lists` builds that from per-pair (b1, b2) arrays, and
`relative_pose_ransac` is the drop-in of `opensfm.multiview.relative_pose_ransac` for one pair.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import _lib
from ._lib import ptr

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


class RelativePose:
    """osfm_relpose: one stream, its workspaces and the sample stream kept on the device; a new handle, or `handle`
    when given."""

    def __init__(self, device: int = 0, handle: Optional[_lib.Handle] = None):
        self.handle = handle if handle is not None else _lib.Handle("relpose", device)
        self.h, self.L, self.device = self.handle.h, self.handle.L, self.handle.device
        self._trace_cap = 0
        self._num_pairs = 0

    def set_stream_prefix(self, length: int) -> None:
        """How many generator outputs the device keeps (a test hook: pairs that use them all continue from the saved
        generator state)."""
        _lib.check(self.L.osfm_relpose_set_stream_prefix(self.h, int(length)))

    def set_trace(self, capacity: int) -> None:
        """Record up to `capacity` drawn sample indices per pair in the following runs (0: off)."""
        _lib.check(self.L.osfm_relpose_set_trace(self.h, int(capacity)))
        self._trace_cap = int(capacity)

    def trace(self):
        """(drawn indices per pair as a list of arrays, how many were drawn, generator outputs consumed per pair) of
        the last run."""
        P, cap = self._num_pairs, self._trace_cap
        count = np.zeros(P, dtype=np.int32)
        used = np.zeros(P, dtype=np.int64)
        idx = np.zeros(P * cap, dtype=np.int32)
        _lib.check(self.L.osfm_relpose_get_trace(self.h, ptr(count), ptr(used), ptr(idx)))
        idx = idx.reshape(P, cap)
        return [idx[p, :min(int(count[p]), cap)] for p in range(P)], count, used

    def run(self, bearings: np.ndarray, pair_start: np.ndarray, row_a: np.ndarray, row_b: np.ndarray,
            threshold: float, iterations: int = ITERATIONS) -> PairsResult:
        bearings = np.ascontiguousarray(bearings, dtype=np.float64).reshape(-1, 3)
        pair_start = np.ascontiguousarray(pair_start, dtype=np.int64)
        row_a = np.ascontiguousarray(row_a, dtype=np.int64)
        row_b = np.ascontiguousarray(row_b, dtype=np.int64)
        P = len(pair_start) - 1
        if P < 0 or pair_start[-1] != len(row_a) or len(row_a) != len(row_b):
            raise ValueError("pair_start must end at the number of rows, and row_a / row_b must match in length")
        lo = np.zeros((P, 3, 4), dtype=np.float64)
        ransac = np.zeros(P, dtype=np.int32)
        mask = np.zeros(len(row_a), dtype=np.uint8)
        _lib.check(self.L.osfm_relpose_run(self.h, len(bearings), ptr(bearings), P, ptr(pair_start), ptr(row_a),
                                           ptr(row_b), float(threshold), int(iterations), ptr(lo), ptr(ransac),
                                           ptr(mask)))
        self._num_pairs = P
        ms = ctypes.c_float(0)
        _lib.check(self.L.osfm_relpose_last_device_ms(self.h, ctypes.byref(ms)))
        return PairsResult(lo, ransac, mask.view(bool), pair_start, float(ms.value))


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


def pack_lists(b1_list: Sequence[np.ndarray], b2_list: Sequence[np.ndarray]):
    """(bearing table, pair_start, row_a, row_b) of per-pair arrays: the first images' rows, then the second's."""
    if len(b1_list) != len(b2_list) or any(len(a) != len(b) for a, b in zip(b1_list, b2_list)):
        raise ValueError("every pair needs as many second bearings as first bearings")
    n = np.array([len(b) for b in b1_list], dtype=np.int64)
    pair_start = np.zeros(len(n) + 1, dtype=np.int64)
    np.cumsum(n, out=pair_start[1:])
    R = int(pair_start[-1])
    if R == 0:
        return np.zeros((0, 3)), pair_start, np.zeros(0, np.int64), np.zeros(0, np.int64)
    bearings = np.concatenate([np.asarray(b, np.float64).reshape(-1, 3) for b in b1_list] +
                              [np.asarray(b, np.float64).reshape(-1, 3) for b in b2_list])
    rows = np.arange(R, dtype=np.int64)
    return bearings, pair_start, rows, rows + R


def ransac_lists(b1_list: Sequence[np.ndarray], b2_list: Sequence[np.ndarray], threshold: float,
                 iterations: int = ITERATIONS, device: int = 0) -> PairsResult:
    return ransac_pairs(*pack_lists(b1_list, b2_list), threshold, iterations, device)


def relative_pose_ransac(b1: np.ndarray, b2: np.ndarray, threshold: float, iterations: int,
                         probability: float) -> np.ndarray:
    """multiview.relative_pose_ransac: [R^T | -R^T t] (3 x 4) of pyrobust's lo_model [R | t].  `probability` is
    accepted and, as in the reference, not used: pyrobust's stopping rule keeps its default of 0.99."""
    return ransac_lists([b1], [b2], threshold, iterations).poses()[0]
