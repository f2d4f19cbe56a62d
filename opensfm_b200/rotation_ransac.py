"""Rotation-only RANSAC of many image pairs at once on the GPU (opensfm_b200/csrc/rotransac.cu, C ABI
osfm_rotransac_*): the estimator `compute_image_pairs` runs on every pair to rank them for the reconstruction
bootstrap.  The rules, and the one deliberate difference from pyrobust, are stated in
oracle/rotation_ransac_oracle.py.  There is no CPU path.

The input is one fp64 bearing table and, per row, the bearing of the first and of the second image; pairs own
consecutive rows (`pair_start`).  `ransac_pairs_lists` builds that from per-pair (b1, b2) arrays.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import ptr

ITERATIONS = 1000   # what two_view_reconstruction_rotation_only passes

_last_device_ms = 0.0


@dataclass
class PairsResult:
    lo_model: np.ndarray          # (P, 3, 3): pyrobust's result.lo_model; the rotation is its transpose
    ransac_inliers: np.ndarray    # (P,) int32
    chord_inliers: np.ndarray     # (P,) int32: _two_view_rotation_inliers
    chord_mask: np.ndarray        # (R,) bool
    pair_start: np.ndarray        # (P + 1,) int64
    device_ms: float

    def rotations(self) -> np.ndarray:
        return self.lo_model.transpose(0, 2, 1)

    def inliers(self, p: int) -> np.ndarray:
        """Chord inlier rows of pair p, ascending (what _two_view_rotation_inliers returns)."""
        return np.nonzero(self.chord_mask[self.pair_start[p]:self.pair_start[p + 1]])[0]

    def scores(self) -> List[int]:
        """pairwise_reconstructability of every pair."""
        return reconstructability(np.diff(self.pair_start), self.chord_inliers)


def reconstructability(common: np.ndarray, rotation_inliers: np.ndarray) -> List[int]:
    """pairwise_reconstructability (reconstruction.py:193-200) of every pair, as Python ints: the outliers if they are
    at least 30 % of the common tracks, else 0."""
    common = np.asarray(common, dtype=np.int64)
    outliers = common - np.asarray(rotation_inliers, dtype=np.int64)
    return np.where(outliers.astype(np.float64) / common >= 0.3, outliers, 0).tolist()


class RotationRansac:
    """osfm_rotransac: one stream, its workspaces and the sample stream kept on the device; a new handle, or `handle`
    when given."""

    def __init__(self, device: int = 0, handle: Optional[_lib.Handle] = None):
        self.handle = handle if handle is not None else _lib.Handle("rotransac", device)
        self.h, self.L, self.device = self.handle.h, self.handle.L, self.handle.device
        self._trace_cap = 0
        self._num_pairs = 0

    def set_stream_prefix(self, length: int) -> None:
        """How many generator outputs the device keeps (a test hook: pairs that use them all continue from the saved
        generator state)."""
        _lib.check(self.L.osfm_rotransac_set_stream_prefix(self.h, int(length)))

    def set_trace(self, capacity: int) -> None:
        """Record up to `capacity` drawn sample indices per pair in the following runs (0: off)."""
        _lib.check(self.L.osfm_rotransac_set_trace(self.h, int(capacity)))
        self._trace_cap = int(capacity)

    def trace(self):
        """(drawn indices per pair as a list of arrays, generator outputs consumed per pair) of the last run."""
        P, cap = self._num_pairs, self._trace_cap
        count = np.zeros(P, dtype=np.int32)
        used = np.zeros(P, dtype=np.int64)
        idx = np.zeros(P * cap, dtype=np.int32)
        _lib.check(self.L.osfm_rotransac_get_trace(self.h, ptr(count), ptr(used), ptr(idx)))
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
        R = len(row_a)
        lo = np.zeros((max(P, 0), 3, 3), dtype=np.float64)
        ransac = np.zeros(P, dtype=np.int32)
        chord = np.zeros(P, dtype=np.int32)
        mask = np.zeros(R, dtype=np.uint8)
        _lib.check(self.L.osfm_rotransac_run(self.h, len(bearings), ptr(bearings), P, ptr(pair_start), ptr(row_a),
                                             ptr(row_b), float(threshold), int(iterations), ptr(lo), ptr(ransac),
                                             ptr(chord), ptr(mask)))
        self._num_pairs = P
        ms = ctypes.c_float(0)
        _lib.check(self.L.osfm_rotransac_last_device_ms(self.h, ctypes.byref(ms)))
        return PairsResult(lo, ransac, chord, mask.view(bool), pair_start, float(ms.value))


def ransac_pairs(bearings: np.ndarray, pair_start: np.ndarray, row_a: np.ndarray, row_b: np.ndarray,
                 threshold: float, iterations: int = ITERATIONS, device: int = 0) -> PairsResult:
    """Every pair's rotation-only RANSAC and chord inliers; rows index one bearing table."""
    global _last_device_ms
    with _lib.pooled("rotransac", device) as h:
        res = RotationRansac(handle=h).run(bearings, pair_start, row_a, row_b, threshold, iterations)
    _last_device_ms = res.device_ms
    return res


def last_device_ms() -> float:
    """Device time of the last ransac_pairs / ransac_pairs_lists call (and so of the compute_image_pairs* calls)."""
    return _last_device_ms


def pack_lists(b1s: Sequence[np.ndarray], b2s: Sequence[np.ndarray]):
    """(bearing table, pair_start, row_a, row_b) of per-pair bearing arrays: pair p's b1 rows, then its b2 rows."""
    n = np.array([len(b) for b in b1s], dtype=np.int64)
    if any(len(a) != len(b) for a, b in zip(b1s, b2s)):
        raise ValueError("every pair needs as many bearings in its second image as in its first")
    pair_start = np.zeros(len(n) + 1, dtype=np.int64)
    np.cumsum(n, out=pair_start[1:])
    if len(n) == 0:
        return np.zeros((0, 3)), pair_start, np.zeros(0, np.int64), np.zeros(0, np.int64)
    table = np.concatenate([np.concatenate([np.asarray(a, np.float64).reshape(-1, 3), np.asarray(b, np.float64).reshape(-1, 3)])
                            for a, b in zip(b1s, b2s)])
    local = np.arange(pair_start[-1], dtype=np.int64) - np.repeat(pair_start[:-1], n)
    row_a = np.repeat(2 * pair_start[:-1], n) + local
    row_b = row_a + np.repeat(n, n)
    return table, pair_start, row_a, row_b


def ransac_pairs_lists(b1s: Sequence[np.ndarray], b2s: Sequence[np.ndarray], threshold: float,
                       iterations: int = ITERATIONS, device: int = 0) -> PairsResult:
    return ransac_pairs(*pack_lists(b1s, b2s), threshold, iterations, device)
