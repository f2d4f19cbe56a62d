"""Rotation-only RANSAC of many image pairs at once on the GPU (opensfm_b200/csrc/rotransac.cu, C ABI
osfm_rotransac_*): the estimator `compute_image_pairs` runs on every pair to rank them for the reconstruction
bootstrap.  The rules, and the one deliberate difference from pyrobust, are stated in
oracle/rotation_ransac_oracle.py.  There is no CPU path.

The input is one fp64 bearing table and, per row, the bearing of the first and of the second image; pairs own
consecutive rows (`pair_start`).  `ransac_pairs_lists` builds that from per-pair (b1, b2) arrays
(`pack_lists`, the shared `ransac.pack_pairs`).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Sequence

import numpy as np

from . import _lib
from ._lib import ptr
from .ransac import Engine, batch_rows, pack_pairs

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


class RotationRansac(Engine):
    """osfm_rotransac (ransac.Engine): the problems are image pairs."""

    kind = "rotransac"

    def run(self, bearings: np.ndarray, pair_start: np.ndarray, row_a: np.ndarray, row_b: np.ndarray,
            threshold: float, iterations: int = ITERATIONS) -> PairsResult:
        bearings = np.ascontiguousarray(bearings, dtype=np.float64).reshape(-1, 3)
        pair_start, row_a, row_b = batch_rows(pair_start, row_a, row_b)
        P = len(pair_start) - 1
        R = len(row_a)
        lo = np.zeros((P, 3, 3), dtype=np.float64)
        ransac = np.zeros(P, dtype=np.int32)
        chord = np.zeros(P, dtype=np.int32)
        mask = np.zeros(R, dtype=np.uint8)
        _lib.check(self.L.osfm_rotransac_run(self.h, len(bearings), ptr(bearings), P, ptr(pair_start), ptr(row_a),
                                             ptr(row_b), float(threshold), int(iterations), ptr(lo), ptr(ransac),
                                             ptr(chord), ptr(mask)))
        self._num_problems = P
        return PairsResult(lo, ransac, chord, mask.view(bool), pair_start, self._device_ms())


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


pack_lists = pack_pairs   # (bearing table, pair_start, row_a, row_b) of per-pair (b1, b2) arrays


def ransac_pairs_lists(b1s: Sequence[np.ndarray], b2s: Sequence[np.ndarray], threshold: float,
                       iterations: int = ITERATIONS, device: int = 0) -> PairsResult:
    return ransac_pairs(*pack_lists(b1s, b2s), threshold, iterations, device)
