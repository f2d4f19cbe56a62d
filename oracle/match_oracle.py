"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product.

Two checkers for the brute-force matcher:

1. `match_brute_force` / `match_brute_force_symmetric`: the reference code path
   itself, restated line for line from opensfm/matching.py:723-777 around the
   live `cv2` (4.13.0 in this image; reference pins opencv-python>=4.8,
   pyproject.toml:31).  cv2 is importable here and on the GPU box, so this is
   the *real reference* for the matcher ("kind": "reference" in bench.py).

2. `knn2_numpy` / `match_brute_force_numpy`: a numpy restatement of what
   cv2.BFMatcher.knnMatch(k=2) computes (OpenCV is a third-party dependency not
   in the OpenSfM tree; algorithm restated from its published behaviour,
   modules/core/src/batch_distance.cpp): for every query the two smallest
   `sqrt(float32 sum of squared differences)` (L2) or integer Hamming counts,
   ties resolved to the lowest train index (stable insertion with strict `<`),
   masked-out trains skipped, queries with fewer than two candidates dropped by
   matching.py:752.  It is pinned against cv2 in tests/test_match_oracle.py.

Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

import numpy as np


def match_brute_force(f1: np.ndarray, f2: np.ndarray, config: Dict[str, Any],
                      maskij: Optional[np.ndarray] = None) -> List[Tuple[int, int]]:
    """opensfm/matching.py:723-756 (cv2 knnMatch k=2 + Lowe ratio)."""
    import cv2

    assert f1.dtype.type == f2.dtype.type
    if f1.dtype.type == np.uint8:
        matcher_type = "BruteForce-Hamming"
    else:
        matcher_type = "BruteForce"
    matcher = cv2.DescriptorMatcher_create(matcher_type)
    matcher.add([f2])
    if maskij is not None:
        matches = matcher.knnMatch(f1, k=2, masks=np.array([maskij]).astype(np.uint8))
    else:
        matches = matcher.knnMatch(f1, k=2)
    ratio = config["lowes_ratio"]
    good_matches = []
    for match in matches:
        if match and len(match) == 2:
            m, n = match
            if m.distance < ratio * n.distance:
                good_matches.append(m)
    return [(mm.queryIdx, mm.trainIdx) for mm in good_matches]


def match_brute_force_symmetric(fi: np.ndarray, fj: np.ndarray, config: Dict[str, Any],
                                maskij: Optional[np.ndarray] = None) -> List[Tuple[int, int]]:
    """opensfm/matching.py:759-777."""
    matches_ij = [(a, b) for a, b in match_brute_force(fi, fj, config, maskij)]
    maskijT = maskij.T if maskij is not None else None
    matches_ji = [(b, a) for a, b in match_brute_force(fj, fi, config, maskijT)]
    return list(set(matches_ij).intersection(set(matches_ji)))


def l2sqr_cv_order(f1: np.ndarray, f2: np.ndarray) -> np.ndarray:
    """float32 sum of squared differences in the order cv2 computes it (OpenCV core `normL2Sqr_` for
    float, x86-64 baseline of the opencv-python wheels: 4-lane universal intrinsics, no FMA): four 4-lane
    accumulators acc[a][l] += t*t over 16-element blocks (element 16*blk + 4*a + l), combined
    ((acc0 + acc1) + acc2) + acc3 per lane, lanes reduced (v0 + v2) + (v1 + v3), then the dim % 16 tail
    added sequentially.  Pinned bit-for-bit against live cv2 in tests/test_match_oracle.py."""
    a = np.ascontiguousarray(f1, dtype=np.float32)
    b = np.ascontiguousarray(f2, dtype=np.float32)
    n, m, dim = a.shape[0], b.shape[0], a.shape[1]
    nblk = dim // 16
    out = np.zeros((n, m), dtype=np.float32)
    step = max(1, (1 << 24) // max(m * max(dim, 1), 1))
    for q0 in range(0, n, step):
        t = a[q0:q0 + step, None, :] - b[None, :, :]          # float32 subtraction
        sq = t * t                                            # float32 product (rounded before the add)
        acc = np.zeros((t.shape[0], m, 16), dtype=np.float32)
        for blk in range(nblk):
            acc = acc + sq[:, :, 16 * blk:16 * blk + 16]
        acc = acc.reshape(t.shape[0], m, 4, 4)                # [a][l]
        v = ((acc[:, :, 0] + acc[:, :, 1]) + acc[:, :, 2]) + acc[:, :, 3]
        d = (v[:, :, 0] + v[:, :, 2]) + (v[:, :, 1] + v[:, :, 3])
        for e in range(16 * nblk, dim):
            d = d + sq[:, :, e]
        out[q0:q0 + step] = d
    return out


def distance_matrix(f1: np.ndarray, f2: np.ndarray) -> np.ndarray:
    """float32 distances as cv2 returns them: sqrt of the float32 sum of squared differences in cv2's
    summation order, or Hamming bit counts."""
    if f1.dtype == np.uint8:
        x = np.bitwise_xor(f1[:, None, :], f2[None, :, :])
        return np.unpackbits(x, axis=2).sum(axis=2).astype(np.float32)
    return np.sqrt(l2sqr_cv_order(f1, f2))


def knn2_numpy(f1: np.ndarray, f2: np.ndarray, maskij: Optional[np.ndarray] = None):
    """(idx1, d1, idx2, d2) per query; idx -1 where fewer candidates exist."""
    d = distance_matrix(f1, f2).astype(np.float64)
    if maskij is not None:
        d = np.where(maskij.astype(bool), d, np.inf)
    n, m = d.shape
    order = np.argsort(d, axis=1, kind="stable")[:, :2]
    if m < 2:
        order = np.concatenate([order, np.zeros((n, 2 - m), dtype=order.dtype)], axis=1)
    rows = np.arange(n)
    d1 = d[rows, order[:, 0]] if m >= 1 else np.full(n, np.inf)
    d2 = d[rows, order[:, 1]] if m >= 2 else np.full(n, np.inf)
    i1 = np.where(np.isfinite(d1), order[:, 0], -1)
    i2 = np.where(np.isfinite(d2), order[:, 1], -1)
    return i1, d1, i2, d2


def match_brute_force_numpy(f1, f2, config, maskij=None) -> List[Tuple[int, int]]:
    i1, d1, i2, d2 = knn2_numpy(f1, f2, maskij)
    ratio = config["lowes_ratio"]
    # m.distance (float32 -> Python float) < ratio * n.distance, matching.py:754
    ok = (i1 >= 0) & (i2 >= 0) & (np.float32(d1).astype(np.float64) < ratio * np.float32(d2).astype(np.float64))
    return [(int(q), int(i1[q])) for q in np.nonzero(ok)[0]]


def match_brute_force_symmetric_numpy(fi, fj, config, maskij=None) -> List[Tuple[int, int]]:
    mij = set(match_brute_force_numpy(fi, fj, config, maskij))
    mji = set((b, a) for a, b in match_brute_force_numpy(fj, fi, config, None if maskij is None else maskij.T))
    return list(mij & mji)


def _eigen_normalized(v: np.ndarray) -> np.ndarray:
    """Eigen's `normalized()` row by row (Eigen/src/Core/Dot.h since 3.3): v / sqrt(squaredNorm) when the squared
    norm is positive, the vector unchanged (no division by zero) when it is 0."""
    z = np.einsum("...i,...i->...", v, v)[..., None]
    return np.where(z > 0.0, v / np.sqrt(np.where(z > 0.0, z, 1.0)), v)


def epipolar_sym(b1: np.ndarray, b2: np.ndarray, R: np.ndarray, t: np.ndarray) -> np.ndarray:
    """The n1 x n2 fp64 `symmetric_epi` of geometry::EpipolarAngleTwoBearingsMany
    (opensfm/src/geometry/src/triangulation.cc:195-219) on float32 bearings (matching.py:860-861):
    (|e1_i . R b2_j| + |b1_i . e2_j|) / 2 with e1_i = normalized(t^ x b1_i), e2_j = normalized(t^ x R b2_j),
    t^ = normalized(t).  A zero t or a bearing parallel to t gives zero vectors, as in Eigen."""
    b1 = np.asarray(b1).astype(np.float32).astype(np.float64)
    b2 = np.asarray(b2).astype(np.float32).astype(np.float64)
    R = np.asarray(R, dtype=np.float64).reshape(3, 3)
    tn = _eigen_normalized(np.asarray(t, dtype=np.float64).reshape(3))
    b2w = b2 @ R.T
    e1 = _eigen_normalized(np.cross(tn, b1))
    e2 = _eigen_normalized(np.cross(tn, b2w))
    return (np.abs(e1 @ b2w.T) + np.abs(b1 @ e2.T)) / 2.0


def epipolar_angles(b1: np.ndarray, b2: np.ndarray, R: np.ndarray, t: np.ndarray) -> np.ndarray:
    """EpipolarAngleTwoBearingsMany: pi/2 - acos(symmetric_epi), NaN where the fp64 value exceeds 1."""
    with np.errstate(invalid="ignore"):
        return np.pi / 2.0 - np.arccos(epipolar_sym(b1, b2, R, t))


def epipolar_mask(b1: np.ndarray, b2: np.ndarray, R: np.ndarray, t: np.ndarray, threshold: float) -> np.ndarray:
    """matching.compute_inliers_bearing_epipolar (opensfm/matching.py:847-868) around
    geometry::EpipolarAngleTwoBearingsMany (opensfm/src/geometry/src/triangulation.cc:195-219), restated in numpy
    fp64: bearings are cast to float32 first (matching.py:860-861), R = pose.get_R_cam_to_world(),
    t = pose.get_origin() of image 2 relative to image 1.  Returns the boolean n1 x n2 mask `angle < threshold`
    (false where the angle is NaN)."""
    with np.errstate(invalid="ignore"):
        return epipolar_angles(b1, b2, R, t) < threshold


def match_using_words(f1: np.ndarray, words1: np.ndarray, f2: np.ndarray, words2_first: np.ndarray, lowes_ratio: float,
                      max_checks: int) -> np.ndarray:
    """features::MatchUsingWords restated (opensfm/src/features/src/matching.cc:15-72): multimap word -> features of
    image 2 (equal words in insertion order), per feature of image 1 the walk over its words, float32 distances
    summed in dimension order (np.cumsum in float32 is sequential), strict `<` updates, the `checks >= max_checks`
    break after a word, and the float32 ratio test (a single candidate passes: second best = inf)."""
    f1 = np.asarray(f1, dtype=np.float32)
    f2 = np.asarray(f2, dtype=np.float32)
    words1 = np.asarray(words1).reshape(len(f1), -1)
    index2 = {}
    for i, w in enumerate(np.asarray(words2_first).ravel().tolist()):
        index2.setdefault(int(w), []).append(i)
    out = []
    ratio = np.float32(lowes_ratio)
    for i in range(len(f1)):
        best = second = np.float32(np.inf)
        best_match, checks = -1, 0
        for j in range(words1.shape[1]):
            for match in index2.get(int(words1[i, j]), []):
                t = f1[i] - f2[match]
                d = np.sqrt(np.cumsum(t * t, dtype=np.float32)[-1])
                if d < best:
                    second, best, best_match = best, d, match
                elif d < second:
                    second = d
                checks += 1
            if checks >= max_checks:
                break
        if best < np.float32(ratio * second):
            out.append((i, best_match))
    return np.array(out, dtype=np.int32).reshape(-1, 2)
