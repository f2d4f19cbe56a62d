"""numpy restatement of the reference's VLAD pair selection -- test infrastructure only.

    compute_vlad_descriptor   features::compute_vlad_descriptor  (opensfm/src/features/src/matching.cc:90-119)
    signed_square_root_normalize                                  (opensfm/vlad.py)
    compute_vlad_distances    features::compute_vlad_distances   (matching.cc:121-145)
    construct_pairs / pairs_from_neighbors                        (opensfm/pairs_selection.py:471-490, 764-795)

compute_vlad_descriptor is bit for bit: numpy's float32 element-wise subtract, multiply and add are each correctly
rounded with no FMA, a loop over the dimensions reproduces the reference's sequential squared-norm chain, and
np.cumsum in float32 adds the residuals of a centre in feature order.
"""
from __future__ import annotations

from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

FLT_MAX = np.float32(np.finfo(np.float32).max)


def nearest_centers(features: np.ndarray, centers: np.ndarray) -> np.ndarray:
    """The centre each feature is assigned to: the first centre whose squared distance
    s = (f0 - c0)^2, s += (fk - ck)^2 (float32, k ascending) is smallest and below FLT_MAX."""
    F = np.asarray(features, dtype=np.float32)
    C = np.asarray(centers, dtype=np.float32)
    if len(F) == 0:
        return np.zeros(0, dtype=np.int64)
    d = F[:, None, 0] - C[None, :, 0]
    s = d * d
    for k in range(1, F.shape[1]):
        d = F[:, None, k] - C[None, :, k]
        s = s + d * d
    best = np.argmin(s, axis=1)   # first of equal minima = the strict `<` scan in centre order
    if not np.all(s[np.arange(len(F)), best] < FLT_MAX):
        raise ValueError("no centre below FLT_MAX: the reference's behaviour is undefined there")
    return best


def compute_vlad_descriptor(features: np.ndarray, centers: np.ndarray) -> np.ndarray:
    """Sum of the float32 residuals f - c of the features of every centre, in feature order (nc * dim float32)."""
    F = np.asarray(features, dtype=np.float32)
    C = np.asarray(centers, dtype=np.float32)
    if C.shape[0] == 0 or C.shape[1] == 0:
        raise ValueError("Zero VLAD centers or zero length VLAD words.")
    v = np.zeros(C.shape, dtype=np.float32)
    best = nearest_centers(F, C)
    for c in np.unique(best):
        r = F[best == c] - C[c]
        v[c] = np.cumsum(r, axis=0, dtype=np.float32)[-1]
    return v.reshape(-1)


def unnormalized_vlad(features: np.ndarray, centers: np.ndarray) -> Optional[np.ndarray]:
    """vlad.unnormalized_vlad: None when the dimension or the dtype differs."""
    if centers.shape[1] != features.shape[1] or centers.dtype != features.dtype:
        return None
    return compute_vlad_descriptor(features, centers)


def signed_square_root_normalize(v: np.ndarray, fp64_sum: bool = False) -> np.ndarray:
    """vlad.signed_square_root_normalize.  The reference's float32 np.linalg.norm sums through BLAS in a
    host-dependent order; fp64_sum=True takes the sum of squares in fp64 rounded to float32 instead (then the
    float32 square root), which is what the engine does."""
    v = np.sign(v) * np.sqrt(np.abs(v))
    if fp64_sum and v.dtype == np.float32:
        n = np.sqrt(np.float32(np.sum(v.astype(np.float64) ** 2)))
    else:
        n = np.linalg.norm(v)
    with np.errstate(invalid="ignore", divide="ignore"):
        v /= n
    return v


def vlad_distance(a: np.ndarray, b: np.ndarray, fp64: bool = True) -> float:
    """|a - b|: in fp64 from the float32 values (the engine), or the reference's float32 norm of the float32
    difference (fp64=False)."""
    if fp64:
        return float(np.sqrt(np.sum((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2)))
    return float(np.linalg.norm(np.asarray(a, np.float32) - np.asarray(b, np.float32)))


def compute_vlad_distances(histograms: Dict[Any, np.ndarray], image: Any, other_images: Iterable[Any],
                           distance=None) -> Tuple[List[float], List[Any]]:
    """(distances, others): the other images in sorted order (the reference iterates a std::set), the image itself
    and images without a histogram skipped.  distance(image, other) -> float defaults to vlad_distance."""
    if image not in histograms:
        return [], []
    if distance is None:
        def distance(a, b):
            return vlad_distance(histograms[a], histograms[b])
    others = [c for c in sorted(set(other_images)) if c != image and c in histograms]
    return [distance(image, c) for c in others], others


def sorted_pair(im1: Any, im2: Any) -> Tuple[Any, Any]:
    return (im1, im2) if im1 < im2 else (im2, im1)


def pairs_from_neighbors(image: Any, exifs: Dict[Any, Any], distances: Sequence[float], order: Sequence[int],
                         other: Sequence[Any], max_neighbors: int) -> Dict[Tuple[Any, Any], float]:
    """The max_neighbors nearest of the image's camera and the max_neighbors nearest of other cameras."""
    same_camera, other_cameras = [], []
    for i in order:
        im2 = other[i]
        if exifs[im2]["camera"] == exifs[image]["camera"]:
            if len(same_camera) < max_neighbors:
                same_camera.append((im2, distances[i]))
        elif len(other_cameras) < max_neighbors:
            other_cameras.append((im2, distances[i]))
        if len(same_camera) + len(other_cameras) >= 2 * max_neighbors:
            break
    return {sorted_pair(image, im2): d for im2, d in same_camera + other_cameras}


def construct_pairs(results: Sequence[Tuple[Any, Sequence[float], Sequence[Any]]], max_neighbors: int,
                    exifs: Dict[Any, Any], enforce_other_cameras: bool,
                    kind: str = "stable") -> Dict[Tuple[Any, Any], float]:
    """results: (image, distances, others) per reference image.  kind="stable" breaks ties by position (the
    engine's order); the reference's np.argsort default is the unstable quicksort."""
    pairs: Dict[Tuple[Any, Any], float] = {}
    for im, distances, other in results:
        order = np.argsort(np.asarray(distances, dtype=np.float64), kind=kind)
        if enforce_other_cameras:
            pairs.update(pairs_from_neighbors(im, exifs, distances, order, other, max_neighbors))
        else:
            for i in order[:max_neighbors]:
                pairs[sorted_pair(im, other[i])] = distances[i]
    return pairs


def match_candidates_with_vlad(histograms: Dict[Any, np.ndarray], images_ref: Sequence[Any],
                               images_cand: Sequence[Any], exifs: Dict[Any, Any], max_neighbors: int,
                               enforce_other_cameras: bool, candidates: Optional[Dict[Any, Sequence[Any]]] = None,
                               distance=None, kind: str = "stable") -> Dict[Tuple[Any, Any], float]:
    """pairs_selection.match_candidates_with_vlad over given histograms (preemption done by the caller)."""
    if max_neighbors <= 0:
        return {}
    if not candidates:
        candidates = {im: images_cand for im in images_ref}
    results = []
    for im, cands in candidates.items():
        d, o = compute_vlad_distances(histograms, im, cands, distance)
        results.append((im, d, o))
    return construct_pairs(results, max_neighbors, exifs, enforce_other_cameras, kind)
