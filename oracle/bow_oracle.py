"""numpy restatement of the reference's bag-of-words pair selection -- test infrastructure only.

    BagOfWords.weights / histogram / bow_distance           (opensfm/bow.py)
    bow_distances                                           (opensfm/pairs_selection.py:690-708)
    load_histograms (the more-than-8-words rule)            (pairs_selection.py:712-727)
    match_candidates_with_bow over given histograms         (pairs_selection.py:281-348, with vlad_oracle's
                                                             construct_pairs / pairs_from_neighbors)

plus `pairwise_sum`, numpy's summation order for a contiguous float64 array, restated so that the engine's
sums (the histogram's h.sum() and each distance's np.fabs(h - h2).sum()) can follow it operation by operation,
and `pairwise_leaves`, the same order as a list of leaves and a post-order combine program.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle.match_oracle import distance_matrix
from oracle.vlad_oracle import construct_pairs, sorted_pair  # noqa: F401  (re-exported for the tests)

MIN_NUM_FEATURE = 8      # load_histograms: an image needs more than this many words
PW_BLOCKSIZE = 128       # numpy's pairwise-summation leaf size


def pairwise_sum(a: np.ndarray) -> np.float64:
    """np.sum of a contiguous float64 vector, one correctly rounded float64 addition at a time:
    below 8 elements a plain chain from 0; up to 128 elements 8 stride-8 accumulators combined as
    ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the n % 8 tail one by one; above, the halves split at
    n2 = n/2 - (n/2) % 8, each summed the same way, then added."""
    a = np.asarray(a, dtype=np.float64)
    n = len(a)
    if n < 8:
        res = np.float64(0.0)
        for x in a:
            res = np.float64(res + x)
        return res
    if n <= PW_BLOCKSIZE:
        r = [np.float64(a[j]) for j in range(8)]
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] = np.float64(r[j] + a[i + j])
            i += 8
        res = np.float64(np.float64(np.float64(r[0] + r[1]) + np.float64(r[2] + r[3]))
                         + np.float64(np.float64(r[4] + r[5]) + np.float64(r[6] + r[7])))
        for x in a[i:]:
            res = np.float64(res + x)
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return np.float64(pairwise_sum(a[:n2]) + pairwise_sum(a[n2:]))


def pairwise_leaves(n: int) -> Tuple[List[Tuple[int, int]], List[int]]:
    """The order of pairwise_sum for length n as (leaves, program): leaves = [(start, length)] left to right;
    program = post-order ops, -1 = add the two values on top of the stack, i >= 0 = push leaf i's sum."""
    leaves: List[Tuple[int, int]] = []
    prog: List[int] = []

    def rec(start: int, m: int) -> None:
        if m <= PW_BLOCKSIZE:
            prog.append(len(leaves))
            leaves.append((start, m))
            return
        m2 = m // 2
        m2 -= m2 % 8
        rec(start, m2)
        rec(start + m2, m - m2)
        prog.append(-1)

    rec(0, n)
    return leaves, prog


def weights(frequencies: np.ndarray) -> np.ndarray:
    """BagOfWords.weights."""
    return np.log(frequencies.sum() / frequencies)


def histogram(words0: np.ndarray, w: np.ndarray) -> np.ndarray:
    """BagOfWords.histogram of the first words: bincount times the weights over its sum."""
    h = np.bincount(np.asarray(words0), minlength=len(w)) * w
    with np.errstate(invalid="ignore", divide="ignore"):
        return h / h.sum()


def knn_words(descriptors: np.ndarray, vocabulary: np.ndarray, k: int) -> np.ndarray:
    """map_to_words(..., "BRUTEFORCE"): the k nearest words by cv2's float32 distance, ties to the lower index
    (a stable argsort of the distances cv2 computes)."""
    d = distance_matrix(np.asarray(descriptors, np.float32), np.asarray(vocabulary, np.float32))
    return np.argsort(d, axis=1, kind="stable")[:, :min(k, len(vocabulary))].astype(np.int32)


def load_histograms(words: Dict[Any, np.ndarray], w: np.ndarray) -> Dict[Any, np.ndarray]:
    """load_histograms over given word matrices: images with 8 or fewer words are left out."""
    return {im: histogram(wd[:, 0], w) for im, wd in words.items() if len(wd) > MIN_NUM_FEATURE}


def bow_distances(image: Any, other_images: Sequence[Any], histograms: Dict[Any, np.ndarray]
                  ) -> Tuple[Any, List[float], List[Any]]:
    """pairs_selection.bow_distances: the candidates in the order given."""
    if image not in histograms:
        return image, [], []
    distances, other = [], []
    h = histograms[image]
    for im2 in other_images:
        if im2 != image and im2 in histograms:
            distances.append(np.fabs(h - histograms[im2]).sum())
            other.append(im2)
    return image, distances, other


def match_candidates_with_bow(histograms: Dict[Any, np.ndarray], images_ref: Sequence[Any],
                              images_cand: Sequence[Any], exifs: Dict[Any, Any], max_neighbors: int,
                              enforce_other_cameras: bool, candidates: Optional[Dict[Any, Sequence[Any]]] = None,
                              kind: str = "stable") -> Dict[Tuple[Any, Any], float]:
    """pairs_selection.match_candidates_with_bow over given histograms (preemption done by the caller):
    candidates=None is every reference against every candidate; an empty dict gives no pairs (no fallback)."""
    if max_neighbors <= 0:
        return {}
    if candidates is None:
        candidates = {im: images_cand for im in images_ref}
    results = [bow_distances(im, cands, histograms) for im, cands in candidates.items()]
    return construct_pairs(results, max_neighbors, exifs, enforce_other_cameras, kind)
