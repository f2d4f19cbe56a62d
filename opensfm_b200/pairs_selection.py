"""VLAD and BoW pair selection on the GPU: the `opensfm.vlad` / `opensfm.pairs_selection` names this engine replaces.

    unnormalized_vlad(features, centers)                       opensfm/vlad.py
    PairMatcher.vlad_histograms(keys, centers)                 pairs_selection.py:732-745 (vlad_histograms)
    match_candidates_with_vlad(matcher, images_ref, ...)       pairs_selection.py:351-392, 471-490, 764-795
    PairMatcher.compute_words / bow_histograms(keys, bows)     features_processing.py:269-336, pairs_selection.py:712-727
    bow_distances(image, other_images, histograms)             pairs_selection.py:690-708
    match_candidates_with_bow(matcher, images_ref, ...)        pairs_selection.py:281-348, 471-490, 764-795

The VLAD descriptors are computed from the descriptor sets a `PairMatcher` already holds on the device and stay
there (likewise the BoW words and histograms); the all-pairs distances and the neighbour selection run on the device too, so only the selected pairs come
back.  The selected pairs go straight into `PairMatcher.match_pairs` on the same matcher.  GPS preemption
(`preempt_candidates`) needs the dataset's topocentric reference and stays with the caller.
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import ptr
from .matching import PairMatcher


def unnormalized_vlad(features: np.ndarray, centers: np.ndarray, device: int = 0) -> Optional[np.ndarray]:
    """vlad.unnormalized_vlad: the sum of residuals to the nearest centre (float32, len(centers) * dim), bit for bit
    features::compute_vlad_descriptor; None when the descriptor length or dtype differs from the centres'."""
    if centers.shape[1] != features.shape[1] or centers.dtype != features.dtype:
        return None
    f = np.ascontiguousarray(features, dtype=np.float32)
    c = np.ascontiguousarray(centers, dtype=np.float32)
    with _lib.pooled("matcher", device) as m:
        sid = ctypes.c_int()
        _lib.check(m.L.osfm_matcher_add_f32(m.h, ptr(f), f.shape[0], f.shape[1], ctypes.byref(sid)))
        try:
            ids = np.array([sid.value], dtype=np.int32)
            valid = np.zeros(1, dtype=np.int32)
            _lib.check(m.L.osfm_matcher_vlad_compute(m.h, 1, ptr(ids), ptr(c), c.shape[0], c.shape[1], ptr(valid)))
            out = np.empty(c.size, dtype=np.float32)
            _lib.check(m.L.osfm_matcher_vlad_get(m.h, sid.value, 1, ptr(out)))
        finally:
            _lib.check(m.L.osfm_matcher_remove(m.h, sid.value))
    return out


def sorted_pair(im1: Any, im2: Any) -> Tuple[Any, Any]:
    """pairs_selection.sorted_pair."""
    return (im1, im2) if im1 < im2 else (im2, im1)


def _state_check(state_of, kind: str, producer: str):
    """has(image): whether the image has a VLAD descriptor / BoW histogram; raises if `producer` never ran on it."""

    def has(im):
        state = state_of(im)
        if state is None:
            raise ValueError("image %r has no %s state: run PairMatcher.%s on it first" % (im, kind, producer))
        return state

    return has


def _selected_pairs(select, refs: Sequence[Any], cands: Sequence[Any], per_ref: Optional[np.ndarray],
                    exifs: Dict[Any, Any], max_neighbors: int,
                    enforce_other_cameras: bool) -> Dict[Tuple[Any, Any], float]:
    """{sorted pair: distance} of the candidates `select` (PairMatcher.vlad_select / bow_select) keeps for each
    reference, with camera labels from `exifs` when `enforce_other_cameras`."""
    if not refs or not cands:
        return {}
    labels = None
    if enforce_other_cameras:
        names: Dict[Any, int] = {}
        labels = np.array([names.setdefault(exifs[im]["camera"], len(names)) for im in list(refs) + cands], dtype=np.int32)
    pairs: Dict[Tuple[Any, Any], float] = {}
    for im, (cols, dist) in zip(refs, select(refs, cands, max_neighbors, per_ref, labels)):
        for j, d in zip(cols.tolist(), dist.tolist()):
            pairs[sorted_pair(im, cands[j])] = d
    return pairs


def match_candidates_with_vlad(matcher: PairMatcher, images_ref: Sequence[Any], images_cand: Sequence[Any],
                               exifs: Dict[Any, Any], max_neighbors: int, enforce_other_cameras: bool,
                               candidates: Optional[Dict[Any, Sequence[Any]]] = None) -> Dict[Tuple[Any, Any], float]:
    """pairs_selection.match_candidates_with_vlad: {sorted pair: VLAD distance} of every reference image with its
    `max_neighbors` nearest candidates (and as many of other cameras when `enforce_other_cameras`; cameras are
    `exifs[image]["camera"]`).

    `matcher` holds the images' descriptors and their VLAD descriptors (`PairMatcher.vlad_histograms` /
    `compute_vlad`); images whose VLAD could not be computed are skipped, as the reference drops them.
    `candidates`: {reference image: candidate images}, the first value `preempt_candidates` returns; None or empty
    means every reference image against every candidate image, the reference's fallback.

    Distances are fp64, sqrt(sum (double(a) - double(b))^2), where the reference takes a float32 norm; ties go to
    the candidate that comes first in sorted order, which is the order compute_vlad_distances lists them in."""
    if max_neighbors <= 0:
        return {}
    has = _state_check(matcher.has_vlad, "VLAD", "vlad_histograms")
    mask = None
    if not candidates:
        refs = [im for im in dict.fromkeys(images_ref) if has(im)]
        cands = sorted({c for c in images_cand if has(c)})
    else:
        refs = [im for im in candidates if has(im)]
        per_ref = [{c for c in candidates[im] if has(c)} for im in refs]
        cands = sorted(set().union(*per_ref)) if per_ref else []
        col = {c: j for j, c in enumerate(cands)}
        if any(len(s) != len(cands) for s in per_ref):
            mask = np.zeros((len(refs), len(cands)), dtype=bool)
            for r, s in enumerate(per_ref):
                mask[r, [col[c] for c in s]] = True
    return _selected_pairs(matcher.vlad_select, refs, cands, mask, exifs, max_neighbors, enforce_other_cameras)


def bow_distances(image: Any, other_images: Sequence[Any], histograms: Dict[Any, np.ndarray], device: int = 0):
    """pairs_selection.bow_distances: (image, distances, other images) with the candidates that have a histogram, in
    the order given, `image` itself skipped; each distance np.fabs(h - h2).sum() bit for bit."""
    from .bow import bow_distance_rows

    if image not in histograms:
        return image, [], []
    others = [o for o in other_images if o != image and o in histograms]
    if not others:
        return image, [], []
    d = bow_distance_rows(np.stack([histograms[image]] + [histograms[o] for o in others]), 0, device)
    return image, d[1:].tolist(), others


def match_candidates_with_bow(matcher: PairMatcher, images_ref: Sequence[Any], images_cand: Sequence[Any],
                              exifs: Dict[Any, Any], max_neighbors: int, enforce_other_cameras: bool,
                              candidates: Optional[Dict[Any, Sequence[Any]]] = None) -> Dict[Tuple[Any, Any], float]:
    """pairs_selection.match_candidates_with_bow: {sorted pair: BoW distance} of every reference image with its
    `max_neighbors` nearest candidates (and as many of other cameras when `enforce_other_cameras`; cameras are
    `exifs[image]["camera"]`).

    `matcher` holds the images' descriptors and their BoW histograms (`PairMatcher.compute_words`, then
    `bow_histograms`); images without a histogram (8 or fewer words) are skipped, as the reference skips them.
    `candidates`: {reference image: candidate images}, the first value `preempt_candidates` returns.  None means
    every reference image against every candidate image; an empty dict gives no pairs, as the reference has no
    fallback there.

    Distances are the reference's np.fabs(h - h2).sum(), bit for bit.  Each reference's candidates keep the order
    given, and a tie goes to the earlier candidate (the reference's unstable np.argsort leaves it open); a candidate
    listed twice for one reference counts once."""
    if max_neighbors <= 0:
        return {}
    has = _state_check(matcher.has_bow, "BoW", "bow_histograms")
    order = None
    if candidates is None:
        refs = [im for im in dict.fromkeys(images_ref) if has(im)]
        cands = [c for c in dict.fromkeys(images_cand) if has(c)]
    else:
        refs = [im for im in candidates if has(im)]
        lists = [[c for c in dict.fromkeys(candidates[im]) if has(c)] for im in refs]
        cands = list(dict.fromkeys(c for lst in lists for c in lst))
        col = {c: j for j, c in enumerate(cands)}
        order = np.full((len(refs), len(cands)), -1, dtype=np.int32)
        for r, lst in enumerate(lists):
            order[r, [col[c] for c in lst]] = np.arange(len(lst), dtype=np.int32)
    return _selected_pairs(matcher.bow_select, refs, cands, order, exifs, max_neighbors, enforce_other_cameras)
