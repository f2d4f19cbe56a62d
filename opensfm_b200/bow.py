"""Bag of visual words on the GPU: the `opensfm.bow` names this engine replaces.

    BagOfWords(words, frequencies)                  opensfm/bow.py
      .weights                                      log(frequencies.sum() / frequencies), as the reference
      .map_to_words(descriptors, k, matcher_type)   the k nearest vocabulary words of every descriptor
      .histogram(words) / .bow_distance(...)        bit for bit the reference's float64 arithmetic

Word assignment is exact for every matcher type: the indices cv2 BruteForce knnMatch returns, in its order.  The
reference's default FLANN index is approximate, so FLANN configurations get the exact words here, not FLANN's.
For descriptors already resident in a `matching.PairMatcher`, `PairMatcher.compute_words` / `bow_histograms`
do the same without uploading them again.  All arithmetic runs in the CUDA library (csrc/bow.cu); there is no CPU
path here.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import numpy as np

from . import _lib


class BagOfWords:
    def __init__(self, words: np.ndarray, frequencies: np.ndarray, device: int = 0) -> None:
        self.words = words
        self.frequencies = frequencies
        self.weights = np.log(frequencies.sum() / frequencies)
        self.words32 = np.ascontiguousarray(words, dtype=np.float32)
        if self.words32.ndim != 2:
            raise ValueError("words must be nwords x dim")
        self.device = device

    def map_to_words(self, descriptors: np.ndarray, k: int, matcher_type: str = "FLANN") -> np.ndarray:
        """int32 n x min(k, nwords): the k nearest words of every descriptor, nearest first, ties to the lower word
        (cv2 BruteForce knnMatch).  Exact for every `matcher_type`."""
        d = np.ascontiguousarray(descriptors, dtype=np.float32)
        if d.ndim != 2 or d.shape[1] != self.words32.shape[1]:
            raise ValueError("descriptors must be n x %d" % self.words32.shape[1])
        out = np.empty((d.shape[0], min(int(k), len(self.words32))), dtype=np.int32)
        with _lib.pooled("matcher", self.device) as m:
            _lib.check(m.L.osfm_bow_map_to_words(m.h, d.ctypes.data_as(ctypes.c_void_p), d.shape[0], d.shape[1],
                                                 self.words32.ctypes.data_as(ctypes.c_void_p), len(self.words32),
                                                 int(k), out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def histogram(self, words: np.ndarray) -> np.ndarray:
        """bincount(words, minlength=nwords) * weights / its sum, float64, bit for bit the reference (0/0 -> NaN)."""
        w = np.ascontiguousarray(words, dtype=np.int32).reshape(-1)
        if len(w) and (w.min() < 0 or w.max() >= len(self.words32)):
            raise ValueError("word index out of range")
        wt = np.ascontiguousarray(self.weights, dtype=np.float64)
        out = np.empty(len(wt), dtype=np.float64)
        with _lib.pooled("matcher", self.device) as m:
            _lib.check(m.L.osfm_bow_histogram(m.h, w.ctypes.data_as(ctypes.c_void_p), len(w),
                                              wt.ctypes.data_as(ctypes.c_void_p), len(wt),
                                              out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def bow_distance(self, w1: np.ndarray, w2: np.ndarray, h1: Optional[np.ndarray] = None,
                     h2: Optional[np.ndarray] = None) -> float:
        """np.fabs(h1 - h2).sum() in numpy's order, histograms computed from the words where not given."""
        if h1 is None:
            h1 = self.histogram(w1)
        if h2 is None:
            h2 = self.histogram(w2)
        return bow_distance_rows(np.stack([h1, h2]), 0, self.device)[1]


def bow_distance_rows(hist: np.ndarray, query: int, device: int = 0) -> np.ndarray:
    """np.fabs(hist[query] - hist[i]).sum() for every row i, on the device (osfm_bow_distances)."""
    h = np.ascontiguousarray(hist, dtype=np.float64)
    out = np.zeros(h.shape[0], dtype=np.float64)
    with _lib.pooled("matcher", device) as m:
        _lib.check(m.L.osfm_bow_distances(m.h, h.ctypes.data_as(ctypes.c_void_p), h.shape[0], h.shape[1], int(query),
                                          out.ctypes.data_as(ctypes.c_void_p)))
    return out
