"""Drop-in brute-force matching: the `opensfm.matching` names this engine replaces.

    match_brute_force(f1, f2, config, maskij=None)            opensfm/matching.py:723-756
    match_brute_force_symmetric(fi, fj, config, maskij=None)  opensfm/matching.py:759-777
    match_images_with_pairs-style batch: `PairMatcher`        opensfm/matching.py:63-98
    robust_match, robust_match_calibrated                     opensfm/matching.py:871-929

Same argument meaning, same return types (lists of (queryIdx, trainIdx) tuples),
same dtype dispatch (uint8 -> Hamming, else L2, matching.py:738-742).  All
arithmetic happens in the CUDA library (opensfm_b200/csrc/match*.cu) through the
C ABI; there is no CPU path here.

Thread safety: the reference calls these from a joblib *threading* pool
(opensfm/context.py:59-64).  Each call takes a matcher (own CUDA stream) that no
other thread holds meanwhile from the library's handle pool; ctypes releases the
GIL for the duration of the call.
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import ptr


def _prep(f: np.ndarray) -> np.ndarray:
    if f.dtype.type == np.uint8:
        return np.ascontiguousarray(f)
    return np.ascontiguousarray(f, dtype=np.float32)


def _match_raw(f1: np.ndarray, f2: np.ndarray, ratio: float, maskij: Optional[np.ndarray], symmetric: bool,
               device: int = 0) -> np.ndarray:
    assert f1.dtype.type == f2.dtype.type  # matching.py:737
    if f1.ndim != 2 or f2.ndim != 2 or (f1.shape[0] and f2.shape[0] and f1.shape[1] != f2.shape[1]):
        raise ValueError("descriptor matrices must be 2-D with equal row length")
    a, b = _prep(f1), _prep(f2)
    n1, n2 = a.shape[0], b.shape[0]
    out = np.full(n1, -1, dtype=np.int32)
    if n1 == 0 or n2 == 0:
        return out
    dim = a.shape[1]
    mask = None
    mask_p = None
    if maskij is not None:
        mask = np.ascontiguousarray(np.asarray(maskij).astype(np.uint8))  # matching.py:745
        if mask.shape != (n1, n2):
            raise ValueError("maskij must be len(f1) x len(f2)")
        mask_p = mask.ctypes.data_as(ctypes.c_void_p)
    with _lib.pooled("matcher", device) as m:
        fn = m.L.osfm_bf_match_u8 if a.dtype == np.uint8 else m.L.osfm_bf_match_f32
        _lib.check(fn(m.h, a.ctypes.data_as(ctypes.c_void_p), n1, b.ctypes.data_as(ctypes.c_void_p), n2, dim,
                      float(ratio), mask_p, int(symmetric), out.ctypes.data_as(ctypes.c_void_p)))
    return out


def match_brute_force(f1: np.ndarray, f2: np.ndarray, config: Dict[str, Any],
                      maskij: Optional[np.ndarray] = None) -> List[Tuple[int, int]]:
    """Brute force matching and Lowe's ratio filtering (matching.py:723-756)."""
    idx = _match_raw(f1, f2, config["lowes_ratio"], maskij, False)
    q = np.nonzero(idx >= 0)[0]
    return [(int(i), int(idx[i])) for i in q]


def match_brute_force_symmetric(fi: np.ndarray, fj: np.ndarray, config: Dict[str, Any],
                                maskij: Optional[np.ndarray] = None) -> List[Tuple[int, int]]:
    """Match in both directions and keep consistent matches (matching.py:759-777).
    The reference returns `list(set & set)` (arbitrary order); this returns them sorted by i."""
    idx = _match_raw(fi, fj, config["lowes_ratio"], maskij, True)
    q = np.nonzero(idx >= 0)[0]
    return [(int(i), int(idx[i])) for i in q]


def split_match_lists(raw: np.ndarray, counts: np.ndarray) -> List[np.ndarray]:
    """raw = the concatenated per-query train indices (-1 = no match) of consecutive pairs with `counts[p]`
    queries each -> one int64 [K, 2] array of (query, train) per pair, in one vectorised pass (the
    reference builds the same list pair by pair, matching.py:744-756)."""
    npairs = len(counts)
    if npairs == 0:
        return []
    starts = np.concatenate([[0], np.cumsum(counts)])
    hit = np.flatnonzero(raw >= 0)
    pair_of = np.searchsorted(starts, hit, side="right") - 1
    both = np.empty((len(hit), 2), dtype=np.int64)
    both[:, 0] = hit - starts[pair_of]
    both[:, 1] = raw[hit]
    cuts = np.searchsorted(pair_of, np.arange(1, npairs))
    return np.split(both, cuts)


class PairMatcher:
    """Descriptors resident in HBM + a pair list matched in one submission.

    The batched form of the per-pair loop in `match_images_with_pairs`
    (matching.py:63-98): upload every image's descriptors once (`add`), then
    `match_pairs([(im1, im2), ...])` returns {(im1, im2): ndarray[K, 2]} like the
    reference's result dict.
    """

    def __init__(self, device: int = 0, kernel: int = 0):
        self._m = _lib.Handle("matcher", device)
        self._ids: Dict[Any, int] = {}
        self._n: Dict[Any, int] = {}
        self._keep: Dict[Any, np.ndarray] = {}
        self._rows: Optional[np.ndarray] = None
        self._pairs: List[Tuple[Any, Any]] = []
        self._vlad: Dict[Any, int] = {}   # image -> length of its resident VLAD descriptor (0: it has none)
        self._bow: Dict[Any, int] = {}    # image -> length of its resident BoW histogram (0: it has none)
        self._words: Dict[Any, int] = {}  # image -> vocabulary size of its resident first words (0: it has none)
        if kernel:
            _lib.check(self._m.L.osfm_matcher_set_kernel(self._m.h, int(kernel)))

    def add(self, key: Any, desc: np.ndarray, uint8_is_l2: bool = False) -> None:
        """uint8_is_l2: `desc` is the uint8 storage of an L2 descriptor (HAHOG / SIFT as saved by
        opensfm/features.py:526-534), not a binary descriptor: uploaded as bytes, matched exactly like its
        float32 form."""
        d = _prep(desc)
        out = ctypes.c_int()
        if d.dtype == np.uint8:
            fn = self._m.L.osfm_matcher_add_u8_l2 if uint8_is_l2 else self._m.L.osfm_matcher_add_u8
        else:
            fn = self._m.L.osfm_matcher_add_f32
        _lib.check(fn(self._m.h, d.ctypes.data_as(ctypes.c_void_p), d.shape[0], d.shape[1], ctypes.byref(out)))
        if key in self._ids:
            _lib.check(self._m.L.osfm_matcher_remove(self._m.h, self._ids[key]))
        self._ids[key] = out.value
        self._n[key] = d.shape[0]
        self._forget(key)

    def add_many(self, items: Sequence[Tuple[Any, np.ndarray]], uint8_is_l2: bool = False) -> None:
        """Upload many images' descriptors with a single host synchronisation (same dtype and
        descriptor length for all; anything else goes through `add`)."""
        prepped = [(k, _prep(d)) for k, d in items]
        if not prepped:
            return
        d0 = prepped[0][1]
        if any(d.dtype != d0.dtype or d.shape[1] != d0.shape[1] for _, d in prepped):
            for k, d in prepped:
                self.add(k, d, uint8_is_l2)
            return
        cnt = len(prepped)
        ptrs = (ctypes.c_void_p * cnt)(*[d.ctypes.data for _, d in prepped])
        ns = np.array([d.shape[0] for _, d in prepped], dtype=np.int32)
        ids = np.empty(cnt, dtype=np.int32)
        if d0.dtype == np.uint8:
            fn = self._m.L.osfm_matcher_add_batch_u8_l2 if uint8_is_l2 else self._m.L.osfm_matcher_add_batch_u8
        else:
            fn = self._m.L.osfm_matcher_add_batch_f32
        _lib.check(fn(self._m.h, cnt, ctypes.cast(ptrs, ctypes.c_void_p), ns.ctypes.data_as(ctypes.c_void_p), d0.shape[1],
                      ids.ctypes.data_as(ctypes.c_void_p)))
        for (k, d), i in zip(prepped, ids):
            if k in self._ids:
                _lib.check(self._m.L.osfm_matcher_remove(self._m.h, self._ids[k]))
            self._ids[k] = int(i)
            self._n[k] = d.shape[0]
            self._forget(k)

    def clear(self) -> None:
        """Drop every resident descriptor set (device memory stays with the matcher for reuse)."""
        _lib.check(self._m.L.osfm_matcher_clear(self._m.h))
        for d in (self._ids, self._n, self._vlad, self._bow, self._words):
            d.clear()

    def _forget(self, key: Any) -> None:
        """Drop the VLAD / BoW state of an image whose descriptor set was replaced or removed."""
        for state in (self._vlad, self._bow, self._words):
            state.pop(key, None)

    # -- VLAD (opensfm/vlad.py, pairs_selection.vlad_histograms) ---------------------------------------------------
    def compute_vlad(self, keys: Iterable[Any], centers: np.ndarray) -> List[Any]:
        """Compute the VLAD descriptor of every resident image in `keys` against the visual words `centers`
        (ncenters x dim) and keep it on the device.  Returns the keys that have one: Hamming images and images of
        another descriptor length have none, as `vlad.unnormalized_vlad` returns None for them."""
        keys = list(dict.fromkeys(keys))
        c = np.ascontiguousarray(centers, dtype=np.float32)
        if c.ndim != 2:
            raise ValueError("centers must be ncenters x dim")
        ids = np.array([self._ids[k] for k in keys], dtype=np.int32)
        valid = np.zeros(len(keys), dtype=np.int32)
        for k in keys:
            self._vlad.pop(k, None)
        _lib.check(self._m.L.osfm_matcher_vlad_compute(self._m.h, len(keys), ptr(ids), ptr(c), c.shape[0], c.shape[1],
                                                       ptr(valid)))
        for k, v in zip(keys, valid):
            self._vlad[k] = c.size if v else 0
        return [k for k, v in zip(keys, valid) if v]

    def vlad_descriptor(self, key: Any, normalized: bool = True) -> np.ndarray:
        """The resident VLAD descriptor of one image (float32, ncenters * dim): signed-square-root normalised, or the
        unnormalised sum of residuals.  Raises KeyError if the image has none."""
        if not self._vlad.get(key):
            raise KeyError("no VLAD descriptor for image %r" % (key,))
        out = np.empty(self._vlad[key], dtype=np.float32)
        _lib.check(self._m.L.osfm_matcher_vlad_get(self._m.h, self._ids[key], int(not normalized), ptr(out)))
        return out

    def has_vlad(self, key: Any) -> Optional[bool]:
        """None if `compute_vlad` never ran on the image, else whether it has a VLAD descriptor."""
        return None if key not in self._vlad else bool(self._vlad[key])

    def vlad_histograms(self, keys: Iterable[Any], centers: np.ndarray) -> Dict[Any, np.ndarray]:
        """pairs_selection.vlad_histograms (pairs_selection.py:732-745) for resident images: {key: normalised
        float32 VLAD vector}, images without a descriptor left out.  The descriptors stay on the device for
        `pairs_selection.match_candidates_with_vlad`."""
        return {k: self.vlad_descriptor(k) for k in self.compute_vlad(keys, centers)}

    def vlad_select(self, refs: Sequence[Any], cands: Sequence[Any], k: int, cand_mask: Optional[np.ndarray] = None,
                    labels: Optional[np.ndarray] = None) -> List[Tuple[np.ndarray, np.ndarray]]:
        """Per reference image, the columns of `cands` (and their distances) that osfm_matcher_vlad_select keeps:
        the k nearest by (distance, column), per camera group when `labels` (len(refs) + len(cands) ints) is given.
        cand_mask: None or a len(refs) x len(cands) boolean array of allowed candidates."""
        nref, ncand = len(refs), len(cands)
        bits = None
        if cand_mask is not None:
            m = np.asarray(cand_mask, dtype=bool).reshape(nref, ncand)
            packed = np.packbits(m, axis=1, bitorder="little")
            words = (ncand + 31) // 32
            padded = np.zeros((nref, 4 * words), dtype=np.uint8)
            padded[:, :packed.shape[1]] = packed
            bits = np.ascontiguousarray(padded).view("<u4")
        return self._select(self._m.L.osfm_matcher_vlad_select, refs, cands, k, bits, labels)

    def _select(self, fn, refs: Sequence[Any], cands: Sequence[Any], k: int, per_ref: Optional[np.ndarray],
                labels: Optional[np.ndarray]) -> List[Tuple[np.ndarray, np.ndarray]]:
        """Run a selection entry point, `fn` (osfm_matcher_vlad_select or osfm_matcher_bow_select), whose
        per-reference argument is `per_ref` (the VLAD mask bits or the BoW candidate order)."""
        nref, ncand = len(refs), len(cands)
        ri = np.array([self._ids[r] for r in refs], dtype=np.int32)
        ci = np.array([self._ids[c] for c in cands], dtype=np.int32)
        lab = None if labels is None else np.ascontiguousarray(labels, dtype=np.int32)
        if lab is not None and lab.shape != (nref + ncand,):
            raise ValueError("labels must hold len(refs) + len(cands) ints")
        cap = max(nref * min(k, ncand) * (2 if lab is not None else 1), 1)
        offs = np.zeros(nref + 1, dtype=np.int64)
        cols = np.empty(cap, dtype=np.int32)
        dist = np.empty(cap, dtype=np.float64)
        _lib.check(fn(self._m.h, nref, ptr(ri), ncand, ptr(ci), ptr(per_ref), ptr(lab), int(k), ptr(offs),
                      ptr(cols), ptr(dist)))
        return [(cols[offs[r]:offs[r + 1]], dist[offs[r]:offs[r + 1]]) for r in range(nref)]

    # -- BoW (opensfm/bow.py, pairs_selection.load_histograms) ----------------------------------------------------
    def compute_words(self, keys: Iterable[Any], bows: Any, k: int) -> Dict[Any, np.ndarray]:
        """bows.map_to_words(descriptors, k, "BRUTEFORCE") of every resident image in `keys`: {key: int32 n x min(k,
        nwords)}, the k nearest words of `bows` (a `opensfm_b200.bow.BagOfWords`) exactly as cv2 knnMatch ranks them.
        The first word of every feature stays on the device for `bow_histograms`.  Hamming images and images of
        another descriptor length are left out."""
        keys = list(dict.fromkeys(keys))
        vocab = bows.words32
        nw = vocab.shape[0]
        kout = min(int(k), nw)
        ids = np.array([self._ids[key] for key in keys], dtype=np.int32)
        valid = np.zeros(len(keys), dtype=np.int32)
        offs = np.zeros(len(keys) + 1, dtype=np.int64)
        words = np.empty((max(sum(self._n[key] for key in keys), 1), kout), dtype=np.int32)
        for key in keys:
            self._words.pop(key, None)
            self._bow.pop(key, None)
        _lib.check(self._m.L.osfm_matcher_bow_words(self._m.h, len(keys), ptr(ids), ptr(vocab), nw, vocab.shape[1],
                                                    int(k), ptr(offs), ptr(words), ptr(valid)))
        out: Dict[Any, np.ndarray] = {}
        for i, (key, v) in enumerate(zip(keys, valid)):
            self._words[key] = nw if v else 0
            if v:
                out[key] = words[offs[i]:offs[i + 1]].copy()
        return out

    def bow_histograms(self, keys: Iterable[Any], bows: Any) -> Dict[Any, np.ndarray]:
        """pairs_selection.load_histograms (pairs_selection.py:712-727) for resident images whose words
        `compute_words` computed: {key: float64 histogram of the first words}, bit for bit BagOfWords.histogram;
        images with 8 or fewer words are left out.  The histograms stay on the device for
        `pairs_selection.match_candidates_with_bow`."""
        keys = list(dict.fromkeys(keys))
        for key in keys:
            if self._words.get(key) is None:
                raise ValueError("image %r has no words: run PairMatcher.compute_words on it first" % (key,))
        w = np.ascontiguousarray(bows.weights, dtype=np.float64)
        ids = np.array([self._ids[key] for key in keys], dtype=np.int32)
        valid = np.zeros(len(keys), dtype=np.int32)
        _lib.check(self._m.L.osfm_matcher_bow_histograms(self._m.h, len(keys), ptr(ids), ptr(w), len(w), ptr(valid)))
        out: Dict[Any, np.ndarray] = {}
        for key, v in zip(keys, valid):
            self._bow[key] = len(w) if v else 0
            if v:
                h = np.empty(len(w), dtype=np.float64)
                _lib.check(self._m.L.osfm_matcher_bow_get(self._m.h, self._ids[key], ptr(h)))
                out[key] = h
        return out

    def has_bow(self, key: Any) -> Optional[bool]:
        """None if `bow_histograms` never ran on the image, else whether it has a BoW histogram."""
        return None if key not in self._bow else bool(self._bow[key])

    def bow_select(self, refs: Sequence[Any], cands: Sequence[Any], k: int, cand_order: Optional[np.ndarray] = None,
                   labels: Optional[np.ndarray] = None) -> List[Tuple[np.ndarray, np.ndarray]]:
        """Per reference image, the columns of `cands` (and their BoW distances) that osfm_matcher_bow_select keeps:
        the k nearest by (distance, column), per camera group when `labels` (len(refs) + len(cands) ints) is given.
        cand_order: None or a len(refs) x len(cands) int array, the position of each candidate in the reference's own
        candidate list (-1: not a candidate), which then breaks ties instead of the column."""
        order = None
        if cand_order is not None:
            order = np.ascontiguousarray(cand_order, dtype=np.int32).reshape(len(refs), len(cands))
        return self._select(self._m.L.osfm_matcher_bow_select, refs, cands, k, order, labels)

    def submit(self, pairs: Sequence[Tuple[Any, Any]], lowes_ratio: float, symmetric: bool = True) -> None:
        ia = np.array([self._ids[a] for a, _ in pairs], dtype=np.int32)
        ib = np.array([self._ids[b] for _, b in pairs], dtype=np.int32)
        self._pairs = list(pairs)
        _lib.check(self._m.L.osfm_matcher_match_pairs_async(
            self._m.h, len(pairs), ia.ctypes.data_as(ctypes.c_void_p), ib.ctypes.data_as(ctypes.c_void_p),
            float(lowes_ratio), int(symmetric)))

    # -- guided matching (matching._match_descriptors_guided_impl, matching.py:260-338) ----------------------
    def set_bearings(self, key: Any, bearings: np.ndarray) -> None:
        """Unit bearing vectors of the image's features (n x 3), as `feature_loader.load_bearings` returns them;
        cast to float32 like matching.compute_inliers_bearing_epipolar does (matching.py:860-861)."""
        b = np.ascontiguousarray(bearings, dtype=np.float32)
        if b.shape != (self._n[key], 3):
            raise ValueError("bearings must be n x 3 for the %d descriptors of this image" % self._n[key])
        _lib.check(self._m.L.osfm_matcher_set_bearings(self._m.h, self._ids[key], b.ctypes.data_as(ctypes.c_void_p)))

    def match_pairs_guided(self, pairs: Sequence[Tuple[Any, Any]], poses: Sequence[Tuple[np.ndarray, np.ndarray]],
                           threshold: float, config: Dict[str, Any],
                           mask_budget_bytes: int = 1 << 30) -> Dict[Tuple[Any, Any], np.ndarray]:
        """Guided matching of a pair list: poses[p] = (R, t) = (pose.get_R_cam_to_world(), pose.get_origin()) of
        image b relative to image a.  Always symmetric, like the reference (matching.py:319).  The epipolar masks
        are built on the device, `mask_budget_bytes` of them at a time."""
        out: Dict[Tuple[Any, Any], np.ndarray] = {}
        start = 0
        while start < len(pairs):
            end, used = start, 0
            while end < len(pairs):
                a, b = pairs[end]
                need = (self._n[a] * ((self._n[b] + 31) // 32) + self._n[b] * ((self._n[a] + 31) // 32)) * 4
                if end > start and used + need > mask_budget_bytes:
                    break
                used += need
                end += 1
            chunk = list(pairs[start:end])
            ia = np.array([self._ids[a] for a, _ in chunk], dtype=np.int32)
            ib = np.array([self._ids[b] for _, b in chunk], dtype=np.int32)
            pose12 = np.array([np.concatenate([np.asarray(R, dtype=np.float64).reshape(9), np.asarray(t, dtype=np.float64).reshape(3)])
                               for R, t in poses[start:end]], dtype=np.float64).reshape(-1, 12)
            self._pairs = chunk
            _lib.check(self._m.L.osfm_matcher_match_pairs_guided_async(
                self._m.h, len(chunk), ia.ctypes.data_as(ctypes.c_void_p), ib.ctypes.data_as(ctypes.c_void_p),
                pose12.ctypes.data_as(ctypes.c_void_p), float(threshold), float(config["lowes_ratio"]), 1))
            for pr, lst in zip(chunk, self.fetch_lists()):
                out[pr] = lst
            start = end
        return out

    def last_epipolar_masks(self, i: int) -> Tuple[np.ndarray, np.ndarray]:
        """Test hook: the epipolar masks the last guided submission built on the device for its pair i, as boolean
        arrays (n1 x n2 for the a -> b pass, n2 x n1 for the b -> a pass).  `match_pairs_guided` submits in rounds of
        `mask_budget_bytes`; this reads the last round, whose pairs are numbered from 0.  Raises ValueError if the
        last submission was not guided or i is out of range."""
        n1 = n2 = 0
        if 0 <= i < len(self._pairs):
            a, b = self._pairs[i]
            n1, n2 = self._n[a], self._n[b]
        F = np.zeros((n1, (n2 + 31) // 32), dtype=np.uint32)
        T = np.zeros((n2, (n1 + 31) // 32), dtype=np.uint32)
        _lib.check(self._m.L.osfm_matcher_get_epipolar_masks(self._m.h, int(i), F.ctypes.data_as(ctypes.c_void_p),
                                                             T.ctypes.data_as(ctypes.c_void_p)))

        def bits(words: np.ndarray, ncols: int) -> np.ndarray:
            # word w, bit k = column 32 w + k: little-endian bytes, least significant bit first
            u8 = words.astype("<u4").view(np.uint8).reshape(words.shape[0], -1)
            return np.unpackbits(u8, axis=1, bitorder="little")[:, :ncols].astype(bool)

        return bits(F, n2), bits(T, n1)

    def sync(self) -> None:
        _lib.check(self._m.L.osfm_matcher_sync(self._m.h))

    def fetch_raw(self) -> np.ndarray:
        total = sum(self._n[a] for a, _ in self._pairs)
        out = np.empty(max(total, 1), dtype=np.int32)
        _lib.check(self._m.L.osfm_matcher_fetch(self._m.h, out.ctypes.data_as(ctypes.c_void_p), total))
        return out[:total]

    def fetch_lists(self) -> List[np.ndarray]:
        """The last batch as one [K, 2] (query, train) array per pair, compacted on the device
        (osfm_matcher_fetch_pairs): the host only slices one packed buffer."""
        npairs = len(self._pairs)
        cap = sum(self._n[a] for a, _ in self._pairs)
        if self._rows is None or len(self._rows) < max(cap, 1):
            self._rows = np.empty((max(cap, 1), 2), dtype=np.int32)
        offs = np.empty(npairs + 1, dtype=np.int64)
        total = ctypes.c_int64()
        _lib.check(self._m.L.osfm_matcher_fetch_pairs(self._m.h, offs.ctypes.data_as(ctypes.c_void_p),
                                                      self._rows.ctypes.data_as(ctypes.c_void_p), cap, ctypes.byref(total)))
        rows = self._rows[:total.value].copy()
        o = offs.tolist()
        return [rows[o[p]:o[p + 1]] for p in range(npairs)]

    def device_ms(self) -> Tuple[float, float]:
        a, b = ctypes.c_float(), ctypes.c_float()
        _lib.check(self._m.L.osfm_matcher_last_device_ms(self._m.h, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def last_kernel(self) -> int:
        return self._m.L.osfm_matcher_last_kernel(self._m.h)

    def device_bytes(self) -> Tuple[int, int]:
        """(bytes reserved by the descriptor slabs, bytes in use by live descriptor sets)."""
        a, b = ctypes.c_int64(), ctypes.c_int64()
        _lib.check(self._m.L.osfm_matcher_device_bytes(self._m.h, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def match_pairs(self, pairs: Sequence[Tuple[Any, Any]], config: Dict[str, Any],
                    symmetric: Optional[bool] = None) -> Dict[Tuple[Any, Any], np.ndarray]:
        if symmetric is None:
            symmetric = bool(config.get("symmetric_matching", True))  # config.py:101
        self.submit(pairs, config["lowes_ratio"], symmetric)
        return dict(zip(self._pairs, self.fetch_lists()))


def match_words(f1: np.ndarray, words1: np.ndarray, f2: np.ndarray, words2: np.ndarray, config: Dict[str, Any],
                device: int = 0) -> np.ndarray:
    """matching.match_words (matching.py:636-656) -> pyfeatures.match_using_words
    (opensfm/src/features/src/matching.cc:24-88) on the GPU.  Returns the int array [K, 2] of (feature of image 1,
    feature of image 2) the reference returns; like the reference it reads every column of `words1` and the first
    column of `words2`."""
    f1 = np.ascontiguousarray(f1, dtype=np.float32)
    f2 = np.ascontiguousarray(f2, dtype=np.float32)
    w1 = np.ascontiguousarray(words1, dtype=np.int32)
    w1 = w1.reshape(len(f1), -1)
    w2 = np.ascontiguousarray(np.asarray(words2).reshape(len(f2), -1)[:, 0], dtype=np.int32)
    if f1.ndim != 2 or f2.ndim != 2 or f1.shape[1] != f2.shape[1]:
        raise ValueError("descriptor matrices must be n x dim with the same dim")
    out = np.full(len(f1), -1, dtype=np.int32)
    with _lib.pooled("matcher", device) as m:
        _lib.check(m.L.osfm_match_words(m.h, ptr(f1), len(f1), ptr(w1), w1.shape[1], ptr(f2), len(f2), ptr(w2),
                                        f1.shape[1], float(config["lowes_ratio"]), int(config["bow_num_checks"]),
                                        ptr(out)))
    q = np.flatnonzero(out >= 0)
    return np.stack([q, out[q]], axis=1).astype(np.int32)


def match_words_symmetric(f1: np.ndarray, words1: np.ndarray, f2: np.ndarray, words2: np.ndarray,
                          config: Dict[str, Any], device: int = 0) -> List[Tuple[int, int]]:
    """matching.match_words_symmetric (matching.py:659-680)."""
    mij = {(int(a), int(b)) for a, b in match_words(f1, words1, f2, words2, config, device)}
    mji = {(int(b), int(a)) for a, b in match_words(f2, words2, f1, words1, config, device)}
    return list(mij & mji)


def vlad_distances(image: Any, other_images: Sequence[Any], histograms: Dict[Any, np.ndarray], device: int = 0):
    """pairs_selection.vlad_distances (pairs_selection.py:690-708) -> pyfeatures.compute_vlad_distances
    (features/src/matching.cc:122-145): (image, distances, other images) with the candidates that have a VLAD
    descriptor, `image` itself skipped."""
    if image not in histograms:
        return image, [], []
    others = [o for o in other_images if o != image and o in histograms]
    if not others:
        return image, [], []
    mat = np.ascontiguousarray(np.stack([histograms[image]] + [histograms[o] for o in others]), dtype=np.float32)
    out = np.zeros(len(mat), dtype=np.float64)
    with _lib.pooled("matcher", device) as m:
        _lib.check(m.L.osfm_vlad_distances(m.h, ptr(mat), mat.shape[0], mat.shape[1], 0, ptr(out)))
    return image, out[1:].tolist(), others


def unfilter_matches(matches: np.ndarray, m1: np.ndarray, m2: np.ndarray) -> np.ndarray:
    """matching.unfilter_matches (matching.py:932-936): indexes in the masked feature sets -> indexes in the original
    sets, vectorised."""
    matches = np.asarray(matches, dtype=np.int64).reshape(-1, 2)
    i1, i2 = np.flatnonzero(m1), np.flatnonzero(m2)
    return np.stack([i1[matches[:, 0]], i2[matches[:, 1]]], axis=1) if len(matches) else np.zeros((0, 2), dtype=np.int64)


ROBUST_MIN_MATCHES = 8   # robust_match_fundamental / robust_match_calibrated return nothing below this


def robust_match_fundamental(p1: np.ndarray, p2: np.ndarray, matches: np.ndarray, config: Dict[str, Any]):
    """matching.robust_match_fundamental (matching.py:780-802): (F, inlier matches) of cv2.findFundamentalMat with
    FM_RANSAC, robust_matching_threshold and confidence 0.9999, on the host as the reference runs it."""
    import cv2

    matches = np.asarray(matches)
    if len(matches) < ROBUST_MIN_MATCHES:
        return np.array([]), np.array([])
    q1 = p1[matches[:, 0]][:, :2].copy()
    q2 = p2[matches[:, 1]][:, :2].copy()
    F, mask = cv2.findFundamentalMat(q1, q2, cv2.FM_RANSAC, config["robust_matching_threshold"], 0.9999)
    if F is None or F[2, 2] == 0.0:
        return F, np.array([])
    return F, matches[mask.ravel().nonzero()]


def robust_match_calibrated(p1: np.ndarray, p2: np.ndarray, camera1, camera2, matches: np.ndarray,
                            config: Dict[str, Any]) -> np.ndarray:
    """matching.robust_match_calibrated (matching.py:871-903) on the GPU: five-point RANSAC of the matches' bearings
    (camera.pixel_bearing_many), then the bearing inliers at 4, 2 and 1 times robust_matching_calib_threshold, each
    refined with five_point_refine_match_iterations; returns the matches the refined pose keeps."""
    from . import relative_pose

    matches = np.asarray(matches)
    if len(matches) < ROBUST_MIN_MATCHES:
        return np.array([])
    b1 = camera1.pixel_bearing_many(p1[matches[:, 0]][:, :2].copy())
    b2 = camera2.pixel_bearing_many(p2[matches[:, 1]][:, :2].copy())
    res = relative_pose.robust_match_lists([b1], [b2], config["robust_matching_calib_threshold"],
                                           relative_pose.ITERATIONS, config["five_point_refine_match_iterations"])
    return matches[res.mask(0)]


def uses_fundamental(camera1, camera2) -> bool:
    """robust_match's dispatch: both cameras perspective or brown with k1 = k2 = 0 (matching.py:919-926)."""
    return all(c.projection_type in ["perspective", "brown"] and c.k1 == 0.0 and c.k2 == 0.0
               for c in (camera1, camera2))


def robust_match(p1: np.ndarray, p2: np.ndarray, camera1, camera2, matches: np.ndarray,
                 config: Dict[str, Any]) -> np.ndarray:
    """matching.robust_match (matching.py:906-929): the fundamental matrix for undistorted perspective cameras, the
    essential matrix on the GPU for every other camera."""
    if uses_fundamental(camera1, camera2):
        return robust_match_fundamental(p1, p2, matches, config)[1]
    return robust_match_calibrated(p1, p2, camera1, camera2, matches, config)


def _verify_pairs(ms: Dict[Tuple[Any, Any], np.ndarray], verify: Dict[str, Any], config: Dict[str, Any],
                  device: int) -> Dict[Tuple[Any, Any], np.ndarray]:
    """robust_match of every pair in `ms` (its descriptor matches): the calibrated pairs in one device call over one
    bearing table (each image's points' bearings computed once), the others through robust_match_fundamental."""
    from . import relative_pose

    cameras, points = verify["cameras"], verify["points"]
    out: Dict[Tuple[Any, Any], np.ndarray] = {}
    calibrated = []
    for p, m in ms.items():
        if uses_fundamental(cameras[p[0]], cameras[p[1]]):
            out[p] = robust_match_fundamental(points[p[0]], points[p[1]], m, config)[1]
        elif len(m) < ROBUST_MIN_MATCHES:
            out[p] = np.array([])
        else:
            calibrated.append(p)
    if not calibrated:
        return out
    images = list(dict.fromkeys(i for p in calibrated for i in p))
    base, tables, n = {}, [], 0
    for im in images:
        base[im] = n
        tables.append(cameras[im].pixel_bearing_many(np.asarray(points[im])[:, :2].copy()))
        n += len(tables[-1])
    starts = np.concatenate([[0], np.cumsum([len(ms[p]) for p in calibrated])]).astype(np.int64)
    row_a = np.concatenate([base[p[0]] + ms[p][:, 0] for p in calibrated]).astype(np.int64)
    row_b = np.concatenate([base[p[1]] + ms[p][:, 1] for p in calibrated]).astype(np.int64)
    res = relative_pose.robust_match_pairs(np.concatenate(tables), starts, row_a, row_b,
                                           config["robust_matching_calib_threshold"], relative_pose.ITERATIONS,
                                           config["five_point_refine_match_iterations"], device)
    for k, p in enumerate(calibrated):
        out[p] = ms[p][res.mask(k)]
    return out


def match_images_with_pairs(descriptors: Dict[Any, np.ndarray], pairs: Sequence[Tuple[Any, Any]], config: Dict[str, Any],
                            robust_filter=None, feature_masks: Optional[Dict[Any, np.ndarray]] = None,
                            guided: Optional[Dict[str, Any]] = None, device: int = 0, rank: int = 0, world: int = 1,
                            uint8_is_l2: bool = False,
                            verify: Optional[Dict[str, Any]] = None) -> Dict[Tuple[Any, Any], np.ndarray]:
    """The pair loop of `matching.match_images_with_pairs` / `matching.match` (matching.py:63-98, 563-634) as one
    batched submission: every image's descriptors are uploaded once, the pair list (this rank's shard of it) is
    matched in one launch sequence, then per pair the reference's post-processing runs on the host:

      * fewer than config["robust_matching_min_match"] descriptor matches -> empty result (:583-590);
      * `robust_filter(im1, im2, matches) -> matches` (the geometric verification `_match_robust_impl`, :547-560 --
        host-side geometry, outside this engine) if given, and the same gate on its output (:629-631);
      * `unfilter_matches` when both images have a feature mask (:596-600).

    descriptors: image -> the (masked) descriptor matrix `feature_loader.load_all_data(masked=True)` returns.
    guided: None, or {"bearings": image -> n x 3, "poses": (im1, im2) -> (R, t), "threshold": rad}: pairs with a
    pose are matched under the epipolar mask (`_match_descriptors_guided_impl`), always symmetric.
    verify: None, or {"cameras": image -> camera, "points": image -> the (masked) feature points}: the reference's
    own geometric verification, `robust_match`, of every pair past the first gate instead of `robust_filter`; the
    calibrated pairs are verified in one device call (`robust_match_calibrated` for all of them at once).
    Returns {(im1, im2): int array [K, 2]} for this rank's pairs; `opensfm_b200.dist.gather_pair_results` merges
    the ranks."""
    if robust_filter is not None and verify is not None:
        raise ValueError("pass robust_filter or verify, not both")
    sizes = {k: len(v) for k, v in descriptors.items()}
    mine = shard_pairs(list(pairs), sizes, world)[rank] if world > 1 else list(pairs)
    pm = PairMatcher(device=device)
    needed = sorted({i for p in mine for i in p}, key=lambda k: str(k))
    pm.add_many([(k, descriptors[k]) for k in needed], uint8_is_l2=uint8_is_l2)
    gp = [p for p in mine if guided is not None and p in guided["poses"]]
    up = [p for p in mine if not (guided is not None and p in guided["poses"])]
    raw: Dict[Tuple[Any, Any], np.ndarray] = {}
    if up:
        raw.update(pm.match_pairs(up, config))
    if gp:
        for k in {i for p in gp for i in p}:
            pm.set_bearings(k, guided["bearings"][k])
        raw.update(pm.match_pairs_guided(gp, [guided["poses"][p] for p in gp], guided["threshold"], config))
    min_match = int(config.get("robust_matching_min_match", 20))
    out: Dict[Tuple[Any, Any], np.ndarray] = {}
    empty = np.zeros((0, 2), dtype=np.int64)
    verified: Dict[Tuple[Any, Any], np.ndarray] = {}
    if verify is not None:
        verified = _verify_pairs({p: raw[p] for p in mine if len(raw[p]) >= min_match}, verify, config, device)
    for p in mine:
        m = raw[p]
        if len(m) < min_match:
            out[p] = empty
            continue
        if robust_filter is not None:
            m = np.asarray(robust_filter(p[0], p[1], m), dtype=np.int64).reshape(-1, 2)
        if verify is not None:
            m = np.asarray(verified[p], dtype=np.int64).reshape(-1, 2)
        if feature_masks is not None and feature_masks.get(p[0]) is not None and feature_masks.get(p[1]) is not None:
            m = unfilter_matches(m, feature_masks[p[0]], feature_masks[p[1]])
        out[p] = empty if len(m) < min_match else m
    return out


def shard_pairs(pairs: Sequence[Tuple[Any, Any]], sizes: Dict[Any, int], world: int) -> List[List[Tuple[Any, Any]]]:
    """Split a pair list over `world` GPUs: balanced sum(N_i * M_i), and pairs that share an image on the same GPU
    so that every rank uploads / keeps resident only ~1/world of the descriptor sets (SURVEY.md 8e).

    The images are ordered by a breadth-first walk of the pair graph (neighbouring images get neighbouring ranks in
    the order), the pairs are sorted by that order and cut into `world` contiguous runs of equal work.  Image pairs
    are independent units (matching.py:83 maps a pure function over them), so no collective is needed."""
    if world <= 1 or not pairs:
        return [list(pairs)] + [[] for _ in range(max(world - 1, 0))]
    adj: Dict[Any, List[Any]] = {}
    for a, b in pairs:
        adj.setdefault(a, []).append(b)
        adj.setdefault(b, []).append(a)
    rank: Dict[Any, int] = {}
    for root in adj:                       # insertion order: deterministic on every rank
        if root in rank:
            continue
        queue, head = [root], 0
        rank[root] = len(rank)
        while head < len(queue):
            u = queue[head]
            head += 1
            for v in adj[u]:
                if v not in rank:
                    rank[v] = len(rank)
                    queue.append(v)
    order = sorted(range(len(pairs)), key=lambda i: (min(rank[pairs[i][0]], rank[pairs[i][1]]),
                                                     max(rank[pairs[i][0]], rank[pairs[i][1]]), i))
    work = [sizes[pairs[i][0]] * sizes[pairs[i][1]] for i in order]
    total = float(sum(work))
    shards: List[List[int]] = [[] for _ in range(world)]
    acc, r = 0.0, 0
    for i, w in zip(order, work):
        # close the current run once it holds its share (the last rank takes the remainder)
        if r < world - 1 and acc + 0.5 * w > total * (r + 1) / world:
            r += 1
        shards[r].append(i)
        acc += w
    return [[pairs[i] for i in sorted(s)] for s in shards]
