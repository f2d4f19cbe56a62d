"""Drop-in track creation: the `opensfm.tracking` names this engine replaces.

    create_tracks_manager(features, colors, segmentations, instances, matches, min_length, depths, ...)
                                                                    opensfm/tracking.py:72-150
    common_tracks / all_common_tracks[_with_features|_without_features]   opensfm/tracking.py:153-235
    TracksManager (read-only part of pymap.TracksManager)           opensfm/src/map/src/tracks_manager.cc

The connected components of the match graph, the reference's track filter and the common tracks of every image
pair are computed by the CUDA library (opensfm_b200/csrc/tracks.cu) through the C ABI; there is no CPU path.
The host side only marshals: it concatenates the per-pair match arrays, and builds `Observation` objects lazily
from the structure-of-arrays result when an accessor asks for them.  A TracksManager keeps the tracks handle that
built it, with the observations on the device, for as long as it lives: `TracksManager.triangulate`
(opensfm_b200/triangulation.py) runs on them without uploading the tracks again.

One stated difference from the reference: tracks are numbered 0 .. T - 1 by their smallest (image, feature) with
images in name order, whereas the reference numbers them in the iteration order of its union-find's dictionary.
Track ids are opaque strings in both; the partition of the features into tracks is identical.
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import ptr
from .map_types import Depth, Observation

NO_SEMANTIC_VALUE = -1   # pymap.Observation.NO_SEMANTIC_VALUE


class TracksManager:
    """Array-backed, read-only mirror of the part of pymap.TracksManager the pipeline reads.  Observations are
    kept as arrays sorted by (track, image); `Observation` objects are made when an accessor returns them."""

    def __init__(self, handle: _lib.Handle, images: List[Any], obs_track: np.ndarray, obs_image: np.ndarray,
                 obs_feature: np.ndarray, track_start: np.ndarray, features, colors, segmentations, instances, depths,
                 depth_is_radial: bool, depth_std_deviation: float, device_ms: float):
        self._handle: Optional[_lib.Handle] = handle   # holds the observations on the device; released with self
        self.images = images
        self.obs_track, self.obs_image, self.obs_feature, self.track_start = obs_track, obs_image, obs_feature, track_start
        self._features, self._colors, self._segmentations, self._instances = features, colors, segmentations, instances
        self._depths = depths or {}
        self._depth_is_radial, self._depth_std = depth_is_radial, depth_std_deviation
        self._index = {im: i for i, im in enumerate(images)}
        self._by_image: Optional[Tuple[np.ndarray, np.ndarray]] = None
        self._xy_scale: Optional[Tuple[np.ndarray, np.ndarray]] = None
        self._common: Optional[Tuple[np.ndarray, ...]] = None
        self._pair_row: Optional[Dict[Tuple[int, int], int]] = None
        self._ids: Optional[np.ndarray] = None
        self.build_device_ms = device_ms
        self.common_device_ms = 0.0
        self.triangulate_device_ms = 0.0

    def __del__(self):
        self._give_back()

    def _give_back(self) -> None:
        h, self._handle = self._handle, None
        if h is not None:
            _lib.release(h)

    # -- structure-of-arrays views ----------------------------------------------------------------------------
    def _shot_order(self) -> Tuple[np.ndarray, np.ndarray]:
        """(observation rows sorted by (image, track), first row of every image)."""
        if self._by_image is None:
            order = np.argsort(self.obs_image, kind="stable")
            start = np.searchsorted(self.obs_image[order], np.arange(len(self.images) + 1), side="left")
            self._by_image = (order, start)
        return self._by_image

    def _points(self) -> Tuple[np.ndarray, np.ndarray]:
        if self._xy_scale is None:
            xy = np.zeros((len(self.obs_image), 2), dtype=np.float64)
            scale = np.zeros(len(self.obs_image), dtype=np.float64)
            order, start = self._shot_order()
            for i, im in enumerate(self.images):
                rows = order[start[i]:start[i + 1]]
                if len(rows):
                    f = np.asarray(self._features[im])[self.obs_feature[rows]]
                    xy[rows] = f[:, :2]
                    scale[rows] = f[:, 2]
            self._xy_scale = (xy, scale)
        return self._xy_scale

    def as_arrays(self) -> Dict[str, Any]:
        """The observations as arrays sorted by (track, image): what `ba_problem.make_problem` and
        `add_observations_bulk` take, without building one object per observation.  obs_image indexes `images`."""
        xy, scale = self._points()
        return dict(obs_track=self.obs_track, obs_image=self.obs_image, obs_feature=self.obs_feature, xy=xy,
                    scale=scale, track_start=self.track_start, images=list(self.images))

    def _observation(self, row: int) -> Observation:
        im = self.images[self.obs_image[row]]
        f = int(self.obs_feature[row])
        x, y, s = np.asarray(self._features[im])[f][:3]
        r, g, b = self._colors[im][f]
        seg = int(self._segmentations[im][f]) if im in self._segmentations else NO_SEMANTIC_VALUE
        inst = int(self._instances[im][f]) if im in self._instances else NO_SEMANTIC_VALUE
        obs = Observation(x, y, s, int(r), int(g), int(b), f, seg, inst)
        if im in self._depths:
            d = float(self._depths[im][f])
            if not np.isnan(d) and not np.isinf(d):
                obs.depth_prior = Depth(d, max(self._depth_std * d, self._depth_std), self._depth_is_radial)
        return obs

    def _shot(self, shot_id: Any) -> int:
        i = self._index.get(shot_id)
        if i is None or self._shot_order()[1][i] == self._shot_order()[1][i + 1]:
            raise RuntimeError("Accessing invalid shot ID")
        return i

    def _track(self, track_id: str) -> int:
        try:
            t = int(track_id)
        except (TypeError, ValueError):
            t = -1
        if not (0 <= t < self.num_tracks()) or str(t) != track_id:
            raise RuntimeError("Accessing invalid track ID")
        return t

    # -- pymap.TracksManager ----------------------------------------------------------------------------------
    def num_shots(self) -> int:
        return int(np.count_nonzero(np.diff(self._shot_order()[1])))

    def num_tracks(self) -> int:
        return len(self.track_start) - 1

    def get_shot_ids(self) -> List[Any]:
        n = np.diff(self._shot_order()[1])
        return [im for i, im in enumerate(self.images) if n[i]]

    def _track_ids(self) -> np.ndarray:
        """str(k) of every track as an object array: id lists are then one fancy index, not one str() per entry."""
        if self._ids is None:
            self._ids = np.array([str(t) for t in range(self.num_tracks())], dtype=object)
        return self._ids

    def get_track_ids(self) -> List[str]:
        return self._track_ids().tolist()

    def get_shot_observations(self, shot_id: Any) -> Dict[str, Observation]:
        i = self._shot(shot_id)
        order, start = self._shot_order()
        return {str(self.obs_track[r]): self._observation(r) for r in order[start[i]:start[i + 1]]}

    def get_track_observations(self, track_id: str) -> Dict[Any, Observation]:
        t = self._track(track_id)
        return {self.images[self.obs_image[r]]: self._observation(r)
                for r in range(self.track_start[t], self.track_start[t + 1])}

    def get_observation(self, shot_id: Any, track_id: str) -> Observation:
        i, t = self._shot(shot_id), self._track(track_id)
        b, e = self.track_start[t], self.track_start[t + 1]
        r = b + np.searchsorted(self.obs_image[b:e], i)
        if r >= e or self.obs_image[r] != i:
            raise RuntimeError("Accessing invalid track ID")
        return self._observation(int(r))

    def _common_arrays(self) -> Tuple[np.ndarray, ...]:
        """(pair_a, pair_b, pair_start, common_obs_a, common_obs_b) of every connected image pair, from the device."""
        if self._common is None:
            h = self._handle
            nq, nr = ctypes.c_int64(0), ctypes.c_int64(0)
            _lib.check(h.L.osfm_tracks_common(h.h, ctypes.byref(nq), ctypes.byref(nr)))
            pa, pb = np.zeros(nq.value, dtype=np.int32), np.zeros(nq.value, dtype=np.int32)
            ps = np.zeros(nq.value + 1, dtype=np.int64)
            ca, cb = np.zeros(nr.value, dtype=np.int64), np.zeros(nr.value, dtype=np.int64)
            _lib.check(h.L.osfm_tracks_get_common(h.h, ptr(pa), ptr(pb), ptr(ps), ptr(ca), ptr(cb)))
            ms = ctypes.c_float(0)
            _lib.check(h.L.osfm_tracks_last_device_ms(h.h, None, ctypes.byref(ms)))
            self.common_device_ms = float(ms.value)
            self._common = (pa, pb, ps, ca, cb)
        return self._common

    def triangulate(self, image_rt: np.ndarray, image_origin: np.ndarray, image_in: np.ndarray, bearings: np.ndarray,
                    selected: np.ndarray, threshold: float, min_ray_angle: float, min_depth: float, iterations: int
                    ) -> Tuple[np.ndarray, np.ndarray]:
        """TrackTriangulator.triangulate (opensfm/reconstruction.py:1032-1073) of every selected track at once, on
        the device, from the observations the tracks handle keeps there: (X[T, 3], status[T]).

        Per image of `images`: image_rt (R^T of the world-to-camera rotation, 3 x 3), image_origin (3) and image_in
        (whether the image is in the reconstruction; only its observations are used).  Per observation, in the
        (track, image) order of `obs_track`: bearings (camera frame, 3; read only in images of the reconstruction).
        Per track: selected.  threshold and min_ray_angle are in radians.  status is one of the STATUS_* codes of
        opensfm_b200.triangulation; X is NaN unless the status is STATUS_OK."""
        h = self._handle
        I, T, N = len(self.images), self.num_tracks(), len(self.obs_track)
        rt = np.ascontiguousarray(image_rt, dtype=np.float64).reshape(I, 9)
        origin = np.ascontiguousarray(image_origin, dtype=np.float64).reshape(I, 3)
        inn = np.ascontiguousarray(image_in, dtype=np.uint8).reshape(I)
        b = np.ascontiguousarray(bearings, dtype=np.float64).reshape(N, 3)
        sel = np.ascontiguousarray(selected, dtype=np.uint8).reshape(T)
        status = np.zeros(T, dtype=np.int8)
        X = np.zeros((T, 3), dtype=np.float64)
        _lib.check(h.L.osfm_tracks_triangulate(h.h, I, ptr(rt), ptr(origin), ptr(inn), N, ptr(b), T, ptr(sel),
                                               float(threshold), float(min_ray_angle), float(min_depth),
                                               int(iterations), ptr(status), ptr(X)))
        ms = ctypes.c_float(0)
        _lib.check(h.L.osfm_tracks_last_triangulate_ms(h.h, ctypes.byref(ms)))
        self.triangulate_device_ms = float(ms.value)
        return X, status

    def get_all_pairs_connectivity(self, shots: Sequence[Any] = (), tracks: Sequence[str] = ()
                                   ) -> Dict[Tuple[Any, Any], int]:
        """{(shot1, shot2): tracks in common}, shot1 < shot2, optionally restricted to some shots and tracks."""
        if not len(shots) and not len(tracks):
            pa, pb, ps, _, _ = self._common_arrays()
            n = np.diff(ps)
            return {(self.images[a], self.images[b]): int(c) for a, b, c in zip(pa.tolist(), pb.tolist(), n.tolist())}
        # the restricted form, on the host: pairs of kept observations d rows apart inside one track
        keep = np.ones(len(self.obs_track), dtype=bool)
        if len(shots):
            ids = [self._index[s] for s in shots if s in self._index]
            keep &= np.isin(self.obs_image, np.asarray(ids, dtype=np.int32))
        if len(tracks):
            ids = [int(t) for t in tracks if str(t).isdigit() and int(t) < self.num_tracks()]
            keep &= np.isin(self.obs_track, np.asarray(ids, dtype=np.int32))
        trk, img = self.obs_track[keep], self.obs_image[keep].astype(np.int64)
        out: Dict[Tuple[Any, Any], int] = {}
        n_img = len(self.images)
        keys = []
        d = 1
        while d < len(trk):
            same = trk[d:] == trk[:-d]
            if not same.any():
                break
            keys.append(img[:-d][same] * n_img + img[d:][same])
            d += 1
        if keys:
            k, c = np.unique(np.concatenate(keys), return_counts=True)
            out = {(self.images[a], self.images[b]): int(n) for a, b, n in zip((k // n_img).tolist(), (k % n_img).tolist(),
                                                                                 c.tolist())}
        return out

    def _pair_rows(self, shot1: Any, shot2: Any) -> Tuple[np.ndarray, np.ndarray]:
        """Observation rows of shot1 and shot2 in their common tracks, tracks ascending."""
        i, j = self._shot(shot1), self._shot(shot2)
        pa, pb, ps, ca, cb = self._common_arrays()
        if self._pair_row is None:
            self._pair_row = {(a, b): q for q, (a, b) in enumerate(zip(pa.tolist(), pb.tolist()))}
        q = self._pair_row.get((min(i, j), max(i, j)))
        if q is None or i == j:
            return ca[:0], cb[:0]
        ra, rb = ca[ps[q]:ps[q + 1]], cb[ps[q]:ps[q + 1]]
        return (ra, rb) if i < j else (rb, ra)

    def get_all_common_observations(self, shot1: Any, shot2: Any) -> List[Tuple[str, Observation, Observation]]:
        r1, r2 = self._pair_rows(shot1, shot2)
        return [(str(self.obs_track[a]), self._observation(int(a)), self._observation(int(b)))
                for a, b in zip(r1, r2)]


def create_tracks_manager(features: Dict[Any, np.ndarray], colors: Dict[Any, np.ndarray],
                          segmentations: Dict[Any, np.ndarray], instances: Dict[Any, np.ndarray],
                          matches: Dict[Tuple[Any, Any], Any], min_length: int,
                          depths: Optional[Dict[Any, np.ndarray]] = None, depth_is_radial: bool = True,
                          depth_std_deviation: float = 1.0, device: int = 0) -> TracksManager:
    """Link matches into tracks (opensfm/tracking.py:72-150) on the GPU.

    matches: {(im1, im2): K x 2 (feature of im1, feature of im2)} as lists of tuples or integer arrays; both
    orders of a pair may be present.  Images are ordered by name.  An image that occurs in `matches` but not in
    `features` counts towards a track's length and duplicates and yields no observation, as in the reference."""
    images = sorted(set(features) | {im for pair in matches for im in pair})
    index = {im: i for i, im in enumerate(images)}
    num_features = np.array([len(features[im]) if im in features else 0 for im in images], dtype=np.int32)
    has_features = np.array([im in features for im in images], dtype=np.uint8)
    rows = [np.asarray(m, dtype=np.int32).reshape(-1, 2) for m in matches.values()]
    pair_a = np.array([index[a] for a, _ in matches], dtype=np.int32)
    pair_b = np.array([index[b] for _, b in matches], dtype=np.int32)
    match_start = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], dtype=np.int64, out=match_start[1:])
    if not has_features.all():
        # no feature file: the image has as many features as the matches name
        for (a, b), r in zip(matches, rows):
            for im, col in ((a, 0), (b, 1)):
                if im not in features and len(r):
                    num_features[index[im]] = max(num_features[index[im]], int(r[:, col].max()) + 1)
    allrows = np.ascontiguousarray(np.concatenate(rows)) if rows else np.zeros((0, 2), dtype=np.int32)

    h = _lib.acquire("tracks", device)
    try:
        nt, no = ctypes.c_int64(0), ctypes.c_int64(0)
        _lib.check(h.L.osfm_tracks_build(h.h, len(images), ptr(num_features), ptr(has_features), len(rows),
                                         ptr(pair_a), ptr(pair_b), ptr(match_start), ptr(allrows),
                                         int(min_length), ctypes.byref(nt), ctypes.byref(no)))
        obs_track, obs_image, obs_feature = (np.zeros(no.value, dtype=np.int32) for _ in range(3))
        track_start = np.zeros(nt.value + 1, dtype=np.int64)
        _lib.check(h.L.osfm_tracks_get(h.h, ptr(obs_track), ptr(obs_image), ptr(obs_feature), ptr(track_start)))
        ms = ctypes.c_float(0)
        _lib.check(h.L.osfm_tracks_last_device_ms(h.h, ctypes.byref(ms), None))
    except Exception:
        _lib.release(h)
        raise
    return TracksManager(h, images, obs_track, obs_image, obs_feature, track_start, features, colors, segmentations,
                         instances, depths, depth_is_radial, depth_std_deviation, float(ms.value))


def common_tracks(tracks_manager: TracksManager, im1: Any, im2: Any) -> Tuple[List[str], np.ndarray, np.ndarray]:
    """Tracks observed in both images: (track ids, points in im1, points in im2) (opensfm/tracking.py:153-176)."""
    r1, r2 = tracks_manager._pair_rows(im1, im2)
    if not len(r1):
        return [], np.array([]), np.array([])
    xy = tracks_manager._points()[0]
    return tracks_manager._track_ids()[tracks_manager.obs_track[r1]].tolist(), xy[r1], xy[r2]


def all_common_tracks(tracks_manager: TracksManager, include_features: bool = True, min_common: int = 50):
    """{(im1, im2): (track ids, points in im1, points in im2)} (or just the track ids) of every image pair with at
    least min_common tracks in common (opensfm/tracking.py:202-235), from the device's per-pair lists."""
    pa, pb, ps, ca, cb = tracks_manager._common_arrays()
    xy = tracks_manager._points()[0] if include_features else None
    track_ids = tracks_manager._track_ids()
    out = {}
    for q in np.nonzero(np.diff(ps) >= min_common)[0].tolist():
        r1, r2 = ca[ps[q]:ps[q + 1]], cb[ps[q]:ps[q + 1]]
        ids = track_ids[tracks_manager.obs_track[r1]].tolist()
        key = (tracks_manager.images[pa[q]], tracks_manager.images[pb[q]])
        out[key] = (ids, xy[r1], xy[r2]) if include_features else ids
    return out


def all_common_tracks_with_features(tracks_manager: TracksManager, min_common: int = 50):
    return all_common_tracks(tracks_manager, include_features=True, min_common=min_common)


def all_common_tracks_without_features(tracks_manager: TracksManager, min_common: int = 50):
    return all_common_tracks(tracks_manager, include_features=False, min_common=min_common)
