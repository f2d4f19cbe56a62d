"""Dense depthmaps on the GPU: pydense's DepthmapEstimator, DepthmapCleaner and DepthmapPruner
(opensfm/src/dense/src/depthmap.cc) over the `osfm_dense` handle.

The three classes have pydense's methods, argument order, return values and defaults, so

    opensfm.dense.pydense = opensfm_b200.dense

re-points the reference's dense stage.  Each call runs on a pooled handle.  `depthmaps()` is the bulk form: every
reference of a submission is estimated, cleaned and pruned on the device, with the maps kept resident in between.

The one deliberate difference from pydense: random draws come from Philox4x32-10 keyed by (seed, reference key), not
from rand() and a std::random_device-seeded mt19937, so results are reproducible and do not depend on the batch.
"""
from __future__ import annotations

import ctypes
import logging
import zlib
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib

METHODS = {"BRUTE_FORCE": 0, "PATCH_MATCH": 1, "PATCH_MATCH_SAMPLE": 2}
MAX_PATCH = 15
MAX_VIEWS = 32
_WD = 2 * ((MAX_PATCH - 1) // 2) ** 2 + 1


def bilateral_weights() -> np.ndarray:
    """DepthmapEstimator::BilateralWeight as a table over (|dcolor| in 0..255, dx^2 + dy^2): the argument formed in f32
    as the reference forms it, float32(exp(float64(arg)))."""
    f32 = np.float32
    dcolor_factor = f32(1.0) / (f32(2) * f32(50.0) * f32(50.0))
    dx_factor = f32(1.0) / (f32(2) * f32(5.0) * f32(5.0))
    dc = np.arange(256, dtype=f32)[:, None]
    d2 = np.arange(_WD, dtype=f32)[None, :]
    arg = (-dc) * dc * dcolor_factor - d2 * dx_factor
    return np.exp(arg.astype(np.float64)).astype(np.float32)


def view_terms(Ks, Rs, ts) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """K^-1 per view, and Q = R_v R_0^T, a = Q t_0 - t_v of every view against view 0, in fp64 (AddView)."""
    K = np.asarray(Ks, dtype=np.float64).reshape(-1, 3, 3)
    R = np.asarray(Rs, dtype=np.float64).reshape(-1, 3, 3)
    t = np.asarray(ts, dtype=np.float64).reshape(-1, 3)
    Kinv = np.ascontiguousarray(np.linalg.inv(K))
    Q = np.ascontiguousarray(R @ R[0].T)
    a = np.ascontiguousarray(np.einsum("nij,j->ni", Q, t[0]) - t)
    return Kinv, Q, a


@dataclass
class View:
    """One view at depthmap resolution.  gray / mask for estimation, color / labels for pruning; the maps of an
    earlier run (raw depth with its plane, clean depth) may be given to be reused."""
    K: np.ndarray
    R: np.ndarray
    t: np.ndarray
    width: int
    height: int
    gray: Optional[np.ndarray] = None
    mask: Optional[np.ndarray] = None
    color: Optional[np.ndarray] = None
    labels: Optional[np.ndarray] = None
    raw_depth: Optional[np.ndarray] = None
    plane: Optional[np.ndarray] = None
    clean_depth: Optional[np.ndarray] = None


@dataclass
class Reference:
    """One reference shot: its views as indices into the view list, itself first, and its estimation options."""
    views: List[int]
    min_depth: float = 0.0
    max_depth: float = 0.0
    method: str = "PATCH_MATCH_SAMPLE"
    patch_size: int = 7
    num_depth_planes: int = 50
    patchmatch_iterations: int = 3
    min_patch_sd: float = 5.0
    key: int = 0


@dataclass
class Depthmaps:
    depth: List[np.ndarray] = field(default_factory=list)
    plane: List[np.ndarray] = field(default_factory=list)
    score: List[np.ndarray] = field(default_factory=list)
    nghbr: List[np.ndarray] = field(default_factory=list)
    device_ms: float = 0.0


def _u8(a, shape, what):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    if a.shape != shape:
        raise ValueError("%s has shape %s, expected %s" % (what, a.shape, shape))
    return a


def _f32(a, shape, what):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.shape != shape:
        raise ValueError("%s has shape %s, expected %s" % (what, a.shape, shape))
    return a


def _lists(refs: Sequence[Reference], key=lambda r: r.views):
    lists = [list(key(r)) for r in refs]
    start = np.zeros(len(lists) + 1, dtype=np.int32)
    start[1:] = np.cumsum([len(v) for v in lists])
    flat = np.array([v for lst in lists for v in lst], dtype=np.int32)
    return start, flat if len(flat) else np.zeros(1, np.int32)


class Engine:
    """The views of one submission, resident on a dense handle held until `close()`."""

    def __init__(self, views: Sequence[View], device: int = 0):
        self.views = list(views)
        self.handle = _lib.acquire("dense", device)
        try:
            self._upload()
        except BaseException:
            self.close()
            raise

    def _upload(self):
        L, h = self.handle.L, self.handle.h
        n = len(self.views)
        shape = [(v.height, v.width) for v in self.views]
        size = np.array([(v.width, v.height) for v in self.views], dtype=np.int32).reshape(-1, 2)
        K = np.ascontiguousarray([np.asarray(v.K, np.float64).reshape(3, 3) for v in self.views]).reshape(-1, 9)
        R = np.ascontiguousarray([np.asarray(v.R, np.float64).reshape(3, 3) for v in self.views]).reshape(-1, 9)
        t = np.ascontiguousarray([np.asarray(v.t, np.float64).reshape(3) for v in self.views]).reshape(-1, 3)
        Kinv = view_terms(K, R, t)[0] if n else np.zeros((0, 3, 3))

        def slab(attr, channels):
            if n == 0 or any(getattr(v, attr) is None for v in self.views):
                return None
            parts = [_u8(getattr(v, attr), s + ((channels,) if channels > 1 else ()), "view %d %s" % (k, attr))
                     for k, (v, s) in enumerate(zip(self.views, shape))]
            return np.ascontiguousarray(np.concatenate([p.reshape(-1) for p in parts]))

        gray, mask, rgb, labels = slab("gray", 1), slab("mask", 1), slab("color", 3), slab("labels", 1)
        self._keep = (size, K, Kinv, R, t, gray, mask, rgb, labels)
        _lib.check(L.osfm_dense_set_views(h, n, _lib.ptr(size), _lib.ptr(K), _lib.ptr(np.ascontiguousarray(Kinv)),
                                          _lib.ptr(R), _lib.ptr(t), _lib.ptr(gray), _lib.ptr(mask),
                                          _lib.ptr(rgb if labels is not None else None),
                                          _lib.ptr(labels if rgb is not None else None)))
        for k, (v, s) in enumerate(zip(self.views, shape)):
            if v.raw_depth is not None or v.plane is not None or v.clean_depth is not None:
                self.set_maps(k, v.raw_depth, v.plane, v.clean_depth)

    def close(self):
        if self.handle is not None:
            _lib.release(self.handle)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _shape(self, k):
        return (self.views[k].height, self.views[k].width)

    def set_maps(self, k, raw_depth=None, plane=None, clean_depth=None):
        s = self._shape(k)
        rd = None if raw_depth is None else _f32(raw_depth, s, "raw depth of view %d" % k)
        pl = None if plane is None else _f32(plane, s + (3,), "plane of view %d" % k)
        cd = None if clean_depth is None else _f32(clean_depth, s, "clean depth of view %d" % k)
        _lib.check(self.handle.L.osfm_dense_set_maps(self.handle.h, k, _lib.ptr(rd), _lib.ptr(pl), _lib.ptr(cd)))

    def estimate(self, refs: Sequence[Reference], seed: int = 0, min_score: float = -np.inf) -> Depthmaps:
        """The ungated maps of every reference; the gated depth (score > min_score, depth < max_depth) goes to the
        reference view's raw slot for `clean`."""
        start, flat = _lists(refs)
        Q, A = np.zeros((len(flat), 9)), np.zeros((len(flat), 3))
        o = 0
        for r in refs:
            n = len(r.views)
            if all(0 <= v < len(self.views) for v in r.views):   # otherwise the engine rejects the list
                vs = [self.views[v] for v in r.views]
                _, q, a = view_terms([v.K for v in vs], [v.R for v in vs], [v.t for v in vs])
                Q[o:o + n], A[o:o + n] = q.reshape(n, 9), a
            o += n
        params = np.array([(METHODS.get(r.method, -1) if isinstance(r.method, str) else r.method, r.patch_size,
                            r.num_depth_planes, r.patchmatch_iterations, r.key & 0xFFFFFFFF) for r in refs],
                          dtype=np.int64).reshape(-1, 5).astype(np.uint32).view(np.int32)   # the key as its bits
        rng = np.array([(r.min_depth, r.max_depth) for r in refs], dtype=np.float64).reshape(-1, 2)
        var = np.array([np.float32(r.min_patch_sd) * np.float32(r.min_patch_sd) for r in refs], dtype=np.float32)
        sizes = [self._shape(r.views[0]) if 0 <= r.views[0] < len(self.views) else (0, 0) for r in refs]
        total = sum(h * w for h, w in sizes)
        depth = np.zeros(max(total, 1), np.float32)
        plane = np.zeros(max(total, 1) * 3, np.float32)
        score = np.zeros(max(total, 1), np.float32)
        nghbr = np.zeros(max(total, 1), np.int32)
        weights = bilateral_weights()
        L, h = self.handle.L, self.handle.h
        _lib.check(L.osfm_dense_estimate(h, len(refs), _lib.ptr(start), _lib.ptr(flat), _lib.ptr(Q), _lib.ptr(A),
                                         _lib.ptr(params), _lib.ptr(rng), _lib.ptr(var), _lib.ptr(weights),
                                         int(seed) & 0xFFFFFFFF, float(min_score), _lib.ptr(depth), _lib.ptr(plane),
                                         _lib.ptr(score), _lib.ptr(nghbr)))
        out = Depthmaps(device_ms=self.last_device_ms()[0])
        o = 0
        for (hh, ww) in sizes:
            n = hh * ww
            out.depth.append(depth[o:o + n].reshape(hh, ww))
            out.plane.append(plane[3 * o:3 * (o + n)].reshape(hh, ww, 3))
            out.score.append(score[o:o + n].reshape(hh, ww))
            out.nghbr.append(nghbr[o:o + n].reshape(hh, ww))
            o += n
        return out

    def clean(self, lists: Sequence[Sequence[int]], same_depth_threshold: float = 0.01,
              min_consistent_views: int = 2) -> List[np.ndarray]:
        start, flat = _lists(lists, key=lambda x: x)
        sizes = [self._shape(lst[0]) if 0 <= lst[0] < len(self.views) else (0, 0) for lst in lists]
        out = np.zeros(max(sum(h * w for h, w in sizes), 1), np.float32)
        _lib.check(self.handle.L.osfm_dense_clean(self.handle.h, len(lists), _lib.ptr(start), _lib.ptr(flat),
                                                  same_depth_threshold, int(min_consistent_views), _lib.ptr(out)))
        res, o = [], 0
        for hh, ww in sizes:
            res.append(out[o:o + hh * ww].reshape(hh, ww))
            o += hh * ww
        return res

    def prune(self, lists: Sequence[Sequence[int]], same_depth_threshold: float = 0.01):
        """Per reference, pydense's (points, normals, colors, labels)."""
        start, flat = _lists(lists, key=lambda x: x)
        counts = np.zeros(max(len(lists), 1), np.int64)
        L, h = self.handle.L, self.handle.h
        _lib.check(L.osfm_dense_prune(h, len(lists), _lib.ptr(start), _lib.ptr(flat), same_depth_threshold,
                                      _lib.ptr(counts)))
        n = int(counts[:len(lists)].sum())
        pts, nrm = np.zeros((max(n, 1), 3), np.float32), np.zeros((max(n, 1), 3), np.float32)
        col, lab = np.zeros((max(n, 1), 3), np.uint8), np.zeros(max(n, 1), np.uint8)
        _lib.check(L.osfm_dense_get_pruned(h, _lib.ptr(pts), _lib.ptr(nrm), _lib.ptr(col), _lib.ptr(lab)))
        res, o = [], 0
        for c in counts[:len(lists)].tolist():
            res.append((pts[o:o + c], nrm[o:o + c], col[o:o + c], lab[o:o + c]))
            o += c
        return res

    def last_device_ms(self) -> Tuple[float, float, float]:
        e, c, p = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
        _lib.check(self.handle.L.osfm_dense_last_device_ms(self.handle.h, ctypes.byref(e), ctypes.byref(c),
                                                           ctypes.byref(p)))
        return e.value, c.value, p.value


def depthmaps(views: Sequence[View], refs: Sequence[Reference], min_score: float, same_depth_threshold: float,
              min_consistent_views: int, seed: int = 0, device: int = 0):
    """Every reference estimated in one submission, then cleaned in one over every view of its list with a raw map,
    then pruned in one over every view with a clean map; nothing leaves the device in between.  Returns the ungated
    estimates, the clean depths and the pruned arrays per reference, and the device ms per stage."""
    with Engine(views, device) as E:
        est = E.estimate(refs, seed, min_score)
        have = [v.raw_depth is not None and v.plane is not None for v in views]
        for r in refs:
            have[r.views[0]] = True
        lists = [[v for v in r.views if have[v]] for r in refs]
        clean = E.clean(lists, same_depth_threshold, min_consistent_views)
        pruned = E.prune(lists, same_depth_threshold)
        return est, clean, pruned, E.last_device_ms()


# ---- pydense's classes --------------------------------------------------------------------------------------------


class DepthmapEstimator:
    """pydense.DepthmapEstimator.  seed and key select the generator's stream (see the module docstring)."""

    def __init__(self, seed: int = 0, device: int = 0, key: int = 0):
        self.views: List[View] = []
        self.patch_size, self.min_depth, self.max_depth = 7, 0.0, 0.0
        self.num_depth_planes, self.patchmatch_iterations = 50, 3
        self.min_patch_sd = 5.0
        self.seed, self.device, self.key = seed, device, key

    def set_depth_range(self, min_depth, max_depth, num_depth_planes):
        self.min_depth, self.max_depth, self.num_depth_planes = float(min_depth), float(max_depth), int(num_depth_planes)

    def set_patchmatch_iterations(self, n):
        self.patchmatch_iterations = int(n)

    def set_patch_size(self, size):
        self.patch_size = int(size)

    def set_min_patch_sd(self, sd):
        self.min_patch_sd = float(sd)

    def add_view(self, K, R, t, image, mask):
        image = np.asarray(image)
        if image.ndim != 2:
            raise ValueError("image must be a gray (h, w) array")
        h, w = image.shape
        self.views.append(View(K=np.asarray(K, np.float64), R=np.asarray(R, np.float64), t=np.asarray(t, np.float64),
                               width=w, height=h, gray=_u8(image, (h, w), "image"),
                               mask=_u8(mask, (h, w), "mask")))

    def _compute(self, method):
        ref = Reference(views=list(range(len(self.views))), min_depth=self.min_depth, max_depth=self.max_depth,
                        method=method, patch_size=self.patch_size, num_depth_planes=self.num_depth_planes,
                        patchmatch_iterations=self.patchmatch_iterations, min_patch_sd=self.min_patch_sd,
                        key=self.key)
        with Engine(self.views, self.device) as E:
            m = E.estimate([ref], self.seed)
        return [m.depth[0], m.plane[0], m.score[0], m.nghbr[0]]

    def compute_patch_match(self):
        return self._compute("PATCH_MATCH")

    def compute_patch_match_sample(self):
        return self._compute("PATCH_MATCH_SAMPLE")

    def compute_brute_force(self):
        return self._compute("BRUTE_FORCE")


class DepthmapCleaner:
    def __init__(self, device: int = 0):
        self.views: List[View] = []
        self.same_depth_threshold, self.min_consistent_views = 0.01, 2
        self.device = device

    def set_same_depth_threshold(self, t):
        self.same_depth_threshold = float(t)

    def set_min_consistent_views(self, n):
        self.min_consistent_views = int(n)

    def add_view(self, K, R, t, depth):
        depth = np.asarray(depth, np.float32)
        h, w = depth.shape
        self.views.append(View(K=np.asarray(K, np.float64), R=np.asarray(R, np.float64), t=np.asarray(t, np.float64),
                               width=w, height=h, raw_depth=depth, plane=np.zeros((h, w, 3), np.float32)))

    def clean(self):
        with Engine(self.views, self.device) as E:
            return E.clean([list(range(len(self.views)))], self.same_depth_threshold, self.min_consistent_views)[0]


class DepthmapPruner:
    def __init__(self, device: int = 0):
        self.views: List[View] = []
        self.same_depth_threshold = 0.01
        self.device = device

    def set_same_depth_threshold(self, t):
        self.same_depth_threshold = float(t)

    def add_view(self, K, R, t, depth, plane, color, labels):
        depth = np.asarray(depth, np.float32)
        h, w = depth.shape
        self.views.append(View(K=np.asarray(K, np.float64), R=np.asarray(R, np.float64), t=np.asarray(t, np.float64),
                               width=w, height=h, plane=_f32(plane, (h, w, 3), "plane"),
                               color=_u8(color, (h, w, 3), "color"), labels=_u8(labels, (h, w), "labels"),
                               clean_depth=depth))

    def prune(self):
        with Engine(self.views, self.device) as E:
            return list(E.prune([list(range(len(self.views)))], self.same_depth_threshold)[0])


# ---- opensfm/dense.py: the driver and its host helpers --------------------------------------------------------------

logger = logging.getLogger(__name__)


def shot_key(shot_id: str) -> int:
    """The generator key of a shot in `compute_depthmaps`: CRC-32 of its id, so a shot draws the same variates
    whatever else is computed with it."""
    return zlib.crc32(str(shot_id).encode("utf-8"))


def angle_between_points(origin, p1, p2):
    """The angle at `origin` between p1 and p2; the arrays may carry leading dimensions (opensfm/dense.py)."""
    origin, p1, p2 = (np.asarray(x, dtype=np.float64) for x in (origin, p1, p2))
    a0, a1, a2 = p1[..., 0] - origin[..., 0], p1[..., 1] - origin[..., 1], p1[..., 2] - origin[..., 2]
    b0, b1, b2 = p2[..., 0] - origin[..., 0], p2[..., 1] - origin[..., 1], p2[..., 2] - origin[..., 2]
    dot = a0 * b0 + a1 * b1 + a2 * b2
    la = a0 * a0 + a1 * a1 + a2 * a2
    lb = b0 * b0 + b1 * b1 + b2 * b2
    return np.arccos(dot / np.sqrt(la * lb))


def common_tracks_double_dict(tracks_manager) -> Dict[Any, Dict[Any, List[str]]]:
    """res[im1][im2]: the tracks of every image pair with at least 50 in common, from this engine's TracksManager
    (its device pair lists) or from pymap's (through its shot observations)."""
    from . import tracking

    if isinstance(tracks_manager, tracking.TracksManager):
        pairs = tracking.all_common_tracks_without_features(tracks_manager)
    else:
        shots = tracks_manager.get_shot_ids()
        seen: Dict[str, List[Any]] = {}
        for s in shots:
            for t in tracks_manager.get_shot_observations(s):
                seen.setdefault(t, []).append(s)
        acc: Dict[Tuple[Any, Any], List[str]] = {}
        for t, ss in seen.items():
            for x in range(len(ss)):
                for y in range(x + 1, len(ss)):
                    acc.setdefault((ss[x], ss[y]), []).append(t)
        pairs = {k: v for k, v in acc.items() if len(v) >= 50}
    res: Dict[Any, Dict[Any, List[str]]] = {image: {} for image in tracks_manager.get_shot_ids()}
    for (im1, im2), v in pairs.items():
        res[im1][im2] = v
        res[im2][im1] = v
    return res


def find_neighboring_images(shot, common_tracks, reconstruction, num_neighbors: int) -> list:
    """The shot followed by its best `num_neighbors` neighbours by the number of common reconstructed tracks seen at
    an angle in (pi/60, pi/6), with more than 20 of them (opensfm/dense.py); the angles of a pair in one pass."""
    theta_min, theta_max = np.pi / 60, np.pi / 6
    ns = []
    C1 = shot.pose.get_origin()
    points = reconstruction.points
    for other_id, tracks in common_tracks.get(shot.id, {}).items():
        if other_id not in reconstruction.shots:
            continue
        other = reconstruction.shots[other_id]
        C2 = other.pose.get_origin()
        P = np.array([points[t].coordinates for t in tracks if t in points], dtype=np.float64).reshape(-1, 3)
        theta = angle_between_points(P, C1, C2) if len(P) else np.zeros(0)
        score = int(np.count_nonzero((theta > theta_min) & (theta < theta_max)))
        if score > 20:
            ns.append((other, score))
    ns.sort(key=lambda ns: ns[1], reverse=True)
    return [shot] + [n for n, s in ns[:num_neighbors]]


def compute_depth_range(tracks_manager, reconstruction, shot, config) -> Tuple[float, float]:
    """10th percentile x 0.9 and 90th x 1.1 of the depths of the shot's reconstructed tracks, unless the config sets
    them (opensfm/dense.py); the depths in one pass."""
    points = reconstruction.points
    P = np.array([points[t].coordinates for t in tracks_manager.get_shot_observations(shot.id) if t in points],
                 dtype=np.float64).reshape(-1, 3)
    R = shot.pose.get_rotation_matrix()
    tz = shot.pose.translation[2]
    depths = R[2, 0] * P[:, 0] + R[2, 1] * P[:, 1] + R[2, 2] * P[:, 2] + tz
    min_depth = np.percentile(depths, 10) * 0.9
    max_depth = np.percentile(depths, 90) * 1.1
    return config["depthmap_min_depth"] or min_depth, config["depthmap_max_depth"] or max_depth


def _ply_header(count_vertices: int, with_normals: bool = False) -> List[str]:
    """io.ply_header (without the number of views)."""
    header = ["ply", "format ascii 1.0", "element vertex {}".format(count_vertices),
              "property float x", "property float y", "property float z"]
    if with_normals:
        header += ["property float nx", "property float ny", "property float nz"]
    return header + ["property uchar red", "property uchar green", "property uchar blue", "end_header"]


def depthmap_to_ply(shot, depth: np.ndarray, image: np.ndarray) -> str:
    """The non-zero pixels of a depthmap as a PLY string (opensfm/dense.py)."""
    height, width = depth.shape
    K = shot.camera.get_K_in_pixel_coordinates(width, height)
    R = shot.pose.get_rotation_matrix()
    t = shot.pose.translation
    y, x = np.mgrid[:height, :width]
    v = np.vstack((x.ravel(), y.ravel(), np.ones(width * height)))
    camera_coords = depth.reshape((1, -1)) * np.linalg.inv(K).dot(v)
    points = R.T.dot(camera_coords - np.asarray(t).reshape(3, 1))
    vertices = []
    for p, c, d in zip(points.T, image.reshape(-1, 3), depth.reshape(-1, 1)):
        if d != 0:
            vertices.append("{} {} {} {} {} {}".format(p[0], p[1], p[2], c[0], c[1], c[2]))
    return "\n".join(_ply_header(len(vertices)) + vertices + [""])


def aggregate_depthmaps(shot_ids: Iterable[str], depthmap_provider: Callable[[str], Tuple]) -> Tuple:
    points, normals, colors, labels = [], [], [], []
    for shot_id in shot_ids:
        p, n, c, l = depthmap_provider(shot_id)
        points.append(p)
        normals.append(n)
        colors.append(c)
        labels.append(l)
    return np.concatenate(points), np.concatenate(normals), np.concatenate(colors), np.concatenate(labels)


def merge_depthmaps_from_provider(shot_ids: Iterable[str], depthmap_provider: Callable[[str], Tuple]) -> Tuple:
    if not shot_ids:
        logger.warning("Depthmaps contain no points.  Try using more images.")
        return np.array([]), np.array([]), np.array([]), np.array([])
    return aggregate_depthmaps(shot_ids, depthmap_provider)


def merge_depthmaps(data, reconstruction) -> Tuple:
    shot_ids = [s for s in reconstruction.shots if data.pruned_depthmap_exists(s)]
    return merge_depthmaps_from_provider(shot_ids, data.load_pruned_depthmap)


def scale_down_image(image, width, height, interpolation=None):
    import cv2

    width, height = min(width, image.shape[1]), min(height, image.shape[0])
    return cv2.resize(image, (width, height), interpolation=cv2.INTER_AREA if interpolation is None else interpolation)


def _load_view(data, shot, resolution: int) -> View:
    """A shot's images at depthmap resolution, as add_views_to_depth_estimator / _pruner load them."""
    import cv2

    assert shot.camera.projection_type == "perspective"
    color = data.load_undistorted_image(shot.id)
    gray = cv2.cvtColor(color, cv2.COLOR_RGB2GRAY)
    oh, ow = gray.shape
    width = min(ow, int(resolution))
    height = width * oh // ow
    image = scale_down_image(gray, width, height)
    mask = data.load_undistorted_combined_mask(shot.id)
    if mask is None:
        mask = np.ones((int(shot.camera.height), int(shot.camera.width)), dtype=np.uint8)
    mask = cv2.resize(mask, (image.shape[1], image.shape[0]), interpolation=cv2.INTER_NEAREST)
    if data.undistorted_segmentation_exists(shot.id):
        labels = data.load_undistorted_segmentation(shot.id)
    else:
        labels = np.zeros((shot.camera.height, shot.camera.width), dtype=np.uint8)
    h, w = image.shape
    rgb = scale_down_image(color, w, h)
    labels = cv2.resize(labels, (rgb.shape[1], rgb.shape[0]), interpolation=cv2.INTER_NEAREST)
    return View(K=shot.camera.get_K_in_pixel_coordinates(w, h), R=shot.pose.get_rotation_matrix(),
                t=np.asarray(shot.pose.translation, np.float64), width=w, height=h, gray=image, mask=mask,
                color=rgb, labels=labels)


def compute_depthmaps(data, tracks_manager, reconstruction, device: int = 0, seed: int = 0) -> None:
    """opensfm.dense.compute_depthmaps on the GPU: the same steps, files and reuse of existing maps, with every shot
    estimated in one submission, then cleaned in one and pruned in one.  Shot s draws from the stream of key
    shot_key(s.id).  `interactive` is not supported.  Raises RuntimeError naming the bytes needed when the views and
    maps do not fit in device memory."""
    config = data.config
    if config.get("interactive"):
        raise NotImplementedError("compute_depthmaps: interactive display is not supported")
    common = common_tracks_double_dict(tracks_manager)
    neighbors = {s.id: find_neighboring_images(s, common, reconstruction, config["depthmap_num_neighbors"])
                 for s in reconstruction.shots.values()}
    shots = [s for s in reconstruction.shots.values() if len(neighbors[s.id]) > 1]
    if not shots:
        data.save_point_cloud(*merge_depthmaps(data, reconstruction), filename="merged.ply")
        return
    debug = config["depthmap_save_debug_files"]
    num_matching = config["depthmap_num_matching_views"]

    index: Dict[str, int] = {}
    views: List[View] = []
    raw_score: Dict[str, np.ndarray] = {}
    for s in shots:
        for n in neighbors[s.id]:
            if n.id in index:
                continue
            v = _load_view(data, n, config["depthmap_resolution"])
            if data.raw_depthmap_exists(n.id):
                d, p, sc, _, _ = data.load_raw_depthmap(n.id)
                v.raw_depth, v.plane, raw_score[n.id] = d, p, sc
            if data.clean_depthmap_exists(n.id):
                v.clean_depth, v.plane = data.load_clean_depthmap(n.id)[:2]
            index[n.id] = len(views)
            views.append(v)

    with Engine(views, device) as E:
        todo = [s for s in shots if not data.raw_depthmap_exists(s.id)]
        refs = []
        for s in todo:
            mind, maxd = compute_depth_range(tracks_manager, reconstruction, s, config)
            maxd = np.float64(maxd)   # the gate compares depth < max_depth in fp64, on the device as here
            refs.append(Reference([index[n.id] for n in neighbors[s.id][:num_matching + 1]], mind, maxd,
                                  config["depthmap_method"], config["depthmap_patch_size"], 100,
                                  config["depthmap_patchmatch_iterations"], config["depthmap_min_patch_sd"],
                                  key=shot_key(s.id)))
        if any(r.method not in METHODS for r in refs):
            raise ValueError("Unknown depthmap method type (must be BRUTE_FORCE, PATCH_MATCH or PATCH_MATCH_SAMPLE)")
        est = E.estimate(refs, seed, config["depthmap_min_correlation_score"]) if refs else Depthmaps()
        for k, (s, r) in enumerate(zip(todo, refs)):
            good = est.score[k] > config["depthmap_min_correlation_score"]
            depth = est.depth[k] * (est.depth[k] < r.max_depth) * good
            views[index[s.id]].raw_depth, views[index[s.id]].plane = depth, est.plane[k]
            raw_score[s.id] = est.score[k]
            data.save_raw_depthmap(s.id, depth, est.plane[k], est.score[k], est.nghbr[k],
                                   [n.id for n in neighbors[s.id][1:]])
            if debug:
                with open(data.depthmap_file(s.id, "raw.npz.ply"), "w") as f:
                    f.write(depthmap_to_ply(s, depth, views[index[s.id]].color))

        has_raw = {sid: views[i].raw_depth is not None for sid, i in index.items()}
        clean_todo = [s for s in shots if not data.clean_depthmap_exists(s.id) and has_raw[s.id]]
        lists = [[index[n.id] for n in neighbors[s.id] if has_raw[n.id]] for s in clean_todo]
        cleaned = E.clean(lists, config["depthmap_same_depth_threshold"],
                          config["depthmap_min_consistent_views"]) if lists else []
        for s, depth in zip(clean_todo, cleaned):
            v = views[index[s.id]]
            v.clean_depth = depth
            data.save_clean_depthmap(s.id, depth, v.plane, raw_score[s.id])
            if debug:
                with open(data.depthmap_file(s.id, "clean.npz.ply"), "w") as f:
                    f.write(depthmap_to_ply(s, depth, v.color))

        has_clean = {sid: views[i].clean_depth is not None for sid, i in index.items()}
        prune_todo = [s for s in shots if not data.pruned_depthmap_exists(s.id) and has_clean[s.id]]
        lists = [[index[n.id] for n in neighbors[s.id] if has_clean[n.id]] for s in prune_todo]
        pruned = E.prune(lists, config["depthmap_same_depth_threshold"]) if lists else []
        for s, (points, normals, colors, labels) in zip(prune_todo, pruned):
            data.save_pruned_depthmap(s.id, points, normals, colors, labels)
            if debug:
                data.save_point_cloud(points, normals, colors, labels, "pruned.npz.ply")

    data.save_point_cloud(*merge_depthmaps(data, reconstruction), filename="merged.ply")
