"""Synthetic scenes of BASELINE.json's configs, restated in numpy.

The reference's generators (`opensfm/synthetic_data/synthetic_scene.py:88-145`
SyntheticCubeScene, `synthetic_generator.py:364-471` generate_track_data) need
`pymap`/`pygeometry`, which cannot be built in this image.  This module restates
their sampling with the same constants and the same order of `np.random` draws,
and emits the SoA arrays the engine consumes (SURVEY.md §8d):

* cameras: per camera phi = U*pi, theta = U*2pi, position r=2 on the sphere,
  alpha = U, look-at origin with up = (0.2a, 0.2a, 1) (synthetic_scene.py:103-120,
  camera_pose :57-80); perspective f=0.9, k1=-0.1, k2=0.01, 800x600, one camera
  per shot (:94-99);
* points: U(0,1)^3 - 0.5 (:122);
* descriptors: 128-D float32 zeros with 5 random slots = round(U*255)
  (synthetic_generator.py:385-397);
* observations: projections inside the frame and in front of the camera
  (:433-439,508-523) plus N(0, (noise/800)^2), sigma 0.004 (:404).

Everything here is host-side fixture generation; it is not on the hot path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import ba_problem as bp


def _normalized(x):
    return x / np.linalg.norm(x)


def rotation_to_angle_axis(R: np.ndarray) -> np.ndarray:
    """Angle-axis vector of a rotation matrix (host-side helper, fp64)."""
    from scipy.spatial.transform import Rotation

    return Rotation.from_matrix(R).as_rotvec()


def angle_axis_to_rotation(r: np.ndarray) -> np.ndarray:
    from scipy.spatial.transform import Rotation

    return Rotation.from_rotvec(r).as_matrix()


def camera_pose(position, lookat, up) -> Tuple[np.ndarray, np.ndarray]:
    """World->camera rotation rows (ex, ey, ez) and origin (synthetic_scene.py:57-80)."""
    ez = _normalized(np.array(lookat) - np.array(position))
    ex = _normalized(np.cross(ez, up))
    ey = _normalized(np.cross(ez, ex))
    return np.array([ex, ey, ez]), np.array(position, dtype=np.float64)


def pose_to_params(R_wc: np.ndarray, origin: np.ndarray) -> np.ndarray:
    """[angle-axis of R(camera->world) | origin] (bundle/data/pose.h:34-43)."""
    return np.concatenate([rotation_to_angle_axis(R_wc.T), origin])


def project_perspective(points_cam: np.ndarray, k1: float, k2: float, focal: float) -> np.ndarray:
    """Perspective + Disto24 + UniformScale (camera_instances.h:181-182) for fixture generation."""
    x = points_cam[:, 0] / points_cam[:, 2]
    y = points_cam[:, 1] / points_cam[:, 2]
    r2 = x * x + y * y
    d = 1.0 + r2 * (k1 + k2 * r2)
    return np.stack([focal * x * d, focal * y * d], axis=1)


@dataclass
class SyntheticScene:
    R_wc: np.ndarray            # (S,3,3) world->camera rotations
    origins: np.ndarray         # (S,3)
    points: np.ndarray          # (P,3)
    cam_params: np.ndarray      # (S,3) [k1,k2,focal] per camera
    obs_shot: np.ndarray        # (N,)
    obs_point: np.ndarray       # (N,)
    obs_xy: np.ndarray          # (N,2) noisy normalised image coordinates
    obs_sigma: np.ndarray       # (N,)
    track_descriptors: Optional[np.ndarray] = None  # (P,128) float32
    width: int = 800
    height: int = 600

    @property
    def num_shots(self) -> int:
        return len(self.origins)

    def features_of_shot(self, s: int) -> Tuple[np.ndarray, np.ndarray]:
        """(descriptor matrix rows of visible points, their point ids) of one image."""
        sel = np.nonzero(self.obs_shot == s)[0]
        pts = self.obs_point[sel]
        return self.track_descriptors[pts], pts


def _inside(proj: np.ndarray, width: int, height: int) -> np.ndarray:
    w, h = float(width), float(height)
    if w > h:
        return (np.abs(proj[:, 0]) < 0.5) & (np.abs(proj[:, 1]) < h / (2 * w))
    return (np.abs(proj[:, 1]) < 0.5) & (np.abs(proj[:, 0]) < w / (2 * h))


def cube_scene(num_cameras: int, num_points: int, projection_noise: float = 1.0, seed: int = 42,
               with_descriptors: bool = True, max_obs_per_point: Optional[int] = None,
               maximum_depth: float = 40.0) -> SyntheticScene:
    """SyntheticCubeScene + generate_track_data, restated (see module docstring).

    max_obs_per_point: BASELINE config 4 thins visibility to the N cameras whose view axis is
    closest to the point direction (SURVEY.md §8d) — deterministic, not in the reference.
    """
    rng = np.random.RandomState(seed)  # same stream as np.random.seed(seed) + global draws
    r = 2.0
    R_wc = np.zeros((num_cameras, 3, 3))
    origins = np.zeros((num_cameras, 3))
    for i in range(num_cameras):
        phi = rng.rand() * math.pi
        theta = rng.rand() * 2.0 * math.pi
        position = np.array([r * np.sin(theta) * np.cos(phi), r * np.sin(theta) * np.sin(phi), r * np.cos(theta)])
        alpha = rng.rand()
        up = np.array([alpha * 0.2, alpha * 0.2, 1.0])
        R_wc[i], origins[i] = camera_pose(position, [0.0, 0.0, 0.0], up)
    points = rng.rand(num_points, 3) - [0.5, 0.5, 0.5]
    k1, k2, focal = -0.1, 0.01, 0.9
    cam_params = np.tile(np.array([k1, k2, focal]), (num_cameras, 1))

    desc = None
    if with_descriptors:
        desc = np.zeros((num_points, 128), dtype=np.float64)
        if num_points <= 20000:
            # 5 x (randint, random) per point, in this order (synthetic_generator.py:391-397)
            for p in range(num_points):
                for _ in range(5):
                    index = rng.randint(0, 128)
                    desc[p, index] = rng.random_sample() * 255
        else:
            # same distribution, vectorised draws (the large scenes have no reference sequence to follow)
            idx = rng.randint(0, 128, (num_points, 5))
            val = rng.random_sample((num_points, 5)) * 255
            for k in range(5):
                desc[np.arange(num_points), idx[:, k]] = val[:, k]
        desc = desc.round().astype(np.float32)

    if max_obs_per_point is not None:
        return _cube_scene_thinned(rng, R_wc, origins, points, cam_params, desc, projection_noise,
                                   max_obs_per_point, maximum_depth)

    width, height = 800, 600
    perturbation = float(projection_noise) / float(max(width, height))
    obs_shot: List[np.ndarray] = []
    obs_point: List[np.ndarray] = []
    obs_xy: List[np.ndarray] = []
    vis_score: List[np.ndarray] = []
    for s in range(num_cameras):
        d = points - origins[s]
        near = np.nonzero(np.linalg.norm(d, axis=1) <= maximum_depth)[0]  # sorted ball query
        pc = d[near] @ R_wc[s].T
        proj = project_perspective(pc, k1, k2, focal)
        noise = rng.normal(0.0, perturbation, (len(near), 2)) if perturbation > 0 else np.zeros((len(near), 2))
        ok = _inside(proj, width, height) & (pc[:, 2] > 0)
        ids = near[ok]
        obs_shot.append(np.full(len(ids), s, dtype=np.int32))
        obs_point.append(ids.astype(np.int32))
        obs_xy.append(proj[ok] + noise[ok])
        # cosine between the view axis and the point direction (for thinning)
        vis_score.append(pc[ok, 2] / np.linalg.norm(pc[ok], axis=1))
    o_s = np.concatenate(obs_shot)
    o_p = np.concatenate(obs_point)
    o_xy = np.concatenate(obs_xy)
    score = np.concatenate(vis_score)
    if max_obs_per_point is not None:
        # keep, per point, the max_obs_per_point observations with the largest cosine
        order = np.lexsort((-score, o_p))
        o_s, o_p, o_xy, score = o_s[order], o_p[order], o_xy[order], score[order]
        start = np.searchsorted(o_p, np.arange(num_points), side="left")
        rank = np.arange(len(o_p)) - start[o_p]
        keep = rank < max_obs_per_point
        o_s, o_p, o_xy = o_s[keep], o_p[keep], o_xy[keep]
        order = np.lexsort((o_p, o_s))  # back to shot-major order
        o_s, o_p, o_xy = o_s[order], o_p[order], o_xy[order]
    return SyntheticScene(R_wc=R_wc, origins=origins, points=points, cam_params=cam_params, obs_shot=o_s,
                          obs_point=o_p, obs_xy=o_xy, obs_sigma=np.full(len(o_s), 0.004),
                          track_descriptors=desc, width=width, height=height)


def _cube_scene_thinned(rng, R_wc, origins, points, cam_params, desc, projection_noise, max_obs, maximum_depth,
                        width=800, height=600, chunk=20000) -> SyntheticScene:
    """Visibility thinned to the `max_obs` cameras whose view axis is closest to the point
    direction (largest cosine), chunked over points so the 500 x 200k scene fits in memory.
    Fixture generation only: uses torch (fp64; on the GPU when one is present) for the
    S x P visibility sweep."""
    import torch

    dev = torch.device("cuda" if torch.cuda.is_available() else "cpu")
    S, P = len(origins), len(points)
    k1, k2, focal = (float(v) for v in cam_params[0])
    perturbation = float(projection_noise) / float(max(width, height))
    R = torch.from_numpy(R_wc).to(dev)
    O = torch.from_numpy(origins).to(dev)
    A = R.reshape(S * 3, 3)
    Ao = torch.einsum("sij,sj->si", R, O).reshape(S * 3, 1)
    o2 = (O * O).sum(1)[:, None]
    kk = min(max_obs, S)
    o_s, o_p, o_xy = [], [], []
    for c0 in range(0, P, chunk):
        pts = torch.from_numpy(points[c0:c0 + chunk]).to(dev)
        n = pts.shape[0]
        pc = (A @ pts.T - Ao).reshape(S, 3, n)
        dist = torch.sqrt(torch.clamp((pts * pts).sum(1)[None, :] - 2.0 * (O @ pts.T) + o2, min=0.0))
        z = pc[:, 2, :]
        x = pc[:, 0, :] / z
        y = pc[:, 1, :] / z
        r2 = x * x + y * y
        dd = 1.0 + r2 * (k1 + k2 * r2)
        px, py = focal * x * dd, focal * y * dd
        ok = (z > 0) & (dist <= maximum_depth) & (px.abs() < 0.5) & (py.abs() < height / (2.0 * width))
        score = torch.where(ok, z / dist, torch.full_like(z, -float("inf")))
        # ties broken by camera index (stable sort) so the selection is deterministic
        order = torch.sort(-score, dim=0, stable=True).indices[:kk]      # kk x n camera ids
        cols = torch.arange(n, device=dev)[None, :].expand(kk, n)
        keep = torch.isfinite(score[order, cols])
        cams = order[keep]
        pidx = cols[keep]
        o_s.append(cams.to(torch.int32).cpu().numpy())
        o_p.append((pidx + c0).to(torch.int32).cpu().numpy())
        o_xy.append(torch.stack([px[cams, pidx], py[cams, pidx]], dim=1).cpu().numpy())
    o_s = np.concatenate(o_s)
    o_p = np.concatenate(o_p)
    o_xy = np.concatenate(o_xy)
    order = np.lexsort((o_p, o_s))  # shot-major, like the reference's per-shot loop
    o_s, o_p, o_xy = o_s[order], o_p[order], o_xy[order]
    if perturbation > 0:
        o_xy = o_xy + rng.normal(0.0, perturbation, o_xy.shape)
    return SyntheticScene(R_wc=R_wc, origins=origins, points=points, cam_params=cam_params, obs_shot=o_s,
                          obs_point=o_p, obs_xy=o_xy, obs_sigma=np.full(len(o_s), 0.004),
                          track_descriptors=desc, width=width, height=height)


def scene_to_problem(scene: SyntheticScene, perturb_seed: Optional[int] = 43, point_noise: float = 0.01,
                     position_noise: float = 0.02, rotation_noise: float = 0.01,
                     shared_intrinsics: bool = False, optimize_cameras: bool = True,
                     loss_name: str = "SoftLOneLoss", loss_threshold: float = 1.0,
                     max_iterations: int = 100, drop_unobserved: bool = True) -> bp.BAProblem:
    """BA start = ground truth perturbed (SURVEY.md §8d: points N(0,0.01^2), positions
    N(0,0.02^2), rotations N(0,0.01^2) rad, seed 43); config defaults of
    opensfm/config.py:241-245,283 (SoftLOneLoss 1, 100 iterations)."""
    S = scene.num_shots
    inst = np.stack([pose_to_params(scene.R_wc[i], scene.origins[i]) for i in range(S)])
    points = scene.points.copy()
    obs_point = scene.obs_point
    if drop_unobserved:
        # landmarks without observations never enter a reconstruction
        seen = np.zeros(len(points), dtype=bool)
        seen[obs_point] = True
        remap = np.cumsum(seen) - 1
        points = points[seen]
        obs_point = remap[obs_point].astype(np.int32)
    if perturb_seed is not None:
        rng = np.random.RandomState(perturb_seed)
        points = points + rng.normal(0.0, point_noise, points.shape)
        inst = inst.copy()
        inst[:, 3:] += rng.normal(0.0, position_noise, (S, 3))
        inst[:, :3] += rng.normal(0.0, rotation_noise, (S, 3))
    if shared_intrinsics:
        cam_type = [bp.PERSPECTIVE]
        cam_params = [scene.cam_params[0]]
        shot_cam = np.zeros(S, dtype=np.int32)
    else:
        cam_type = [bp.PERSPECTIVE] * S
        cam_params = [scene.cam_params[i] for i in range(S)]
        shot_cam = np.arange(S, dtype=np.int32)
    return bp.make_problem(
        cam_type, cam_params, inst, points, scene.obs_shot, obs_point, scene.obs_xy, scene.obs_sigma,
        shot_cam=shot_cam, cam_const=None if optimize_cameras else np.ones(len(cam_type), dtype=np.int32),
        # config.py:247-263 defaults of the prior sds
        prior_sd=dict(focal_sd=0.01, aspect_ratio_sd=0.01, c_sd=0.01, k1_sd=0.01, k2_sd=0.01, p1_sd=0.01,
                      p2_sd=0.01, k3_sd=0.01, k4_sd=0.01),
        loss_name=loss_name, loss_threshold=loss_threshold, max_iterations=max_iterations)


def hahog_like_descriptors(n: int, seed: int, dim: int = 128) -> np.ndarray:
    """Integer-valued float32 descriptors as HAHOG stores them: (362*sqrt(x)).clip(0,255).round()
    of an L1-normalised non-negative histogram (opensfm/features.py:526-534), loaded as float32
    (features.py:169-170)."""
    rng = np.random.RandomState(seed)
    h = rng.gamma(0.6, 1.0, (n, dim))
    h /= h.sum(axis=1, keepdims=True)
    return (362.0 * np.sqrt(h)).clip(0, 255).round().astype(np.float32)


def binary_descriptors(n: int, seed: int, nbytes: int = 61) -> np.ndarray:
    """AKAZE-MLDB-sized (486 bit -> 61 byte) random binary descriptors."""
    rng = np.random.RandomState(seed)
    return rng.randint(0, 256, (n, nbytes)).astype(np.uint8)


def guided_scene(n_images: int, n_desc: int, seed: int = 7, bearing_noise: float = 0.002, dim: int = 128):
    """Stand-in for BASELINE configs[2] (lund sequence, HAHOG features, guided matching; SURVEY.md 8d): `n_images`
    cameras on an arc looking at a point cloud, each with `n_desc` features = bearings of points it sees (+ angular
    noise) and HAHOG-like uint8-valued descriptors (the point's descriptor + small integer noise).
    Returns (descriptors [n_images] float32 n_desc x dim, bearings [n_images] float32 n_desc x 3,
    R_wc [n_images] 3x3 world->camera, origins [n_images])."""
    rng = np.random.RandomState(seed)
    n_points = int(n_desc * 1.6)
    pts = rng.uniform(-1.0, 1.0, (n_points, 3)) * np.array([2.0, 1.0, 1.0])
    base = hahog_like_descriptors(n_points, seed + 1, dim)
    descs, bears, Rs, Os = [], [], [], []
    for i in range(n_images):
        ang = -0.6 + 1.2 * i / max(n_images - 1, 1)
        origin = np.array([4.0 * np.sin(ang), 0.3 * np.sin(3 * ang), -4.0 * np.cos(ang)])
        R_wc, _ = camera_pose(origin, np.zeros(3), np.array([0.0, -1.0, 0.0]))
        idx = rng.choice(n_points, n_desc, replace=False)
        xc = (pts[idx] - origin) @ R_wc.T
        b = xc / np.linalg.norm(xc, axis=1, keepdims=True)
        b = b + rng.normal(0.0, bearing_noise, b.shape)
        b /= np.linalg.norm(b, axis=1, keepdims=True)
        d = np.clip(base[idx] + rng.randint(-4, 5, (n_desc, dim)), 0, 255).astype(np.float32)
        descs.append(d); bears.append(b.astype(np.float32)); Rs.append(R_wc); Os.append(origin)
    return descs, bears, Rs, Os


def relative_pose(R_wc_a, origin_a, R_wc_b, origin_b):
    """(R, t) of image b relative to image a as matching.py passes them to the epipolar mask:
    R = rotation camera b -> camera a, t = origin of camera b in camera a's frame."""
    R = R_wc_a @ R_wc_b.T
    t = R_wc_a @ (np.asarray(origin_b) - np.asarray(origin_a))
    return R, t


@dataclass
class TexturedScene:
    """Images and exact depth maps of a piecewise-planar scene, in OpenSfM's conventions: x_cam = R X + t, pixel
    coordinates through K, depth = z_cam (0 where a ray hits nothing)."""
    K: np.ndarray        # (S,3,3)
    R: np.ndarray        # (S,3,3)
    t: np.ndarray        # (S,3)
    gray: np.ndarray     # (S,H,W) u8
    rgb: np.ndarray      # (S,H,W,3) u8
    depth: np.ndarray    # (S,H,W) f32
    flat: np.ndarray     # (S,H,W) bool: the flat-coloured face


def _texture(X: np.ndarray, seed: int) -> np.ndarray:
    """Procedural texture in 0..1 from world points: sines over three scales plus a hashed cell pattern."""
    rng = np.random.RandomState(seed)
    f = rng.uniform(3.0, 9.0, (4, 3))
    v = sum(np.sin(X @ f[k] + k) for k in range(4)) / 8.0 + 0.5
    cell = np.floor(X * 4.0).astype(np.int64)
    h = (cell[..., 0] * 73856093) ^ (cell[..., 1] * 19349663) ^ (cell[..., 2] * 83492791)
    return np.clip(0.6 * v + 0.4 * ((h % 1000) / 1000.0), 0.0, 1.0)


def textured_scene(num_cameras: int = 4, width: int = 160, height: int = 120, seed: int = 3,
                   arc_degrees: float = 40.0, radius: float = 6.0, focal: float = 0.9,
                   sizes: Optional[List[Tuple[int, int]]] = None) -> TexturedScene:
    """A ground plane (z = 0) with two boxes, seen from cameras on an arc around the origin, rendered by analytic
    ray casting.  Every face is textured except the top of the first box, which is one flat colour.  `sizes` gives
    each camera its own (width, height); `focal` is relative to the larger image side."""
    boxes = [(np.array([-1.2, -0.6, 0.0]), np.array([-0.2, 0.4, 0.9])),
             (np.array([0.4, -0.2, 0.0]), np.array([1.3, 0.9, 0.6]))]
    S = num_cameras
    sizes = sizes or [(width, height)] * S
    Ks, Rs, ts, grays, rgbs, depths, flats = [], [], [], [], [], [], []
    for c in range(S):
        w, h = sizes[c]
        ang = np.radians(-arc_degrees / 2 + arc_degrees * c / max(S - 1, 1))
        C = np.array([radius * np.sin(ang), -radius * np.cos(ang), 3.0])
        fwd = _normalized(np.array([0.0, 0.0, 0.2]) - C)
        right = _normalized(np.cross(fwd, np.array([0.0, 0.0, 1.0])))
        down = np.cross(fwd, right)
        R = np.stack([right, down, fwd])
        t = -R @ C
        f = focal * max(w, h)
        K = np.array([[f, 0, (w - 1) / 2.0], [0, f, (h - 1) / 2.0], [0, 0, 1.0]])
        jj, ii = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
        pix = np.stack([jj, ii, np.ones_like(jj)], -1)
        dcam = pix @ np.linalg.inv(K).T                    # z_cam = 1 along each ray
        dw = dcam @ R                                      # world direction with z_cam = 1
        best = np.full((h, w), np.inf)
        face = np.full((h, w), -1)
        with np.errstate(divide="ignore", invalid="ignore"):
            s = -C[2] / dw[..., 2]                         # ground plane
            ok = s > 0
            best = np.where(ok, s, best)
            face = np.where(ok, 0, face)
            for b, (lo, hi) in enumerate(boxes):
                for ax in range(3):
                    for side, val in ((0, lo[ax]), (1, hi[ax])):
                        s = (val - C[ax]) / dw[..., ax]
                        X = C + s[..., None] * dw
                        o1, o2 = [k for k in range(3) if k != ax]
                        inside = ((X[..., o1] >= lo[o1]) & (X[..., o1] <= hi[o1]) & (X[..., o2] >= lo[o2]) &
                                  (X[..., o2] <= hi[o2]) & (s > 0) & (s < best))
                        best = np.where(inside, s, best)
                        face = np.where(inside, 1 + 6 * b + 2 * ax + side, face)
        hit = np.isfinite(best)
        X = C + np.where(hit, best, 0.0)[..., None] * dw
        tex = _texture(X, seed)
        flat = face == 1 + 2 * 2 + 1                       # top of box 0
        tex = np.where(flat, 0.55, tex)
        shade = 0.6 + 0.4 * ((face % 5) / 4.0)
        gray = np.clip(255.0 * tex * np.where(hit, shade, 0.0), 0, 255)
        rgb = np.stack([gray, np.clip(gray * 0.8 + 30 * (face % 3), 0, 255), np.clip(255 - gray * 0.7, 0, 255)], -1)
        Ks.append(K)
        Rs.append(R)
        ts.append(t)
        grays.append(gray.astype(np.uint8))
        rgbs.append(rgb.astype(np.uint8))
        depths.append(np.where(hit, best, 0.0).astype(np.float32))
        flats.append(flat)
    stack = (lambda a: np.stack(a)) if len(set(sizes)) == 1 else (lambda a: np.array(a + [None], dtype=object)[:-1])
    return TexturedScene(np.stack(Ks), np.stack(Rs), np.stack(ts), stack(grays), stack(rgbs), stack(depths),
                         stack(flats))
