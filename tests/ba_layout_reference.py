"""Host restatement of the point layout the bundle adjustment builds on the device (opensfm_b200/csrc/ba_order.cuh),
written from its rule, not from the kernels:

* a point is segment-eligible when it has between 1 and SEG_KMAX = 16 observations, k * wc <= SEG_NA = 96
  camera-side columns, wc <= SEG_WCMAX = 16, no point prior, and the per-point Schur fallback is off; constant points
  are eligible like free ones;
* the eligible points come first (p_fast of them, with n_fast observations), the others after them (p_slow);
* eligible points with the same shot list (their shots in (shot) order, a shot repeated for each duplicate observation)
  and the same constant flag form one group, and a group is cut into segments of at most SEG_MAX_POINTS = 64 points.
  nseg is the number of those segments.

The device finds the groups by sorting on a 64-bit hash of (shot list, constant flag); without a collision its groups
are these.  Single rank (world = 1) only.

Not a test module: the test files import it (pytest puts tests/ on sys.path)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Sequence

import numpy as np

SEG_KMAX = 16
SEG_NA = 96
SEG_WCMAX = 16
SEG_MAX_POINTS = 64


@dataclass
class Layout:
    eligible: np.ndarray   # (P,) bool, per caller's point
    p_fast: int
    p_slow: int
    n_fast: int            # observations of the eligible points
    nseg: int
    group_sizes: list      # points per group of eligible points, largest first


def layout(obs_shot: Sequence[int], obs_point: Sequence[int], point_const: Sequence[int], point_prior: Sequence[bool],
           wc: int, per_point_fallback: bool = False) -> Layout:
    obs_shot = np.asarray(obs_shot, dtype=np.int64)
    obs_point = np.asarray(obs_point, dtype=np.int64)
    const = np.asarray(point_const) != 0
    prior = np.asarray(point_prior, dtype=bool)
    P = len(const)
    shots = [[] for _ in range(P)]
    for s, p in zip(obs_shot.tolist(), obs_point.tolist()):
        shots[p].append(s)
    k = np.array([len(l) for l in shots], dtype=np.int64)
    eligible = (~prior) & (k >= 1) & (k <= SEG_KMAX) & (k * wc <= SEG_NA)
    if per_point_fallback or wc > SEG_WCMAX:
        eligible[:] = False
    groups = {}
    for p in np.nonzero(eligible)[0].tolist():
        key = (tuple(sorted(shots[p])), bool(const[p]))
        groups[key] = groups.get(key, 0) + 1
    sizes = sorted(groups.values(), reverse=True)
    nseg = sum(-(-n // SEG_MAX_POINTS) for n in sizes)
    p_fast = int(eligible.sum())
    return Layout(eligible=eligible, p_fast=p_fast, p_slow=P - p_fast, n_fast=int(k[eligible].sum()), nseg=nseg,
                  group_sizes=sizes)


def camera_side_width(pb) -> int:
    """wc of a BAProblem: the widest camera side of any shot (camera parameters + instance pose + rig-camera pose when
    the shot goes through its rig camera), at least 1; shots without observations count too."""
    from opensfm_b200 import ba_problem as bp

    wc = 1
    for s in range(len(pb.shot_inst)):
        wc = max(wc, bp.camera_num_params(pb.cam_type[pb.shot_cam[s]]) + 6 + (6 if pb.shot_use_rc[s] else 0))
    return wc


def problem_layout(pb, per_point_fallback: bool = False) -> Layout:
    prior = np.zeros(len(pb.points), dtype=bool)
    prior[np.asarray(pb.pp_point, dtype=np.int64)] = True
    return layout(pb.obs_shot, pb.obs_point, pb.point_const, prior, camera_side_width(pb), per_point_fallback)
