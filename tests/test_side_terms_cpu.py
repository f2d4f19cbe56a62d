"""The oracle's side-term rows (robustified residual and Jacobian of each of the 17 types) against the independent
mpmath restatement of the reference's functors (tests/side_terms_mp.py), on random configurations of every type and
on the named edge cases where the functors branch.  Also the builders the GPU test (test_ba_side_terms_gpu.py) solves:
one problem of many independent terms, each on its own parameter blocks.

Errors are measured per residual row, relative to the row's largest |J| (and, for r, to the term's largest |r| or
|J|): a formula slip, a wrong branch or a wrong column moves that ratio to O(1); fp64 round-off keeps it near 1e-15."""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import numpy as np
import pytest
from scipy.optimize import brentq
from scipy.spatial.transform import Rotation

import side_terms_mp as smp
from opensfm_b200 import ba_problem as bp
from oracle import ba_lm as oracle

# worst row error (oracle vs mpmath) over the random configurations and the edge cases below: J 1.2e-13 (a roll term),
# r 8.5e-15; the bounds are at most 100x that.  The two roll terms 10 % outside the guards divide by la ~ 1e-5 or by
# cos(roll) ~ 5e-3 and lose that much more: worst 4.5e-12 there.
J_TOL = 1e-11
R_TOL = 5e-13
ROLL_GUARD_J_TOL = 4e-10
N_RANDOM = 200


# ---- building problems of independent terms ----------------------------------------------------------------
class Builder:
    """Allocates parameter blocks (rig instances, rig cameras, ext blocks, DUAL cameras) and collects terms; problem()
    is a BAProblem without shots, points or observations: its cost is the side terms (plus the camera priors of the
    free cameras)."""

    def __init__(self):
        self.inst, self.inst_const, self.rc, self.rc_const, self.cams, self.cam_const = [], [], [], [], [], []
        self.ext = []          # (values, constant, lower)
        self.terms: List[bp.SideTerm] = []
        self.names: List[str] = []

    def add_inst(self, v, const=False):
        self.inst.append(np.asarray(v, dtype=np.float64))
        self.inst_const.append(int(const))
        return len(self.inst) - 1

    def add_rc(self, v, const=False):
        self.rc.append(np.asarray(v, dtype=np.float64))
        self.rc_const.append(int(const))
        return len(self.rc) - 1

    def add_ext(self, v, const=False, lower=None):
        self.ext.append((np.atleast_1d(np.asarray(v, dtype=np.float64)), bool(const), lower))
        return len(self.ext) - 1

    def add_dual(self, v, const=False):
        self.cams.append(np.asarray(v, dtype=np.float64))
        self.cam_const.append(int(const))
        return len(self.cams) - 1

    def add(self, name, term):
        self.terms.append(term)
        self.names.append(name)

    def problem(self) -> bp.BAProblem:
        NI, NR, K = len(self.inst), max(len(self.rc), 1), len(self.cams)
        z = lambda n: np.zeros(n, dtype=np.int32)
        cam_params = np.concatenate(self.cams) if K else np.zeros(0)
        sd = dict(focal_sd=0.1, aspect_ratio_sd=0.1, c_sd=0.1, k1_sd=0.1, k2_sd=0.1)
        pb = bp.BAProblem(
            cam_type=np.full(K, bp.DUAL, dtype=np.int32), cam_params=cam_params,
            cam_const=np.array(self.cam_const, dtype=np.int32), cam_prior=cam_params.copy(),
            cam_prior_sigma=np.concatenate([bp.default_prior_sigma(bp.DUAL, **sd)] * K) if K else np.zeros(0),
            cam_prior_log=np.concatenate([bp.prior_log_mask(bp.DUAL)] * K) if K else z(0),
            inst=np.array(self.inst).reshape(NI, 6), inst_const=np.array(self.inst_const, dtype=np.int32),
            inst_has_prior=z(NI), inst_prior_pos=np.zeros((NI, 3)), inst_prior_std=np.ones((NI, 3)),
            rigcam=np.array(self.rc).reshape(-1, 6) if self.rc else np.zeros((1, 6)),
            rigcam_const=np.array(self.rc_const, dtype=np.int32) if self.rc else np.ones(1, dtype=np.int32),
            shot_inst=z(0), shot_cam=z(0), shot_rc=z(0), shot_use_rc=z(0), points=np.zeros((0, 3)), point_const=z(0),
            obs_shot=z(0), obs_point=z(0), obs_xy=np.zeros((0, 2)), obs_sigma=np.zeros(0), loss_name="TrivialLoss",
            loss_threshold=1.0, max_iterations=1)
        for v, c, lo in self.ext:
            pb.add_ext_block(v, c, lo)
        pb.side_terms = list(self.terms)
        assert NR == len(pb.rigcam)
        return pb


def block_values(pb: bp.BAProblem, kind: int, idx: int) -> np.ndarray:
    if kind == bp.SB_INST:
        return pb.inst[idx]
    if kind == bp.SB_RIGCAM:
        return pb.rigcam[idx]
    if kind == bp.SB_EXT:
        o = pb.ext_off
        return pb.ext_values[o[idx]:o[idx + 1]]
    o = pb.cam_off
    return pb.cam_params[o[idx]:o[idx + 1]]


def block_constant(pb: bp.BAProblem, kind: int, idx: int) -> bool:
    return bool({bp.SB_INST: pb.inst_const, bp.SB_RIGCAM: pb.rigcam_const, bp.SB_EXT: pb.ext_const,
                 bp.SB_CAM: pb.cam_const}[kind][idx])


def mp_rows(pb: bp.BAProblem):
    """Per term: (r, J over its distinct blocks with the columns of constant blocks zeroed, ok) from mpmath."""
    out = []
    for t in pb.side_terms:
        blocks = smp.distinct_blocks(t)
        r, J, ok = smp.rows(t, {b: block_values(pb, *b) for b in blocks})
        if ok:
            c = 0
            for b in blocks:
                n = pb.block_size(*b)
                if block_constant(pb, *b):
                    J[:, c:c + n] = 0.0
                c += n
        out.append((r, J, ok))
    return out


def split_rows(pb: bp.BAProblem, r: np.ndarray, J: np.ndarray):
    """Flat packed rows (capture / oracle_side_rows layout) -> per term (r, J folded onto its distinct blocks)."""
    nrow, nJ = pb.side_row_sizes()
    ro, jo = np.concatenate([[0], np.cumsum(nrow)]), np.concatenate([[0], np.cumsum(nJ)])
    out = []
    for k, t in enumerate(pb.side_terms):
        sizes = [pb.block_size(*b) for b in t.blocks]
        Jl = J[jo[k]:jo[k + 1]].reshape(t.nres, sum(sizes))
        out.append((r[ro[k]:ro[k + 1]], smp.fold_columns(t, Jl, sizes)))
    return out


def row_errors(got, want) -> Tuple[float, float]:
    """(worst J error per row relative to the row's max |J|, worst r error relative to max(|r|, |J|) of the term)."""
    (rg, Jg), (rw, Jw) = got, want
    den = np.max(np.abs(Jw), axis=1)
    dJ = np.max(np.abs(Jg - Jw), axis=1)
    ej = float(np.max(np.where(den > 0, dJ / np.where(den > 0, den, 1.0), np.where(dJ > 0, np.inf, 0.0))))
    scale = max(float(np.max(np.abs(rw))), float(np.max(np.abs(Jw))))
    dr = float(np.max(np.abs(rg - rw)))
    er = dr / scale if scale > 0 else (np.inf if dr > 0 else 0.0)
    return ej, er


# ---- random configurations -------------------------------------------------------------------------------------
def rotvec(rng, max_angle=3.0):
    a = rng.normal(size=3)
    return a / np.linalg.norm(a) * rng.uniform(0.05, max_angle)


def pose(rng, max_angle=3.0, t_scale=2.0):
    return np.concatenate([rotvec(rng, max_angle), rng.normal(0, t_scale, 3)])


def const_flag(rng):
    return rng.uniform() < 0.12


def scale_matrix(rng, n):
    return np.eye(n) * rng.uniform(0.5, 2.0) + rng.normal(0, 0.2, (n, n))


def rc_or_none(B, rng, p=0.6):
    return B.add_rc(pose(rng, 0.5, 0.5), const_flag(rng)) if rng.uniform() < p else None


def random_term(B: Builder, ty: int, rng) -> bp.SideTerm:
    inst = lambda **kw: B.add_inst(kw.get("v", pose(rng)), const_flag(rng))
    loss = lambda: (int(rng.choice([bp.LOSS_CAUCHY, bp.LOSS_SOFTLONE, 1, 4, 0, bp.LOSS_NONE])), float(rng.uniform(0.3, 3)))
    if ty in (bp.SIDE_UP_VECTOR, bp.SIDE_PAN, bp.SIDE_TILT, bp.SIDE_ROLL):
        i, rc = inst(), B.add_rc(pose(rng, 0.5, 0.5), const_flag(rng))
        if ty == bp.SIDE_UP_VECTOR:
            return bp.up_vector_term(i, rc, rng.normal(size=3), rng.uniform(0.1, 2))
        angle = rng.uniform(-1.5, 1.5) if ty == bp.SIDE_TILT else rng.uniform(-3.1, 3.1)
        return bp.angle_term(ty, i, rc, angle, rng.uniform(0.1, 2))
    if ty == bp.SIDE_RELATIVE_MOTION:
        i, j = inst(), inst()
        si = B.add_ext(rng.uniform(0.5, 2), const_flag(rng), [0.0])
        sj = si if rng.uniform() < 0.4 else B.add_ext(rng.uniform(0.5, 2), const_flag(rng), [0.0])
        rts = np.concatenate([rotvec(rng), rng.normal(0, 1, 3), [rng.uniform(0.5, 2)]])
        return bp.relative_motion_term(i, j, si, sj, rts, scale_matrix(rng, 7), bool(rng.uniform() < 0.5), *loss())
    if ty == bp.SIDE_RELATIVE_ROTATION:
        i, j = inst(), inst()
        return bp.relative_rotation_term(i, j, rc_or_none(B, rng), rc_or_none(B, rng), rotvec(rng), scale_matrix(rng, 3),
                                         *loss())
    if ty == bp.SIDE_COMMON_POSITION:
        pi = pose(rng)
        i, j = B.add_inst(pi, const_flag(rng)), B.add_inst(np.concatenate([rotvec(rng), pi[3:] + rng.normal(0, 0.4, 3)]),
                                                          const_flag(rng))
        return bp.common_position_term(i, j, rc_or_none(B, rng), rc_or_none(B, rng), rng.uniform(0, 0.3),
                                       rng.uniform(0.5, 3))
    if ty == bp.SIDE_LINEAR_MOTION:
        ii = [inst() for _ in range(3)]
        rcs = [rc_or_none(B, rng) for _ in range(3)]
        if rcs[0] is not None and rng.uniform() < 0.3:
            rcs[2] = rcs[0]   # one rig camera behind two shots: one block
        return bp.linear_motion_term(ii, rcs, rng.uniform(0.2, 0.8), rng.uniform(0.5, 3), rng.uniform(0.5, 3))
    if ty == bp.SIDE_TRANSLATION_PRIOR:
        return bp.translation_prior_term(inst(), inst(), rng.uniform(0.5, 3))
    if ty == bp.SIDE_PARAMETER_BARRIER:
        c = B.add_dual([rng.uniform(0.05, 0.95), rng.normal(0, 0.05), rng.normal(0, 0.01), rng.uniform(0.5, 1.5)],
                       const_flag(rng))
        return bp.parameter_barrier_term(c, 0, 0.0, 1.0)
    if ty == bp.SIDE_STD_DEVIATION:
        return bp.std_deviation_term(B.add_ext(rng.uniform(0.2, 3), const_flag(rng), [1e-10]))
    if ty == bp.SIDE_POSITION_PRIOR:
        i = inst()
        bias = B.add_ext(np.concatenate([rotvec(rng, 0.5), rng.normal(0, 1, 3), [rng.uniform(0.5, 2)]]), const_flag(rng))
        sd = B.add_ext(rng.uniform(0.5, 2), const_flag(rng), [1e-10])
        return bp.position_prior_term(i, bias, sd, rng.normal(0, 2, 3), rng.uniform(0.2, 2, 3), bool(rng.uniform() < 0.5))
    rec = lambda: B.add_ext(np.concatenate([rotvec(rng), rng.normal(0, 2, 3), [rng.uniform(0.5, 2)]]), const_flag(rng),
                            [-np.inf] * 6 + [0.1])
    if ty == bp.SIDE_RA_RELATIVE_MOTION:
        return bp.SideTerm(ty, 6, [(bp.SB_EXT, rec()), (bp.SB_INST, inst())],
                           np.concatenate([pose(rng), scale_matrix(rng, 6).ravel()]), bp.LOSS_CAUCHY, 1.0)
    if ty == bp.SIDE_RA_ABSOLUTE_POSITION:
        return bp.SideTerm(ty, 3, [(bp.SB_INST, inst())], np.concatenate([rng.normal(0, 2, 3), [rng.uniform(0.5, 3)]]))
    if ty == bp.SIDE_RA_RELATIVE_ABSOLUTE_POSITION:
        return bp.SideTerm(ty, 3, [(bp.SB_EXT, rec())], np.concatenate([rng.normal(0, 2, 3), pose(rng), [rng.uniform(0.5, 3)]]),
                           bp.LOSS_SOFTLONE, 1.0)
    if ty == bp.SIDE_RA_COMMON_POINT:
        return bp.SideTerm(ty, 3, [(bp.SB_EXT, rec()), (bp.SB_EXT, rec())],
                           np.concatenate([rng.normal(0, 2, 6), [rng.uniform(0.5, 3)]]), bp.LOSS_SOFTLONE, 1.0)
    if ty == bp.SIDE_RA_COMMON_CAMERA:
        return bp.SideTerm(ty, 6, [(bp.SB_EXT, rec()), (bp.SB_EXT, rec())],
                           np.concatenate([pose(rng), pose(rng), rng.uniform(0.5, 3, 2)]), bp.LOSS_CAUCHY, 1.0)
    raise ValueError(ty)


TYPE_NAMES = {getattr(bp, n): n[5:].lower() for n in dir(bp) if n.startswith("SIDE_") and isinstance(getattr(bp, n), int)}


def random_builder(types, n, seed) -> Builder:
    B = Builder()
    for ty in types:
        rng = np.random.RandomState(seed + 1000 * ty)
        for k in range(n):
            B.add("%s/%d" % (TYPE_NAMES[ty], k), random_term(B, ty, rng))
    return B


# ---- named edge cases ----------------------------------------------------------------------------------------------
def _rot(R):
    return Rotation.from_matrix(R).as_rotvec()


def _roll_quantities(aa):
    R = Rotation.from_rotvec(aa)
    ex, ez = R.apply([1.0, 0, 0]), R.apply([0, 0, 1.0])
    a = np.array([ez[1], -ez[0], 0.0])
    la = np.hypot(a[0], a[1])
    a /= la
    return la, float(np.dot(ez, np.cross(ex, a)))


def _roll_pose(target_sin_roll):
    """Rotation (tilted 0.4 rad off the horizon) whose roll has sin = target, found on a rotation about the optical
    axis: sin_roll runs through -1 there."""
    base = Rotation.from_rotvec([0.4, 0.0, 0.0])
    f = lambda g: _roll_quantities((base * Rotation.from_rotvec([0, 0, g])).as_rotvec())[1]
    gs = np.linspace(-np.pi, np.pi, 2001)
    g0 = gs[np.argmin([f(g) for g in gs])]
    g = brentq(lambda g: f(g) - target_sin_roll, g0, g0 + 1.0, xtol=1e-15)
    return (base * Rotation.from_rotvec([0, 0, g])).as_rotvec()


def edge_cases(B: Builder) -> None:
    """Adds every named edge case of the side terms to B (names say which branch each one reaches)."""
    rng = np.random.RandomState(77)
    zero6 = np.zeros(6)
    rc0 = lambda: B.add_rc(zero6)
    # rotations exactly 0: AngleAxisToQuaternion's Taylor branch (instance and rig camera both 0)
    B.add("rotation_zero/up_vector", bp.up_vector_term(B.add_inst([0, 0, 0, 1, 2, 3]), rc0(), [0.1, 0.2, 1.0], 0.5))
    B.add("rotation_zero/relative_rotation", bp.relative_rotation_term(
        B.add_inst([0, 0, 0, 1, 0, 0]), B.add_inst([0, 0, 0, 0, 1, 0]), rc0(), None, [0.0, 0.0, 0.0], np.eye(3),
        bp.LOSS_NONE, 1.0))
    B.add("rotation_zero/ra_relative_motion", bp.SideTerm(
        bp.SIDE_RA_RELATIVE_MOTION, 6, [(bp.SB_EXT, B.add_ext([0, 0, 0, 1, 2, 3, 1.5])), (bp.SB_INST, B.add_inst(zero6))],
        np.concatenate([zero6, np.eye(6).ravel()]), bp.LOSS_CAUCHY, 1.0))
    # theta^2 <= DBL_EPSILON: AngleAxisRotatePoint's first-order branch
    tiny = np.array([6e-9, -4e-9, 7e-9])
    B.add("rotation_below_eps/up_vector", bp.up_vector_term(B.add_inst(np.r_[tiny, 0, 0, 0]), rc0(), [0.3, -0.2, 1.0], 0.5))
    B.add("rotation_below_eps/common_position", bp.common_position_term(
        B.add_inst(np.r_[tiny, 0, 0, 0]), B.add_inst([0.1, 0, 0, 0.5, 0.2, 0]), B.add_rc([0.1, 0, 0, 0.3, -0.2, 0.1]),
        None, 0.0, 1.0))
    B.add("rotation_below_eps/ra_absolute_position", bp.SideTerm(
        bp.SIDE_RA_ABSOLUTE_POSITION, 3, [(bp.SB_INST, B.add_inst(np.r_[tiny, 1, 2, 3]))], np.array([0.5, 0.5, 0.5, 2.0])))
    # relative rotations near pi: QuaternionToAngleAxis with cos < 0 (and just below pi, cos > 0)
    for tag, ang in (("below", np.pi - 1e-3), ("above", np.pi + 1e-3), ("far_above", 3.9)):
        B.add("rotation_near_pi_%s/relative_rotation" % tag, bp.relative_rotation_term(
            B.add_inst([0.2, 0, 0, 0, 0, 0]), B.add_inst([0.2 + ang - 3.0, 0, 0, 1, 0, 0]), None, None, [3.0, 0.0, 0.0],
            np.eye(3), bp.LOSS_NONE, 1.0))
    B.add("rotation_near_pi/linear_motion", bp.linear_motion_term(
        [B.add_inst([0, 0, 0, 0, 0, 0]), B.add_inst([0, 1.6, 0, 1, 0, 0]), B.add_inst([0, 0, 1.7, 2, 0.1, 0])],
        [None, None, None], 0.5, 1.0, 1.0))
    # pan: predicted angle near +-pi, observed near -+pi: DiffBetweenAngles wraps
    for tag, target, yaw in (("plus", -3.1, 3.1), ("minus", 3.1, -3.1)):
        R = Rotation.from_rotvec([0, 0, 0.0])
        # z_world = R ez with atan2(z0, z1) = yaw: tilt the optical axis towards (sin yaw, cos yaw)
        axis = np.array([np.sin(yaw), np.cos(yaw), 0.0])
        aa = np.cross([0, 0, 1.0], axis) / np.linalg.norm(np.cross([0, 0, 1.0], axis)) * 1.0
        B.add("pan_wrap_%s" % tag, bp.angle_term(bp.SIDE_PAN, B.add_inst(np.r_[aa, 0, 0, 0]), rc0(), target, 0.5))
    # tilt close to +-pi/2: the optical axis close to the vertical
    for tag, ang in (("up", 1e-6), ("down", np.pi - 1e-6)):
        B.add("tilt_near_half_pi_%s" % tag, bp.angle_term(bp.SIDE_TILT, B.add_inst([ang, 0, 0, 0, 0, 0]), rc0(), 1.5, 0.5))
    # roll: la < 1e-5 and sin_roll <= -(1 - 1e-5), 10 % inside and outside each guard
    for tag, la in (("inside", 0.9e-5), ("outside", 1.1e-5)):
        B.add("roll_la_%s" % tag, bp.angle_term(bp.SIDE_ROLL, B.add_inst([math.asin(la), 0, 0, 0, 0, 0]), rc0(), 0.1, 0.5))
    for tag, d in (("inside", 0.9e-5), ("outside", 1.1e-5)):
        B.add("roll_sin_%s" % tag, bp.angle_term(bp.SIDE_ROLL, B.add_inst(np.r_[_roll_pose(-(1 - d)), 0, 0, 0]), rc0(),
                                                   -1.4, 0.5))
    # common position: margin active on both horizontal axes, inactive, and Tukey beyond its threshold (w = 0)
    # ("margin_exact": |e_x| - margin is exactly 0, where std::max(T(0), m) keeps the constant 0)
    for tag, dt, margin, sd in (("margin_active", [0.1, -0.1, 0.3], 0.2, 2.0), ("margin_inactive", [0.3, -0.4, 0.2], 0.1, 2.0),
                                ("margin_exact", [0.25, 0.5, 0.0], 0.25, 2.0), ("tukey_beyond", [0.3, -0.4, 2.0], 0.1, 1.0)):
        B.add("common_position_%s" % tag, bp.common_position_term(
            B.add_inst([0.1, 0.2, 0.3, 1, 2, 3]), B.add_inst(np.r_[0.3, -0.2, 0.1, np.array([1, 2, 3]) + dt]), None, None,
            margin, sd))
    # linear motion with t2 == t0 (n20 = 0 <= 1e-15)
    B.add("linear_motion_n20_zero", bp.linear_motion_term(
        [B.add_inst([0.1, 0, 0, 1, 2, 3]), B.add_inst([0.2, 0.1, 0, 2, 2, 3]), B.add_inst([0.3, 0, 0.1, 1, 2, 3])],
        [None, None, None], 0.5, 1.0, 1.0))
    # relative motion: observed scale on / off x shared / separate scale blocks, and a zero scale
    for obs in (True, False):
        for shared in (True, False):
            si = B.add_ext(1.3, False, [0.0])
            sj = si if shared else B.add_ext(0.8, False, [0.0])
            B.add("relative_motion_%s_%s" % ("observed" if obs else "unobserved", "shared" if shared else "separate"),
                  bp.relative_motion_term(B.add_inst(pose(rng)), B.add_inst(pose(rng)), si, sj,
                                          np.r_[rotvec(rng), rng.normal(0, 1, 3), 1.1], scale_matrix(rng, 7), obs,
                                          bp.LOSS_SOFTLONE, 1.0))
    # position prior with and without adjust_scales
    for adjust in (True, False):
        B.add("position_prior_adjust_%s" % ("on" if adjust else "off"), bp.position_prior_term(
            B.add_inst(pose(rng)), B.add_ext(np.r_[rotvec(rng, 0.3), rng.normal(0, 1, 3), 1.2]), B.add_ext(1.7, False, [1e-10]),
            rng.normal(0, 1, 3), [0.5, 1.0, 2.0], adjust))
    # every rig-camera variant (aux >= 0): none, i only, j only, both distinct, both the same block
    for tag, (a, b) in (("none", (None, None)), ("i", (0, None)), ("j", (None, 0)), ("both", (0, 1)), ("shared", (0, 0))):
        rcs = [B.add_rc(pose(rng, 0.5, 0.5)), B.add_rc(pose(rng, 0.5, 0.5))]
        pick = lambda k: None if k is None else rcs[k]
        B.add("rigcams_%s/relative_rotation" % tag, bp.relative_rotation_term(
            B.add_inst(pose(rng)), B.add_inst(pose(rng)), pick(a), pick(b), rotvec(rng), scale_matrix(rng, 3),
            bp.LOSS_CAUCHY, 1.0))
        pi = pose(rng)
        B.add("rigcams_%s/common_position" % tag, bp.common_position_term(
            B.add_inst(pi), B.add_inst(np.r_[rotvec(rng), pi[3:] + 0.3]), pick(a), pick(b), 0.05, 2.0))
    for tag, sel in (("lm_none", (None, None, None)), ("lm_0", (0, None, None)), ("lm_1", (None, 0, None)),
                     ("lm_2", (None, None, 0)), ("lm_three", (0, 1, 2)), ("lm_shared", (0, 1, 0))):
        rcs = [B.add_rc(pose(rng, 0.5, 0.5)) for _ in range(3)]
        B.add("rigcams_%s/linear_motion" % tag, bp.linear_motion_term(
            [B.add_inst(pose(rng)) for _ in range(3)], [None if k is None else rcs[k] for k in sel], 0.5, 1.0, 1.0))
    # Cauchy-robustified terms inside (s << 1) and far outside (s >> 1) their scale
    for tag, std in (("inside", 50.0), ("outside", 0.01)):
        B.add("cauchy_%s/up_vector" % tag, bp.up_vector_term(B.add_inst(pose(rng, 0.3)), rc0(), [0, 0.1, 1.0], std))
        B.add("cauchy_%s/relative_rotation" % tag, bp.relative_rotation_term(
            B.add_inst(pose(rng)), B.add_inst(pose(rng)), None, None, rotvec(rng), np.eye(3) / std * 0.1, bp.LOSS_CAUCHY, 1.0))
    # one rig instance listed twice: two shots of one instance through two rig cameras
    i = B.add_inst(pose(rng))
    B.add("duplicate_instance/common_position", bp.common_position_term(
        i, i, B.add_rc(pose(rng, 0.3, 0.5)), B.add_rc(pose(rng, 0.3, 0.5)), 0.0, 2.0))
    i = B.add_inst(pose(rng))
    B.add("duplicate_instance/relative_rotation", bp.relative_rotation_term(
        i, i, B.add_rc(pose(rng, 0.3, 0.5)), B.add_rc(pose(rng, 0.3, 0.5)), rotvec(rng, 0.3), scale_matrix(rng, 3),
        bp.LOSS_NONE, 1.0))
    i = B.add_inst(pose(rng))
    B.add("duplicate_instance/linear_motion", bp.linear_motion_term(
        [i, B.add_inst(pose(rng)), i], [B.add_rc(pose(rng, 0.3, 0.5)), None, B.add_rc(pose(rng, 0.3, 0.5))], 0.5, 1.0, 1.0))


def edge_builder() -> Builder:
    B = Builder()
    edge_cases(B)
    return B


# ---- the tests ---------------------------------------------------------------------------------------------------
def j_tol(name: str) -> float:
    return ROLL_GUARD_J_TOL if name.startswith("roll_") and name.endswith("_outside") else J_TOL


def _compare_oracle(B: Builder):
    pb = B.problem()
    ob = oracle.OracleBA(pb)
    _, r, J = ob.side_rows(pb)
    got = split_rows(pb, r, J)
    want = mp_rows(pb)
    worst = {}
    for name, t, g, (rw, Jw, ok) in zip(B.names, pb.side_terms, got, want):
        assert ok, name
        ej, er = row_errors(g, (rw, Jw))
        worst[name] = (ej, er)
    return worst


@pytest.mark.parametrize("ty", sorted(TYPE_NAMES), ids=lambda t: TYPE_NAMES[t])
def test_oracle_rows_match_mpmath_on_random_terms(ty):
    worst = _compare_oracle(random_builder([ty], N_RANDOM, seed=11))
    ej = max(v[0] for v in worst.values())
    er = max(v[1] for v in worst.values())
    print("%s: worst J %.2e r %.2e" % (TYPE_NAMES[ty], ej, er))
    bad = {k: v for k, v in worst.items() if v[0] > j_tol(k) or v[1] > R_TOL}
    assert not bad, bad


def test_oracle_rows_match_mpmath_on_edge_cases():
    worst = _compare_oracle(edge_builder())
    for k, v in worst.items():
        print("%-48s J %.2e r %.2e" % (k, v[0], v[1]))
    bad = {k: v for k, v in worst.items() if v[0] > j_tol(k) or v[1] > R_TOL}
    assert not bad, bad


def test_edge_cases_reach_their_branches():
    """The edge cases are where they say they are: the guards' values sit on the named side of each threshold."""
    for tag, d in (("inside", 0.9e-5), ("outside", 1.1e-5)):
        la, s = _roll_quantities(_roll_pose(-(1 - d)))
        assert abs(s + (1 - d)) < 1e-12 and la > 1e-5
    for la in (0.9e-5, 1.1e-5):
        assert abs(_roll_quantities([math.asin(la), 0, 0])[0] - la) < 1e-15
    B = edge_builder()
    pb = B.problem()
    rows = dict(zip(B.names, mp_rows(pb)))
    assert np.all(rows["roll_la_inside"][0] == 0) and np.any(rows["roll_la_outside"][1] != 0)
    assert np.all(rows["roll_sin_inside"][0] == 0) and np.any(rows["roll_sin_outside"][1] != 0)
    assert np.all(rows["common_position_margin_active"][1][:2] == 0)
    assert np.all(rows["common_position_margin_exact"][1][0] == 0) and np.any(rows["common_position_margin_exact"][1][1] != 0)
    assert np.all(rows["common_position_tukey_beyond"][1] == 0) and np.all(rows["common_position_tukey_beyond"][0] == 0)
    for tag in ("plus", "minus"):
        assert abs(rows["pan_wrap_%s" % tag][0][0]) < 0.2 * 2   # wrapped: |d| ~ 2 pi - 6.2, times 1/std = 2
    # the instance columns of a common position of two cameras on one instance cancel in translation
    Jd = rows["duplicate_instance/common_position"][1]
    assert np.max(np.abs(Jd[:, 3:6])) == 0.0


def test_duplicate_instance_column_norms_are_those_of_the_summed_column():
    """A term listing one rig instance twice: the column norms and the gradient of the oracle are those of the summed
    local columns (mpmath's Jacobian over the distinct blocks), not the sum of the two local columns' norms."""
    B = Builder()
    rng = np.random.RandomState(3)
    i = B.add_inst(pose(rng))
    B.add("cp", bp.common_position_term(i, i, B.add_rc(pose(rng, 0.3, 0.5)), B.add_rc(pose(rng, 0.3, 0.5)), 0.0, 2.0))
    i = B.add_inst(pose(rng))
    B.add("lm", bp.linear_motion_term([i, B.add_inst(pose(rng)), i], [B.add_rc(pose(rng, 0.3, 0.5)), None,
                                                                     B.add_rc(pose(rng, 0.3, 0.5))], 0.5, 1.0, 1.0))
    pb = B.problem()
    ob = oracle.OracleBA(pb)
    ob.linearize()
    cn, g = ob.colnorm_gradient()
    cn_mp, g_mp = dense_colnorm_gradient(pb, mp_rows(pb), ob.nc)
    assert np.max(np.abs(cn - cn_mp)) <= 1e-12 * np.max(cn_mp), np.c_[cn, cn_mp]
    assert np.max(np.abs(g - g_mp)) <= 1e-12 * np.max(np.abs(g_mp)), np.c_[g, g_mp]


def column_offsets(pb: bp.BAProblem) -> Dict[Tuple[int, int], int]:
    """First reduced column of every free block: [free cameras | instances | rig cameras | ext blocks]."""
    off, col = {}, 0
    for kind, n in ((bp.SB_CAM, len(pb.cam_type)), (bp.SB_INST, len(pb.inst)), (bp.SB_RIGCAM, len(pb.rigcam)),
                    (bp.SB_EXT, len(pb.ext_size))):
        for i in range(n):
            if not block_constant(pb, kind, i):
                off[(kind, i)] = col
                col += pb.block_size(kind, i)
    return off


def dense_jacobian(pb: bp.BAProblem, rows, nc: int):
    """(J, r): the side rows (per-term, distinct blocks) scattered into one dense Jacobian over the reduced columns."""
    off = column_offsets(pb)
    Js, rs = [], []
    for t, (r, J, ok) in zip(pb.side_terms, rows):
        D = np.zeros((t.nres, nc))
        c = 0
        for b in smp.distinct_blocks(t):
            n = pb.block_size(*b)
            if b in off:
                D[:, off[b]:off[b] + n] = J[:, c:c + n]
            c += n
        Js.append(D)
        rs.append(r)
    return np.vstack(Js), np.concatenate(rs)


def dense_colnorm_gradient(pb, rows, nc):
    J, r = dense_jacobian(pb, rows, nc)
    return np.sum(J * J, axis=0), J.T @ r


def prior_rows(pb: bp.BAProblem, nc: int) -> np.ndarray:
    """Jacobian rows of the camera priors of the free cameras (the problems here hold their priors at the current
    values: residual 0; focal on a log scale)."""
    off = column_offsets(pb)
    o = pb.cam_off
    rows = []
    for k in range(len(pb.cam_type)):
        if (bp.SB_CAM, k) not in off:
            continue
        for j in range(o[k], o[k + 1]):
            d = 1.0 / max(pb.cam_prior_sigma[j], np.finfo(np.float64).eps)
            row = np.zeros(nc)
            row[off[(bp.SB_CAM, k)] + j - o[k]] = d / pb.cam_params[j] if pb.cam_prior_log[j] else d
            rows.append(row)
    return np.array(rows).reshape(-1, nc)


def dense_system(pb: bp.BAProblem, rows, nc: int, scale: np.ndarray, diag: np.ndarray, radius: float):
    """From the mpmath rows: column norms, gradient, and the damped, Jacobi-scaled system S, rhs the LM iteration
    solves with the given scale, LM diagonal and radius (no points: S = Js^T Js + D / radius, rhs = Js^T r)."""
    J, r = dense_jacobian(pb, rows, nc)
    P = prior_rows(pb, nc)
    JJ = J.T @ J + P.T @ P
    cn = np.diag(JJ).copy()
    g = J.T @ r
    S = scale[:, None] * JJ * scale[None, :] + np.diag(diag / radius)
    return cn, g, S, scale * g


def system_errors(cn, g, S, rhs, want, cost):
    """Worst relative errors of (column norms, gradient, S, rhs) against want = dense_system(...)."""
    cn_w, g_w, S_w, rhs_w = want
    # |g_j| <= |J_j| |r| and |r|^2 <= 2 cost.  A column that is 0 in exact arithmetic but the sum of two cancelling
    # copies in fp64 (an instance's translation under a common position of two of its cameras) holds round-off of
    # about eps |J|: it is measured against 1e-12 of the largest column, (1e-12)^2 of the largest column norm
    gscale = np.abs(g_w) + np.sqrt(cn_w * 2.0 * cost)
    cscale = np.maximum(cn_w, 1e-24 * np.max(cn_w))
    gscale = np.maximum(gscale, 1e-12 * np.max(gscale))
    d = np.sqrt(np.diag(S_w))
    return (float(np.max(np.abs(cn - cn_w) / cscale)),
            float(np.max(np.abs(g - g_w) / gscale)),
            float(np.max(np.abs(S - S_w) / np.outer(d, d))),
            float(np.max(np.abs(rhs - rhs_w)) / np.max(np.abs(rhs_w))))


def ra_scene() -> bp.BAProblem:
    """Every ReconstructionAlignment constraint, through the ReconstructionAlignment API."""
    from opensfm_b200 import alignment

    rng = np.random.RandomState(21)
    ra = alignment.ReconstructionAlignment()
    for s in range(4):
        ra.add_shot("s%d" % s, *pose(rng, 1.0), s == 0)
    for k in range(3):
        ra.add_reconstruction("r%d" % k, *rotvec(rng, 0.5), *rng.normal(0, 1, 3), rng.uniform(0.7, 1.5), False)
    for s in range(4):
        rm = alignment.RARelativeMotionConstraint("r%d" % (s % 3), "s%d" % s, *pose(rng, 1.0))
        for i in range(6):
            rm.set_scale_matrix(i, i, rng.uniform(0.5, 2))
        ra.add_relative_motion_constraint(rm)
        ra.add_absolute_position_constraint("s%d" % s, *rng.normal(0, 1, 3), 0.5)
        ra.add_relative_absolute_position_constraint("r%d" % (s % 3), "s%d" % s, *rng.normal(0, 1, 3), 0.7)
    for a, b in ((0, 1), (1, 2), (2, 0)):
        ra.add_common_point_constraint("r%d" % a, *rng.normal(0, 1, 3), "r%d" % b, *rng.normal(0, 1, 3), 0.3)
        ra.add_common_camera_constraint("r%d" % a, "s%d" % a, "r%d" % b, "s%d" % b, 0.4, 0.2)
    pb = ra.to_problem()
    pb.max_iterations = 1
    return pb


def system_scene(name: str) -> bp.BAProblem:
    """One small scene per side-term type (six random terms on their own blocks), the RA scene, and a scene of terms
    that list one rig instance twice."""
    if name == "ra_alignment":
        return ra_scene()
    if name == "duplicate_instance":
        B = Builder()
        edge_cases(B)
        keep = [k for k, n in enumerate(B.names) if n.startswith("duplicate_instance/")]
        B.terms, B.names = [B.terms[k] for k in keep], [B.names[k] for k in keep]
        return B.problem()
    ty = {v: k for k, v in TYPE_NAMES.items()}[name]
    return random_builder([ty], 6, seed=5).problem()


SYSTEM_SCENES = sorted(TYPE_NAMES.values()) + ["ra_alignment", "duplicate_instance"]
# worst (column norm, gradient, S, rhs) error of the oracle's system against the one built from the mpmath rows, over
# SYSTEM_SCENES but duplicate_instance: 5.2e-14; the bound is at most 100x that.  duplicate_instance: its cancelling
# columns hold fp64 round-off (worst 3.2e-5 on the floors above); summing the copies' norms instead puts O(1) there.
MP_SYSTEM_TOL = 5e-12
DUPLICATE_SYSTEM_TOL = 3e-3


def mp_system_tol(name: str) -> float:
    return DUPLICATE_SYSTEM_TOL if name == "duplicate_instance" else MP_SYSTEM_TOL


def oracle_system(pb):
    """The oracle's (cost, column norms, gradient, S, rhs, scale, diag) at iteration 1 of a solve of pb."""
    ob = oracle.OracleBA(pb)
    cost = ob.linearize()
    cn, g = ob.colnorm_gradient()
    scale = 1.0 / (1.0 + np.sqrt(cn))
    diag = np.clip(cn * scale * scale, 1e-6, 1e32)
    ob.set_scale(scale)
    S, rhs = ob.schur(diag / 1e4)
    return ob, cost, cn, g, S, rhs, scale, diag


@pytest.mark.parametrize("name", SYSTEM_SCENES)
def test_oracle_system_matches_mpmath_rows(name):
    """Column norms, gradient, S and rhs of the oracle against the dense system of the mpmath rows (the comparison a
    mistake shared by the oracle and the engine cannot pass)."""
    pb = system_scene(name)
    ob, cost, cn, g, S, rhs, scale, diag = oracle_system(pb)
    errs = system_errors(cn, g, S, rhs, dense_system(pb, mp_rows(pb), ob.nc, scale, diag, 1e4), cost)
    print("%s: colnorm %.1e grad %.1e S %.1e rhs %.1e" % ((name,) + errs))
    assert max(errs) <= mp_system_tol(name), (name, errs)


def test_zero_scale_relative_motion_fails_with_zero_rows_and_nan_cost():
    """RelativeMotionError returns false on a zero scale: its rows are 0 and the cost is NaN (the step is rejected)."""
    B = Builder()
    rng = np.random.RandomState(4)
    s0 = B.add_ext(0.0, True, [0.0])
    B.add("zero_scale", bp.relative_motion_term(B.add_inst(pose(rng)), B.add_inst(pose(rng)), s0, s0,
                                                np.r_[rotvec(rng), 1, 0, 0, 1], np.eye(7), True, bp.LOSS_SOFTLONE, 1.0))
    pb = B.problem()
    assert not mp_rows(pb)[0][2]
    cost, r, J = oracle.OracleBA(pb).side_rows(pb)
    assert math.isnan(cost) and np.all(r == 0) and np.all(J == 0), (cost, r, J)
