"""High-precision reference for the bundle adjuster's side terms (test infrastructure, not a test module).

Each of the 17 residuals is restated here in mpmath from the reference's functors -- bundle/error/
absolute_motion_errors.h, relative_motion_errors.h, motion_prior_errors.h, parameters_errors.h, position_functors.h,
prior_error.h with data/bias.h's SimilarityPriorTransform, and reconstruction_alignment.h -- with the ceres rotation
helpers they call (ceres/rotation.h: AngleAxisToQuaternion, QuaternionProduct, QuaternionToAngleAxis,
AngleAxisRotatePoint) including every branch, and the thresholds the functors compare against in double.  Its
Jacobian is taken by central differences at 40 significant digits, on the branches taken at the point (as ceres::Jet
does), with respect to the DISTINCT parameter blocks of a term: a block a term lists twice (two shots of one rig
instance) is one set of columns.  Nothing here is shared with the engine (opensfm_b200/csrc/ba_side.cuh) or the oracle
(oracle/ba_side_terms.hpp), so a mistake the two share shows.

Terms are opensfm_b200.ba_problem.SideTerm records: the block order, constants and aux indices of
include/opensfm_b200.h."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
from mpmath import mp, mpf

from opensfm_b200 import ba_problem as bp

DIGITS = 40
DBL_EPSILON = float(np.finfo(np.float64).eps)
# the functors compare against the double M_PI and add / subtract the double 2 * M_PI
M_PI, TWO_M_PI = mpf(math.pi), mpf(2 * math.pi)


class _Branches:
    """ceres::Jet compares values only, so an autodiff derivative is that of the branch taken at the point, even where
    the point sits on a threshold (std::max(T(0), m) at m = 0, a guard).  rows() records every decision at the point
    and replays it at the perturbed points, which differentiates the same branch."""

    def __init__(self):
        self.log, self.replay, self.pos = [], False, 0

    def __call__(self, cond) -> bool:
        if not self.replay:
            self.log.append(bool(cond))
            return bool(cond)
        self.pos += 1
        return self.log[self.pos - 1]


_branches = None


def br(cond) -> bool:
    return _branches(cond) if _branches is not None else bool(cond)


# ---- ceres/rotation.h ----------------------------------------------------------------------------
def aa_to_quat(a):
    th2 = a[0] * a[0] + a[1] * a[1] + a[2] * a[2]
    if br(th2 > 0):
        th = mp.sqrt(th2)
        k = mp.sin(th / 2) / th
        return [mp.cos(th / 2), a[0] * k, a[1] * k, a[2] * k]
    return [mpf(1), a[0] / 2, a[1] / 2, a[2] / 2]


def quat_product(z, w):
    return [z[0] * w[0] - z[1] * w[1] - z[2] * w[2] - z[3] * w[3],
            z[0] * w[1] + z[1] * w[0] + z[2] * w[3] - z[3] * w[2],
            z[0] * w[2] - z[1] * w[3] + z[2] * w[0] + z[3] * w[1],
            z[0] * w[3] + z[1] * w[2] - z[2] * w[1] + z[3] * w[0]]


def quat_to_aa(q):
    s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    if br(s2 > 0):
        s, c = mp.sqrt(s2), q[0]
        two_theta = 2 * (mp.atan2(-s, -c) if br(c < 0) else mp.atan2(s, c))
        k = two_theta / s
    else:
        k = mpf(2)
    return [q[1] * k, q[2] * k, q[3] * k]


def cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def rotate(aa, p):
    th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2]
    if br(th2 > DBL_EPSILON):
        th = mp.sqrt(th2)
        c, s = mp.cos(th), mp.sin(th)
        w = [x / th for x in aa]
        wxp = cross(w, p)
        tmp = (w[0] * p[0] + w[1] * p[1] + w[2] * p[2]) * (1 - c)
        return [p[i] * c + wxp[i] * s + w[i] * tmp for i in range(3)]
    wxp = cross(aa, p)
    return [p[i] + wxp[i] for i in range(3)]


# ---- error_utils.h / position_functors.h ---------------------------------------------------------------
def mult_rotations(*Rs):
    q = aa_to_quat(Rs[0])
    for R in Rs[1:]:
        q = quat_product(q, aa_to_quat(R))
    return quat_to_aa(q)


def neg(v):
    return [-x for x in v]


def sub(a, b):
    return [x - y for x, y in zip(a, b)]


def shot_rotation(inst, rc):
    return list(inst[:3]) if rc is None else mult_rotations(inst[:3], rc[:3])


def shot_position(inst, rc):
    t = list(inst[3:6])
    return t if rc is None else [x + y for x, y in zip(t, rotate(inst[:3], rc[3:6]))]


def diff_between_angles(a, b):
    d = a - b
    if br(d > M_PI):
        return d - TWO_M_PI
    if br(d < -M_PI):
        return d + TWO_M_PI
    return d


def norm(v):
    return mp.sqrt(sum(x * x for x in v))


def matvec(m, v):
    return [sum(m[i][j] * v[j] for j in range(len(v))) for i in range(len(m))]


# reconstruction_alignment.h transform_point: world point -> frame of a reconstruction [R | t | scale]
def transform_point(rec, point):
    p = [(point[k] - rec[3 + k]) / rec[6] for k in range(3)]
    return rotate(neg(rec[:3]), p)


def shot_centre(shot):   # -R^t t of a [R | t] world-to-camera shot
    return neg(rotate(neg(shot[:3]), shot[3:6]))


# ---- the functors ---------------------------------------------------------------------------------------
def residual(t: bp.SideTerm, x: List[list]) -> Optional[list]:
    """Unrobustified residual of term t with x[b] = values of its b-th listed block; None where the functor returns
    false (relative motion with a zero scale)."""
    c = [mpf(float(v)) for v in np.asarray(t.consts, dtype=np.float64).ravel()]
    aux = list(t.aux) + [-1] * (4 - len(t.aux))
    rc_of = lambda k: x[aux[k]] if aux[k] >= 0 else None
    ez = [mpf(0), mpf(0), mpf(1)]
    ty = t.type
    if ty == bp.SIDE_UP_VECTOR:
        z = rotate(shot_rotation(x[0], x[1]), c[0:3])
        return [c[3] * (z[0] - 0), c[3] * (z[1] - 0), c[3] * (z[2] - 1)]
    if ty == bp.SIDE_PAN:
        z = rotate(shot_rotation(x[0], x[1]), ez)
        if br(abs(z[0]) < 1e-8 and abs(z[1]) < 1e-8):
            return [mpf(0)]
        return [c[1] * diff_between_angles(mp.atan2(z[0], z[1]), c[0])]
    if ty == bp.SIDE_TILT:
        z = rotate(shot_rotation(x[0], x[1]), ez)
        l = mp.sqrt(z[0] * z[0] + z[1] * z[1])
        return [c[1] * diff_between_angles(-mp.atan2(z[2], l), c[0])]
    if ty == bp.SIDE_ROLL:
        R = shot_rotation(x[0], x[1])
        Rt_ex, Rt_ez = rotate(R, [mpf(1), mpf(0), mpf(0)]), rotate(R, ez)
        a = [Rt_ez[1], -Rt_ez[0], mpf(0)]
        la = mp.sqrt(a[0] * a[0] + a[1] * a[1])
        eps = 1e-5
        if br(la < eps):
            return [mpf(0)]
        a = [a[0] / la, a[1] / la, a[2]]
        b = cross(Rt_ex, a)
        sin_roll = Rt_ez[0] * b[0] + Rt_ez[1] * b[1] + Rt_ez[2] * b[2]
        if br(sin_roll <= -(1.0 - eps)):
            return [mpf(0)]
        return [c[1] * diff_between_angles(mp.asin(sin_roll), c[0])]
    if ty == bp.SIDE_RELATIVE_MOTION:
        Ri, ti, Rj, tj = x[0][:3], x[0][3:6], x[1][:3], x[1][3:6]
        si, sj = x[2][0], x[aux[0]][0]
        e = mult_rotations(c[0:3], neg(Ri), Rj)
        rt = rotate(neg(Rj), sub(ti, tj))
        e += [c[3 + k] - sj * rt[k] for k in range(3)]
        if si == 0 or sj == 0:
            return None
        e.append(c[6] - sj / si if c[56] != 0 else mpf(0))
        return matvec([c[7 + 7 * i:14 + 7 * i] for i in range(7)], e)
    if ty == bp.SIDE_RELATIVE_ROTATION:
        Ri, Rj = shot_rotation(x[0], rc_of(0)), shot_rotation(x[1], rc_of(1))
        return matvec([c[3 + 3 * i:6 + 3 * i] for i in range(3)], mult_rotations(c[0:3], neg(Ri), Rj))
    if ty == bp.SIDE_COMMON_POSITION:
        e = sub(shot_position(x[0], rc_of(0)), shot_position(x[1], rc_of(1)))
        for i in range(2):
            m = abs(e[i]) - c[0]
            e[i] = m if br(m > 0) else mpf(0)   # std::max(T(0), m)
        return [c[1] * v for v in e]
    if ty == bp.SIDE_LINEAR_MOTION:
        R = [shot_rotation(x[k], rc_of(k)) for k in range(3)]
        p = [shot_position(x[k], rc_of(k)) for k in range(3)]
        t20, t10 = sub(p[2], p[0]), sub(p[1], p[0])
        n20, n10 = norm(t20), norm(t10)
        far = br(n20 > 1e-15)
        r = [c[1] * (c[0] - n10 / n20) if far else c[1] * (c[0] * t20[i] - t10[i]) for i in range(3)]
        A = [c[0] * v for v in mult_rotations(R[2], neg(R[0]))]
        B = mult_rotations(R[0], neg(R[1]))
        return r + [c[2] * v for v in mult_rotations(A, B)]
    if ty == bp.SIDE_TRANSLATION_PRIOR:
        d = sub(x[0][3:6], x[1][3:6])
        return [mp.log(mp.sqrt(sum(v * v for v in d) + mpf(1e-20)) / c[0])]
    if ty == bp.SIDE_PARAMETER_BARRIER:
        eps = mpf(1e-10)
        value = x[0][aux[0]]
        zero = 2 * mp.log((c[1] - c[0]) * mpf(0.5))
        return [mp.log(value - c[0] + eps) + mp.log(c[1] - value + eps) + zero]
    if ty == bp.SIDE_STD_DEVIATION:
        return [mp.log(1 / mp.sqrt(mpf(2.0 * math.pi) * (x[0][0] * x[0][0] + mpf(1e-20))))]
    if ty == bp.SIDE_POSITION_PRIOR:
        inst, bias, sd = x[0], x[1], x[2]
        rp = rotate(bias[:3], c[0:3])
        out = []
        for k in range(3):
            scale = c[3 + k] / sd[0] if c[6] != 0 else c[3 + k]
            out.append(scale * (inst[3 + k] - (bias[6] * rp[k] + bias[3 + k])))
        return out
    if ty == bp.SIDE_RA_RELATIVE_MOTION:
        rec, shot = x[0], x[1]
        Rit = neg(shot[:3])
        q = quat_product(aa_to_quat(c[0:3]), quat_product(aa_to_quat(rec[:3]), aa_to_quat(Rit)))
        e = quat_to_aa(q)
        a, d = rotate(neg(c[0:3]), c[3:6]), rotate(rec[:3], rotate(Rit, shot[3:6]))
        e += [a[k] - rec[6] * d[k] + rec[3 + k] for k in range(3)]
        return matvec([c[6 + 6 * i:12 + 6 * i] for i in range(6)], e)
    if ty == bp.SIDE_RA_ABSOLUTE_POSITION:
        v = rotate(neg(x[0][:3]), x[0][3:6])
        return [c[3] * (c[k] + v[k]) for k in range(3)]
    if ty == bp.SIDE_RA_RELATIVE_ABSOLUTE_POSITION:
        tr = transform_point(x[0], shot_centre(c[3:9]))
        return [c[9] * (c[k] - tr[k]) for k in range(3)]
    if ty == bp.SIDE_RA_COMMON_POINT:
        ta, tb = transform_point(x[0], c[0:3]), transform_point(x[1], c[3:6])
        sf = x[0][6] + x[1][6]
        return [c[6] * sf * (ta[k] - tb[k]) for k in range(3)]
    if ty == bp.SIDE_RA_COMMON_CAMERA:
        wa, wb = transform_point(x[0], shot_centre(c[0:6])), transform_point(x[1], shot_centre(c[6:12]))
        q = quat_product(aa_to_quat(c[0:3]), aa_to_quat(x[0][:3]))
        q = quat_product(q, aa_to_quat(neg(x[1][:3])))
        q = quat_product(q, aa_to_quat(neg(c[6:9])))
        e = quat_to_aa(q)
        return [e[k] * c[13] for k in range(3)] + [c[12] * (wa[k] - wb[k]) for k in range(3)]
    raise ValueError("unknown side term type %d" % ty)


def loss_derivative(loss: int, a: float, s):
    """rho'(s) of the term's loss (ceres: Huber, SoftLOne, Cauchy, Arctan; Tukey for common position; none)."""
    a = mpf(a)
    b = a * a
    if loss == bp.LOSS_NONE or loss == 0:
        return mpf(1)
    if loss == 1:
        return mpf(1) if s <= b else a / mp.sqrt(s)
    if loss == bp.LOSS_SOFTLONE:
        return 1 / mp.sqrt(1 + s / b)
    if loss == bp.LOSS_CAUCHY:
        return 1 / (1 + s / b)
    if loss == 4:
        return 1 / (1 + s * s / b)
    if loss == bp.LOSS_TUKEY:
        return (1 - s / b) ** 2 if s <= b else mpf(0)
    raise ValueError("unknown loss %d" % loss)


def distinct_blocks(t: bp.SideTerm) -> List[Tuple[int, int]]:
    return list(dict.fromkeys(tuple(b) for b in t.blocks))


def _column(f, x0, b, q):
    """Central difference of f along parameter q of block b, on the branches recorded at x0."""
    h = mpf(10) ** (-(DIGITS // 2)) * max(1, abs(x0[b][q]))
    xp, xm = dict(x0), dict(x0)
    xp[b], xm[b] = list(x0[b]), list(x0[b])
    xp[b][q] += h
    xm[b][q] -= h
    _branches.pos = 0
    fp = f(xp)
    _branches.pos = 0
    fm = f(xm)
    return [(u - v) / (2 * h) for u, v in zip(fp, fm)]


def rows(t: bp.SideTerm, values: Dict[Tuple[int, int], Sequence[float]]):
    """Robustified rows of term t at the (double) block values `values[(kind, idx)]`: (r, J, ok) as float64, J with
    one column per parameter of the distinct blocks (distinct_blocks order).  Ceres' corrector for rho'' <= 0:
    r <- sqrt(rho') r, J <- sqrt(rho') J.  ok = False where the functor fails (then r, J are None)."""
    global _branches
    with mp.workdps(DIGITS):
        blocks = distinct_blocks(t)
        x0 = {b: [mpf(float(v)) for v in values[b]] for b in blocks}
        f = lambda xs: residual(t, [xs[tuple(b)] for b in t.blocks])
        _branches = _Branches()
        try:
            r0 = f(x0)
            if r0 is None:
                return None, None, False
            _branches.replay = True
            cols = [_column(f, x0, b, q) for b in blocks for q in range(len(x0[b]))]
        finally:
            _branches = None
        s = sum(v * v for v in r0)
        w = mp.sqrt(loss_derivative(t.loss, t.loss_a, s))
        r = np.array([float(w * v) for v in r0])
        J = np.array([[float(w * col[k]) for col in cols] for k in range(len(r0))]).reshape(len(r0), len(cols))
        return r, J, True


def fold_columns(t: bp.SideTerm, J_local: np.ndarray, sizes: Sequence[int]) -> np.ndarray:
    """Columns of a term's local Jacobian (one set per listed block, sizes[b] wide) summed onto its distinct blocks,
    the layout rows() returns."""
    blocks = distinct_blocks(t)
    start = np.concatenate([[0], np.cumsum(sizes)])
    dstart = {}
    off = 0
    for b in blocks:
        dstart[b] = off
        off += sizes[[tuple(x) for x in t.blocks].index(b)]
    out = np.zeros((J_local.shape[0], off))
    for k, b in enumerate(t.blocks):
        out[:, dstart[tuple(b)]:dstart[tuple(b)] + sizes[k]] += J_local[:, start[k]:start[k + 1]]
    return out
