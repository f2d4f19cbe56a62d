"""Absolute-pose RANSAC of one shot in numpy: the CPU restatement that opensfm_b200/csrc/resect.cu (and the solvers of
opensfm_b200/csrc/absolute_pose.cuh) are checked against.

What it restates: pyrobust's `ransac_absolute_pose` with RANSAC scoring as `multiview.absolute_pose_ransac` calls it
(only `iterations` is set, so the stopping rule uses probability 0.99), followed by the chord inliers of
`reconstruction.resect`:

  * rows: a bearing, normalised (instanciations.cc), and a world point;
  * the sample stream, the draws and the stopping bound of the rotation RANSAC (rotation_ransac_oracle): mt19937(42)
    restarted for every shot, 3-row samples;
  * the model: P3P of Ke and Roumeliotis (geometry/absolute_pose.h).  No model when sigma = 0, when k3 . b3 = 0 or
    when the quartic's closed form is degenerate; otherwise 4 models, one per root in root order.  A root is the real
    part of foundation::SolveQuartic's complex-pow closed form (principal branches), refined by 5 Newton steps with
    tolerance 1e-20.  The rotation goes through ClosestRotationMatrix (the polar factor, negated if improper); a root
    with |cos| > 1 gives a NaN model, which has no inliers;
  * the error 1 - b . normalize(R X + t), an inlier when its absolute value is below 1 - cos(threshold);
  * the model loop of robust_estimator.h: models scored in order, a model replaces the best one when it has at least
    as many inliers; whenever one does with at least 3 inliers, 10 rounds of local optimisation, each drawing
    max(min(12, floor(inliers / 2)), 3) positions of the best inlier list (ascending rows) and fitting Lu's
    orthogonal iteration (AbsolutePoseNPoints: at most 100 steps, stopping when the relative change of the
    translation is below 1e-7, from a scaled Horn start); the stopping rule after every model with the outer
    iteration index, so a sample can stop the loop part-way through its models;
  * the result [R | t] = lo_model (world to camera); the chord inliers ||normalize(R (X - o)) - b|| < threshold,
    o = -R^T t the camera origin.

Deliberate differences from pyrobust, shared with the engine:
  * rows come in the order the caller gives them (the engine: ascending track index); pyrobust's follow an
    unordered_map's iteration order, which nothing in OpenSfM defines, so against pyrobust only order-independent
    known answers are claimed;
  * a 3-row rotation fit (LO samples of a best model with fewer than 8 inliers, and the Horn start of Lu's
    iteration on them) uses rotation_ransac_oracle.rotation_between's proper completion, where pyrobust's
    RotationBetweenPoints is decided by round-off;
  * a bearing is normalised once; pyrobust normalises it again in every error, which changes it by an ulp at most.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from .rotation_ransac_oracle import (LO_ITERATIONS, LO_SAMPLE_CLAMP, MINIMAL_SAMPLES, SampleStream, cofactor,
                                     polar, rotation_between, sample, stop_bound)

QUARTIC_NEWTON_STEPS = 5
QUARTIC_NEWTON_TOLERANCE = 1e-20
LU_MAX_ITERATIONS = 100
LU_TOLERANCE = 1e-7
EPS = float(np.finfo(np.float64).eps)


# ---------------------------------------------------------------------------------------------------------------
# P3P (Ke and Roumeliotis)
# ---------------------------------------------------------------------------------------------------------------
def _cx_pow(z: complex, y: float) -> complex:
    """std::pow(complex, real): the real pow for a positive real z, else polar(exp(y log|z|), y arg z)."""
    if z.imag == 0.0 and z.real > 0.0:
        return complex(math.pow(z.real, y), 0.0)
    lr = math.log(math.hypot(z.real, z.imag)) if (z.real or z.imag) else -math.inf
    th = math.atan2(z.imag, z.real)
    rho, phi = math.exp(y * lr), y * th
    return complex(rho * math.cos(phi), rho * math.sin(phi))


def _cx_div(a: complex, b: complex) -> complex:
    d = b.real * b.real + b.imag * b.imag
    if d == 0.0:
        return complex(math.nan, math.nan)
    return complex((a.real * b.real + a.imag * b.imag) / d, (a.imag * b.real - a.real * b.imag) / d)


def solve_quartic(coef) -> Optional[List[float]]:
    """foundation::SolveQuartic: the 4 real parts of the closed form, or None when it is degenerate.  coef[k] is the
    coefficient of x^k."""
    c4, c3, c2, c1, c0 = (float(coef[k]) for k in (4, 3, 2, 1, 0))
    a = c4 if abs(c4) > EPS else EPS
    b, c, d, e = c3 / a, c2 / a, c1 / a, c0 / a
    Q1 = c * c - 3. * b * d + 12. * e
    Q2 = 2. * c * c * c - 9. * b * c * d + 27. * d * d + 27. * b * b * e - 72. * c * e
    Q3 = 8. * b * c - 16. * d - 2. * b * b * b
    Q4 = 3. * b * b - 8. * c
    if abs(Q1) < EPS and abs(Q2) < EPS and abs(Q3) < EPS and abs(Q4) < EPS:
        return None
    Q5 = _cx_pow(complex(Q2 / 2.) + _cx_pow(complex(Q2 * Q2 / 4. - Q1 * Q1 * Q1), 1. / 2.), 1. / 3.)
    Q6 = (_cx_div(complex(Q1), Q5) + Q5) / 3.
    Q7 = 2. * _cx_pow(complex(Q4 / 12.) + Q6, 1. / 2.)
    Q3Q7 = _cx_div(complex(Q3), Q7)
    base = complex(4. * Q4 / 6.) - 4. * Q6
    s1, s2 = _cx_pow(base - Q3Q7, 1. / 2.), _cx_pow(base + Q3Q7, 1. / 2.)
    return [(-b - Q7 - s1).real / 4., (-b - Q7 + s1).real / 4., (-b + Q7 - s2).real / 4., (-b + Q7 + s2).real / 4.]


def refine_root(coef, x: float) -> float:
    """RefineQuarticRoots: 5 Newton steps, stopping when the step is below 1e-20 (or the derivative is 0)."""
    c = [float(v) for v in coef]
    for _ in range(QUARTIC_NEWTON_STEPS):
        f = (((c[4] * x + c[3]) * x + c[2]) * x + c[1]) * x + c[0]
        x2 = x * x
        x3 = x2 * x
        df = 4.0 * c[4] * x3 + 3.0 * c[3] * x2 + 2.0 * c[2] * x + c[1]
        decr = 0.0 if df == 0.0 else f / df
        if abs(decr) < QUARTIC_NEWTON_TOLERANCE:
            break
        x -= decr
    return x


def rotation_around_axis(c: float, s: float, v) -> np.ndarray:
    omc = 1.0 - c
    return np.array([[c + v[0] * v[0] * omc, v[2] * s + v[0] * v[1] * omc, -v[1] * s + v[0] * v[2] * omc],
                     [-v[2] * s + v[0] * v[1] * omc, c + v[1] * v[1] * omc, v[0] * s + v[1] * v[2] * omc],
                     [v[1] * s + v[0] * v[2] * omc, -v[0] * s + v[1] * v[2] * omc, c + v[2] * v[2] * omc]])


def closest_rotation(X: np.ndarray) -> Optional[np.ndarray]:
    Q = polar(X)
    if Q is None:
        return None
    return -Q if np.linalg.det(Q) < 0.0 else Q


def p3p_coefficients(b: np.ndarray, p: np.ndarray):
    """(coefficients, g1..g7, sigma, k3_b3, c_barre, c_barre_barre) of a 3-row sample, or None when it has no model."""
    b1, b2, b3 = b
    p1, p2, p3 = p
    k1 = p1 - p2
    k1 = k1 / np.sqrt(k1 @ k1)
    k3 = np.cross(b1, b2)
    b1_b2 = float(np.sqrt(k3 @ k3))
    k3 = k3 / b1_b2
    u1, u2 = p1 - p3, p2 - p3
    v1, v2 = np.cross(b1, b3), np.cross(b2, b3)
    u1_k1 = np.cross(u1, k1)
    sigma = float(np.sqrt(u1_k1 @ u1_k1))
    if sigma == 0.0:
        return None
    k3s = u1_k1 / sigma
    k3_b3 = float(k3 @ b3)
    if k3_b3 == 0.0:
        return None
    b1b2 = float(b1 @ b2)
    f11 = sigma * k3_b3
    f21 = sigma * b1b2 * k3_b3
    f22 = sigma * k3_b3 * b1_b2
    f13 = sigma * float(v1 @ k3)
    f23 = sigma * float(v2 @ k3)
    f24 = float(u2 @ k1) * k3_b3 * b1_b2
    f15 = -float(u1 @ k1) * k3_b3
    f25 = -float(u2 @ k1) * b1b2 * k3_b3
    g1 = f13 * f22
    g2 = f13 * f25 - f15 * f23
    g3 = f11 * f23 - f13 * f21
    g4 = -f13 * f24
    g5 = f11 * f22
    g6 = f11 * f25 - f15 * f21
    g7 = -f15 * f24
    coef = [g7 * g7 - g2 * g2 - g4 * g4,
            2.0 * (g6 * g7 - g1 * g2 - g3 * g4),
            g6 * g6 + 2.0 * g5 * g7 + g2 * g2 + g4 * g4 - g1 * g1 - g3 * g3,
            2.0 * (g5 * g6 + g1 * g2 + g3 * g4),
            g5 * g5 + g1 * g1 + g3 * g3]
    cb = np.column_stack([k1, k3s, np.cross(k1, k3s)])
    cbb = np.array([b1, k3, np.cross(b1, k3)])
    return coef, (g1, g2, g3, g4, g5, g6, g7), sigma, k3_b3, cb, cbb


def p3p(b: np.ndarray, p: np.ndarray) -> List[np.ndarray]:
    """AbsolutePoseThreePoints: [] or 4 poses [R | t] (3 x 4, world to camera), one per root in root order."""
    b = np.asarray(b, dtype=np.float64).reshape(3, 3)
    p = np.asarray(p, dtype=np.float64).reshape(3, 3)
    co = p3p_coefficients(b, p)
    if co is None:
        return []
    coef, (g1, g2, g3, g4, g5, g6, g7), sigma, k3_b3, cb, cbb = co
    roots = solve_quartic(coef)
    if roots is None:
        return []
    sgn = -1.0 if k3_b3 < 0.0 else 1.0
    out = []
    for root in roots:
        cos1 = refine_root(coef, root)
        one = 1.0 - cos1 * cos1
        sin1 = sgn * math.sqrt(one) if one >= 0.0 else math.nan
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            t = float(np.float64(sin1) / np.float64(g5 * cos1 * cos1 + g6 * cos1 + g7))
            cos3 = t * (g1 * cos1 + g2)
            sin3 = t * (g3 * cos1 + g4)
            M = cb @ rotation_around_axis(cos1, sin1, (1.0, 0.0, 0.0)) @ rotation_around_axis(cos3, sin3, (0.0, 1.0, 0.0)) @ cbb
        R = closest_rotation(M)
        if R is None:
            out.append(np.full((3, 4), np.nan))
            continue
        tr = p[2] - (sigma * sin1) / k3_b3 * (R @ b[2])
        out.append(np.column_stack([R.T, -(R.T @ tr)]))
    return out


# ---------------------------------------------------------------------------------------------------------------
# Lu's orthogonal iteration (AbsolutePoseNPoints)
# ---------------------------------------------------------------------------------------------------------------
def lu_pose(b: np.ndarray, p: np.ndarray, margins: Optional[list] = None) -> np.ndarray:
    """[R | t] of k rows from a scaled Horn start; `margins` collects |relative change - 1e-7| of every step."""
    b = np.asarray(b, dtype=np.float64).reshape(-1, 3)
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    k = len(b)
    qbar = b[0].copy()
    pbar = p[0].copy()
    for i in range(1, k):
        qbar += b[i]
        pbar += p[i]
    qbar /= k
    pbar /= k
    s_num = s_den = 0.0
    for i in range(k):
        s_num += float(np.sqrt(np.sum((p[i] - pbar) ** 2))) ** 2
        s_den += float(np.sqrt(np.sum((b[i] - qbar) ** 2))) ** 2
    scale = math.sqrt(s_num / s_den)
    R = rotation_between(b, p)
    t = scale * qbar - R @ pbar
    F = np.einsum("ir,ic->irc", b, b) / np.einsum("ic,ic->i", b, b)[:, None, None]
    I3 = np.eye(3)
    for _ in range(LU_MAX_ITERATIONS):
        q = np.einsum("irc,ic->ir", F, p @ R.T + t)
        R = rotation_between(q, p)
        F1 = F.sum(axis=0) / k
        F2 = np.einsum("irc,ic->r", F - I3, p @ R.T) / k
        A = I3 - F1
        C = cofactor(A)   # A^-1 = cof(A)^T / det(A), as the engine inverts it
        new_t = (C.T @ F2) / float(A[:, 0] @ C[:, 0])
        rel = float(np.linalg.norm(new_t - t) / np.linalg.norm(t))
        if margins is not None:
            margins.append(abs(rel - LU_TOLERANCE))
        if rel < LU_TOLERANCE:
            break
        t = new_t
    return np.column_stack([R, t])


# ---------------------------------------------------------------------------------------------------------------
# the estimator
# ---------------------------------------------------------------------------------------------------------------
def errors(model: np.ndarray, b: np.ndarray, X: np.ndarray) -> np.ndarray:
    """1 - b . normalize(R X + t)."""
    v = X @ model[:, :3].T + model[:, 3]
    with np.errstate(invalid="ignore"):
        return 1.0 - (b[:, 0] * v[:, 0] + b[:, 1] * v[:, 1] + b[:, 2] * v[:, 2]) / np.sqrt(
            v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2])


def chord(model: np.ndarray, b: np.ndarray, X: np.ndarray) -> np.ndarray:
    """||normalize(R (X - o)) - b||, o = -R^T t: resect's inlier test."""
    R, t = model[:, :3], model[:, 3]
    o = -(R.T @ t)
    v = (X - o) @ R.T
    v = v / np.sqrt(v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2])[:, None]
    d = v - b
    return np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])


@dataclass
class ShotResult:
    lo_model: np.ndarray                 # 3 x 4 [R | t], world to camera
    ransac_inliers: int
    chord_mask: np.ndarray               # bool per row
    chord_inliers: int
    draws: List[int] = field(default_factory=list)   # every drawn sample index (LO: inlier-list positions)
    iterations: int = 0                  # outer iterations run
    stream_used: int = 0                 # raw generator outputs consumed
    error_margin: float = np.inf         # min | |e| - (1 - cos threshold) | over every model evaluated
    stop_margin: float = np.inf          # min | bound - i | over every ShouldStop evaluation
    lu_margin: float = np.inf            # min | relative change - 1e-7 | over every step of Lu's iteration
    chord_margin: float = np.inf         # min | chord - threshold | of the final model

    def pose(self) -> np.ndarray:
        """multiview.absolute_pose_ransac's [R_c2w | origin]."""
        R, t = self.lo_model[:, :3], self.lo_model[:, 3]
        return np.column_stack([R.T, -(R.T @ t)])


def normalize_rows(b: np.ndarray) -> np.ndarray:
    b = np.asarray(b, dtype=np.float64).reshape(-1, 3)
    return b / np.sqrt(b[:, 0] * b[:, 0] + b[:, 1] * b[:, 1] + b[:, 2] * b[:, 2])[:, None]


def ransac_absolute_pose(bs: np.ndarray, Xs: np.ndarray, threshold: float, iterations: int = 1000) -> ShotResult:
    b = normalize_rows(bs)
    X = np.ascontiguousarray(Xs, dtype=np.float64).reshape(-1, 3)
    n = len(b)
    if n < MINIMAL_SAMPLES:
        raise ValueError("absolute pose RANSAC needs at least 3 rows, got %d" % n)
    t_err = 1.0 - np.cos(threshold)
    stream = SampleStream()
    res = ShotResult(np.zeros((3, 4)), 0, np.zeros(n, bool), 0)
    best_inliers = np.zeros(0, dtype=np.int64)
    best = np.zeros((3, 4))
    lu_margins: List[float] = []

    def evaluate(model):
        e = np.abs(errors(model, b, X))
        finite = np.isfinite(e)
        if finite.any():
            res.error_margin = min(res.error_margin, float(np.min(np.abs(e[finite] - t_err))))
        with np.errstate(invalid="ignore"):
            return np.nonzero(e < t_err)[0]

    stop = False
    for i in range(iterations):
        idx = sample(stream, MINIMAL_SAMPLES, n)
        res.draws += idx
        res.iterations = i + 1
        for model in p3p(b[idx], X[idx]):
            inl = evaluate(model)
            if len(inl) >= len(best_inliers):
                best_inliers, best = inl, model
                if len(inl) >= MINIMAL_SAMPLES:
                    for _ in range(LO_ITERATIONS):
                        m = len(best_inliers)
                        size = max(min(LO_SAMPLE_CLAMP, int(m * 0.5)), MINIMAL_SAMPLES)
                        pos = sample(stream, size, m)
                        res.draws += pos
                        rows = best_inliers[pos]
                        lo = lu_pose(b[rows], X[rows], lu_margins)
                        lo_inl = evaluate(lo)
                        if len(lo_inl) >= len(best_inliers):
                            best_inliers, best = lo_inl, lo
            bound = stop_bound(len(best_inliers), n)
            if len(best_inliers) < n:   # all rows inliers: the bound is exactly 0, not a rounding question
                res.stop_margin = min(res.stop_margin, abs(bound - i))
            if bound < i:
                stop = True
                break
        if stop:
            break
    res.lo_model = best
    res.ransac_inliers = len(best_inliers)
    if lu_margins:
        res.lu_margin = min(lu_margins)
    with np.errstate(invalid="ignore"):
        c = chord(best, b, X)
        finite = np.isfinite(c)
        if finite.any():
            res.chord_margin = float(np.min(np.abs(c[finite] - threshold)))
        res.chord_mask = c < threshold
    res.chord_inliers = int(res.chord_mask.sum())
    res.stream_used = stream.cursor
    return res
