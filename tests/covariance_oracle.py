"""Rig-instance pose covariances restated on the CPU from the oracle's linearisation (test infrastructure).

Ceres' Covariance with the reference's defaults (bundle_adjuster.cc:1123-1194): (J^T J)^-1 of the robustified
Jacobian at the given parameters over every non-constant block, bounds ignored; each rig instance gets its 6x6
diagonal block, constant instances zeros; an invalid estimate gives every instance the default
diag(1e-5, 1e-5, 1e-5, 1e-2, 1e-2, 1e-2).  Rank is decided as the engine decides it (DESIGN.md, covariances): on the
Jacobi-scaled normal equations, a Cholesky pivot <= TAU times the original diagonal entry, first on every point's
3x3 V, then on the reduced camera system S (oracle.ba_lm.OracleBA.schur with no damping).

Not a test module: the covariance tests import it (pytest puts tests/ on sys.path)."""
from __future__ import annotations

import copy
import ctypes

import numpy as np
import scipy.linalg

from oracle import ba_lm as oracle

TAU = 1e-10
DEFAULT = np.diag([1e-5, 1e-5, 1e-5, 1e-2, 1e-2, 1e-2])


def with_params(pb, cam, inst, rigcam, points, ext=None):
    """A copy of problem `pb` at other parameter values."""
    q = copy.copy(pb)
    q.cam_params = np.array(cam, dtype=np.float64)
    q.inst = np.array(inst, dtype=np.float64).reshape(-1, 6)
    q.rigcam = np.array(rigcam, dtype=np.float64).reshape(-1, 6) if len(rigcam) else pb.rigcam
    q.points = np.array(points, dtype=np.float64).reshape(-1, 3)
    if ext is not None and len(ext):
        q.ext_values = np.array(ext, dtype=np.float64)
    return q


def point_rank_deficient(a, b, c, d, e, f) -> bool:
    """The engine's pivot test on the symmetric [[a b c] [b d e] [c e f]] (ba_reduced.cuh point_rank_deficient)."""
    if not a > TAU * a:
        return True
    p1 = d - b * b / a
    if not p1 > TAU * d:
        return True
    q = e - b * c / a
    p2 = f - c * c / a - q * q / p1
    return not p2 > TAU * f


def point_blocks(pb, scale, nc):
    """Scaled, undamped V of every free point: robustified dual-free analytic Jacobians of the oracle plus the
    point-prior rows.  Returns (free point count, V[npf, 3, 3])."""
    L = oracle.lib()
    free = np.flatnonzero(np.asarray(pb.point_const) == 0)
    pf_of = np.full(len(pb.points), -1)
    pf_of[free] = np.arange(len(free))
    V = np.zeros((len(free), 3, 3))
    r, jc, ji, jrc, jp = np.zeros(3), np.zeros(48), np.zeros(18), np.zeros(18), np.zeros(9)
    rho = np.zeros(2)
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    cam_off = pb.cam_off
    cams = [np.ascontiguousarray(pb.cam_params[cam_off[k]:cam_off[k + 1]], dtype=np.float64) for k in range(len(pb.cam_type))]
    inst = np.ascontiguousarray(pb.inst, dtype=np.float64)
    rcs = np.ascontiguousarray(pb.rigcam, dtype=np.float64).reshape(-1, 6)
    pts = np.ascontiguousarray(pb.points, dtype=np.float64)
    xy = np.ascontiguousarray(pb.obs_xy, dtype=np.float64)
    loss_id = oracle.LOSS_IDS[pb.loss_name]
    for i in range(len(pb.obs_shot)):
        p = int(pb.obs_point[i])
        if pf_of[p] < 0:
            continue
        s = int(pb.obs_shot[i])
        k, ins, rc = int(pb.shot_cam[s]), int(pb.shot_inst[s]), int(pb.shot_rc[s])
        n = L.oracle_reproj_analytic(int(pb.cam_type[k]), dp(cams[k]), dp(inst[ins]), dp(rcs[rc]),
                                     int(bool(pb.shot_use_rc[s])), dp(pts[p]), dp(xy[i]),
                                     ctypes.c_double(float(pb.obs_sigma[i])), dp(r), dp(jc), dp(ji), dp(jrc), dp(jp))
        L.oracle_loss(loss_id, ctypes.c_double(pb.loss_threshold), ctypes.c_double(float(r[:n] @ r[:n])), dp(rho))
        J = jp[:3 * n].reshape(n, 3)
        V[pf_of[p]] += rho[1] * (J.T @ J)
    for q, p in enumerate(np.asarray(pb.pp_point, dtype=int)):
        if pf_of[p] >= 0:
            for j in range(3 if pb.pp_alt[q] else 2):
                V[pf_of[p], j, j] += 1.0 / max(pb.pp_sigma[q, j], np.finfo(float).eps) ** 2
    sp = scale[nc:].reshape(-1, 3)
    return len(free), V * sp[:, :, None] * sp[:, None, :]


def covariances(pb, params=None, termination=None):
    """(valid, status, C[NI, 6, 6], info) at `params` = (cam, inst, rigcam, points, ext) or pb's own parameters.
    `termination` "FAILURE" reproduces a failed solve (nothing is computed).  info: the scaled S (instance columns
    last) and the scale, for the tolerance of the engine comparison."""
    NI = len(pb.inst)
    info = {}
    if termination == "FAILURE":
        return False, "solver_failure", np.tile(DEFAULT, (NI, 1, 1)), info
    q = pb if params is None else with_params(pb, *params)
    ob = oracle.OracleBA(q)
    ob.linearize()
    cn, _ = ob.colnorm_gradient()
    scale = 1.0 / (1.0 + np.sqrt(cn))
    ob.set_scale(scale)
    nc = ob.nc
    npf, V = point_blocks(q, scale, nc)
    status = "ok"
    if any(point_rank_deficient(v[0, 0], v[0, 1], v[0, 2], v[1, 1], v[1, 2], v[2, 2]) for v in V):
        status = "point_rank_deficient"
    C = np.zeros((NI, 6, 6))
    if status == "ok" and nc > 0:
        with np.errstate(all="ignore"):
            S, _ = ob.schur(np.zeros(ob.n))
        # column layout of the reduced vector: [free cameras | free instances | free rig cameras | free ext]
        cam_np = np.diff(np.asarray(q.cam_off))
        off = int(sum(cam_np[k] for k in range(len(q.cam_type)) if not q.cam_const[k]))
        inst_col = {}
        for i in range(NI):
            if not q.inst_const[i]:
                inst_col[i] = off
                off += 6
        icols = np.array([inst_col[i] + j for i in sorted(inst_col) for j in range(6)], dtype=int)
        lead = np.setdiff1d(np.arange(nc), icols)
        perm = np.concatenate([lead, icols])
        Sp = S[np.ix_(perm, perm)]
        info["S"], info["scale"] = Sp, scale[:nc][perm]
        try:
            Lc = scipy.linalg.cholesky(Sp, lower=True, check_finite=False)
            ok = bool(np.all(np.isfinite(Lc)) and np.all(np.diag(Lc) ** 2 > TAU * np.diag(Sp)))
        except np.linalg.LinAlgError:
            ok = False
        if not ok:
            status = "camera_rank_deficient"
        elif len(icols):
            m = len(icols)
            X = scipy.linalg.solve_triangular(Lc[-m:, -m:], np.eye(m), lower=True)
            for qq, i in enumerate(sorted(inst_col)):
                Xi = X[:, 6 * qq:6 * qq + 6]
                s = scale[inst_col[i]:inst_col[i] + 6]
                C[i] = (Xi.T @ Xi) * s[:, None] * s[None, :]
            if not np.all(np.isfinite(C)):
                status = "non_finite"
    if status != "ok":
        C = np.tile(DEFAULT, (NI, 1, 1))
    return status == "ok", status, C, info


def solve(pb):
    """oracle.ba_lm.solve plus the covariances at its solution, in the result layout of bundle.solve(...,
    compute_covariances=True): the oracle backend of BundleAdjuster.apply_results."""
    res = oracle.solve(pb)
    params = (res["cam_params"], res["inst"], res["rigcam"], res["points"], res["ext_values"])
    valid, status, C, _ = covariances(pb, params, termination=res["termination"])
    res["summary"] = {"iterations": res["iterations"], "initial_cost": res["initial_cost"],
                      "final_cost": res["final_cost"], "termination": res["termination"]}
    res.update(covariances=C, covariance_valid=valid, covariance_status=status)
    return res
