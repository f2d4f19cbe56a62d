"""The oracle's reduced camera system against a from-first-principles numpy restatement.

The oracle (oracle/ba_oracle.cpp oba_colnorm_gradient / oba_schur) and the engine were written together, so a
derivation error shared by both would pass every engine-vs-oracle test.  Here the same quantities are formed the
plain way: the full dense robustified Jacobian (per-observation blocks from the dual-number Jacobian, weighted by
sqrt(rho')), the prior rows, the Jacobi scaling 1 / (1 + |J_j|), the LM damping clip(diag(J^T J) s^2, 1e-6, 1e32) / 1e4,
H = Js^T Js + D and S = H_cc - H_cp H_pp^-1 H_pc, rhs = g_c - H_cp H_pp^-1 g_p with numpy.linalg.  Side terms have no
simple numpy restatement; they stay pinned through the oracle and the reference's known-answer tests."""
import numpy as np
import pytest

import ba_linear_system_scenes as scenes
from oracle import ba_lm as oracle
from opensfm_b200 import ba_problem as bp

RADIUS = 1e4


def _layout(pb):
    """Column offsets of the free blocks: [free cameras | free instances | free rig cameras | free points]."""
    cam_np = [bp.camera_num_params(t) for t in pb.cam_type]
    off = 0
    cam_col, inst_col, rc_col = [], [], []
    for k in range(len(pb.cam_type)):
        cam_col.append(-1 if pb.cam_const[k] else off)
        off += 0 if pb.cam_const[k] else cam_np[k]
    for i in range(len(pb.inst)):
        inst_col.append(-1 if pb.inst_const[i] else off)
        off += 0 if pb.inst_const[i] else 6
    for i in range(len(pb.rigcam)):
        rc_col.append(-1 if pb.rigcam_const[i] else off)
        off += 0 if pb.rigcam_const[i] else 6
    nc = off
    pt_col = []
    for p in range(len(pb.points)):
        pt_col.append(-1 if pb.point_const[p] else off)
        off += 0 if pb.point_const[p] else 3
    return nc, off, cam_col, inst_col, rc_col, pt_col


def reference_system(pb):
    """(colnorm2, grad, S, rhs, scale, D) of the first LM iteration, dense numpy."""
    nc, n, cam_col, inst_col, rc_col, pt_col = _layout(pb)
    cam_off = pb.cam_off
    rows_J, rows_r = [], []

    def add_row(r, cols_vals):
        j = np.zeros(n)
        for c, v in cols_vals:
            if c >= 0:
                j[c:c + len(v)] += v
        rows_J.append(j)
        rows_r.append(r)

    for i in range(len(pb.obs_shot)):
        s, p = pb.obs_shot[i], pb.obs_point[i]
        k, ins = pb.shot_cam[s], pb.shot_inst[s]
        use_rc = bool(pb.shot_use_rc[s])
        r, jc, ji, jrc, jp = oracle.reprojection(pb.cam_type[k], pb.cam_params[cam_off[k]:cam_off[k + 1]], pb.inst[ins],
                                                 pb.rigcam[pb.shot_rc[s]], use_rc, pb.points[p], pb.obs_xy[i],
                                                 pb.obs_sigma[i], autodiff=True)
        w = np.sqrt(oracle.loss(pb.loss_name, pb.loss_threshold, float(r @ r))[1])
        for q in range(len(r)):
            blocks = [(cam_col[k], jc[q]), (inst_col[ins], ji[q]), (pt_col[p], jp[q])]
            if use_rc:
                blocks.append((rc_col[pb.shot_rc[s]], jrc[q]))
            add_row(w * r[q], [(c, w * v) for c, v in blocks])
    # camera priors on every free camera parameter: linear, or logarithmic on focal / aspect ratio
    for k in range(len(pb.cam_type)):
        if cam_col[k] < 0:
            continue
        for j in range(cam_off[k + 1] - cam_off[k]):
            x, x0 = pb.cam_params[cam_off[k] + j], pb.cam_prior[cam_off[k] + j]
            sc = 1.0 / max(pb.cam_prior_sigma[cam_off[k] + j], np.finfo(float).eps)
            if pb.cam_prior_log[cam_off[k] + j]:
                add_row(sc * np.log(x / x0), [(cam_col[k] + j, [sc / x])])
            else:
                add_row(sc * (x - x0), [(cam_col[k] + j, [sc])])
    for i in range(len(pb.inst)):   # position priors on the instance translation
        if pb.inst_has_prior[i] and inst_col[i] >= 0:
            for j in range(3):
                sc = 1.0 / max(pb.inst_prior_std[i, j], np.finfo(float).eps)
                add_row(sc * (pb.inst[i, 3 + j] - pb.inst_prior_pos[i, j]), [(inst_col[i] + 3 + j, [sc])])
    if pb.rigcam_prior is not None:   # rig-camera pose priors on free rig cameras
        for i in range(len(pb.rigcam)):
            if rc_col[i] >= 0:
                for j in range(6):
                    sc = 1.0 / max(pb.rigcam_prior_sigma[i, j], np.finfo(float).eps)
                    add_row(sc * (pb.rigcam[i, j] - pb.rigcam_prior[i, j]), [(rc_col[i] + j, [sc])])
    for q, p in enumerate(pb.pp_point):   # point priors: x, y (and z with altitude)
        if pt_col[p] >= 0:
            for j in range(3 if pb.pp_alt[q] else 2):
                sc = 1.0 / max(pb.pp_sigma[q, j], np.finfo(float).eps)
                add_row(sc * (pb.points[p, j] - pb.pp_prior[q, j]), [(pt_col[p] + j, [sc])])
    J, r = np.array(rows_J), np.array(rows_r)
    colnorm2 = (J * J).sum(0)
    grad = J.T @ r
    scale = 1.0 / (1.0 + np.sqrt(colnorm2))
    Js = J * scale
    D = np.clip(colnorm2 * scale * scale, 1e-6, 1e32) / RADIUS
    H = Js.T @ Js + np.diag(D)
    g = Js.T @ r
    Hcc, Hcp, Hpp = H[:nc, :nc], H[:nc, nc:], H[nc:, nc:]
    X = np.linalg.solve(Hpp, np.column_stack([Hcp.T, g[nc:]]))
    S = Hcc - Hcp @ X[:, :nc]
    rhs = g[:nc] - Hcp @ X[:, nc]
    return colnorm2, grad, J, r, S, rhs, scale, D


@pytest.mark.parametrize("name", scenes.CPU_SCENES)
def test_oracle_reduced_system_matches_dense_numpy(name):
    pb = scenes.SCENES[name]()
    cn_ref, g_ref, J, r, S_ref, rhs_ref, scale, D = reference_system(pb)
    ob = oracle.OracleBA(pb)
    ob.linearize()
    cn, g = ob.colnorm_gradient()
    assert cn.shape == cn_ref.shape
    # analytic (oracle) against dual-number (reference) derivatives: fp64 round-off of the column sums
    assert np.all(np.abs(cn - cn_ref) <= 1e-12 * cn_ref), np.max(np.abs(cn - cn_ref) / cn_ref)
    gbound = np.sqrt(cn_ref) * np.linalg.norm(r)   # |g_j| <= |J_j| |r|
    assert np.all(np.abs(g - g_ref) <= 1e-12 * gbound), np.max(np.abs(g - g_ref) / gbound)
    ob.set_scale(scale)
    S, rhs = ob.schur(D)
    d = np.sqrt(np.diag(S_ref))
    ratio = np.abs(S - S_ref) / np.outer(d, d)
    rr = np.abs(rhs - rhs_ref) / np.abs(rhs_ref).max()
    print("%s: nc %d, worst |S - S_ref|_ij / sqrt(S_ii S_jj) %.2e, rhs %.2e" % (name, len(rhs), ratio.max(), rr.max()))
    # measured <= 4e-14 on every scene (S and rhs); the bar is 100x that.  A relative error of 1e-7 in one term
    # of S (e.g. the cross term W V^-1 W^T) is far above it.
    assert ratio.max() <= 4e-12
    assert rr.max() <= 4e-12
