"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product.

CPU restatement of the reference's bundle-adjustment solve: the trust-region
Levenberg-Marquardt loop that `ceres::Solve` runs for
`bundle::BundleAdjuster::Run` (opensfm/src/bundle/src/bundle_adjuster.cc:1104-1113)
with the options the reference sets (linear solver SPARSE_SCHUR -> exact Schur
elimination of the points + Cholesky of the reduced camera system,
`max_num_iterations`, everything else Ceres defaults).

Ceres Solver is a third-party dependency that is NOT in the OpenSfM tree
(pinned: conda `ceres-solver=2.1`, conda.yml:10; Docker ubuntu24 libceres-dev
2.2.0).  Its published algorithm (Ceres docs "Solving non-linear least squares"
/ trust_region_minimizer.cc / levenberg_marquardt_strategy.cc, summarised in
SURVEY.md §8c) is restated here:

* cost = 1/2 sum_blocks rho(|r_block|^2); robustification by sqrt(rho') scaling
  (rho'' <= 0 for every loss the reference can select);
* Jacobi column scaling 1/(1+|J_j|) computed once from the first Jacobian;
* LM diagonal D = clamp(diag(J^T J), 1e-6, 1e32), system (J^T J + D/radius);
  initial radius 1e4, max 1e16; D is reused after a rejected step;
* step quality rho = cost_change / model_cost_change; accept iff rho > 1e-3;
  accept: radius /= max(1/3, 1 - (2 rho - 1)^3), decrease_factor = 2;
  reject: radius /= decrease_factor, decrease_factor *= 2;
* termination: function_tolerance 1e-6, gradient_tolerance 1e-10,
  parameter_tolerance 1e-8, max iterations, <= 5 consecutive invalid steps.

The heavy per-observation pieces are in ba_oracle.cpp (OpenMP); the Cholesky of
the reduced system is LAPACK through scipy.  Parity status: the solver
*trajectory* is unpinned by the reference (no reference test pins Ceres
iterates); the converged solution is pinned by tolerance tests only
(opensfm/test/test_bundle.py:116-165).  See oracle/README.md.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import time
from typing import Any, Dict, Optional

import numpy as np
import scipy.linalg

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libba_oracle.so")

LOSS_IDS = {"TrivialLoss": 0, "HuberLoss": 1, "SoftLOneLoss": 2, "CauchyLoss": 3, "ArctanLoss": 4}

_c_int_p = ctypes.POINTER(ctypes.c_int)
_c_dbl_p = ctypes.POINTER(ctypes.c_double)


def build(force: bool = False) -> str:
    """Compile oracle/_build/libba_oracle.so (g++, a few seconds)."""
    src = [os.path.join(_HERE, f) for f in ("ba_oracle.cpp", "ba_functors.hpp", "ba_side_terms.hpp", "Makefile")]
    if force or not os.path.exists(_LIB_PATH) or any(
        os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in src
    ):
        subprocess.check_call(["make", "-C", _HERE, "-B"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = ctypes.CDLL(_LIB_PATH)
        L.oba_create.restype = ctypes.c_void_p
        L.oba_cost.restype = ctypes.c_double
        L.oba_linearize.restype = ctypes.c_double
        L.oba_x_norm.restype = ctypes.c_double
        L.oba_model_cost_change.restype = ctypes.c_double
        L.oracle_side_rows.restype = ctypes.c_double
        L.oracle_reproj_analytic.restype = ctypes.c_int
        L.oracle_reproj_autodiff.restype = ctypes.c_int
        L.oracle_camera_num_params.restype = ctypes.c_int
        _lib = L
    return _lib


def _d(a: np.ndarray):
    return a.ctypes.data_as(_c_dbl_p)


def _i(a: np.ndarray):
    return a.ctypes.data_as(_c_int_p)


def camera_num_params(ptype: int) -> int:
    return lib().oracle_camera_num_params(int(ptype))


def project(ptype: int, params, point) -> np.ndarray:
    p = np.ascontiguousarray(params, dtype=np.float64)
    x = np.ascontiguousarray(point, dtype=np.float64)
    out = np.zeros(2)
    lib().oracle_project(int(ptype), _d(p), _d(x), _d(out))
    return out


def reprojection(ptype, camera, rig_instance, rig_camera, use_rig_camera, point, observed, sigma,
                 autodiff=False):
    """Residual and Jacobian blocks of one observation (analytic or dual-number)."""
    C = camera_num_params(ptype)
    cam = np.ascontiguousarray(camera, dtype=np.float64)
    ri = np.ascontiguousarray(rig_instance, dtype=np.float64)
    rc = np.ascontiguousarray(rig_camera if rig_camera is not None else np.zeros(6), dtype=np.float64)
    pt = np.ascontiguousarray(point, dtype=np.float64)
    ob = np.ascontiguousarray(observed, dtype=np.float64)
    r = np.zeros(3)
    jc = np.zeros(3 * max(C, 1))
    ji = np.zeros(18)
    jrc = np.zeros(18)
    jp = np.zeros(9)
    fn = lib().oracle_reproj_autodiff if autodiff else lib().oracle_reproj_analytic
    n = fn(int(ptype), _d(cam), _d(ri), _d(rc), int(bool(use_rig_camera)), _d(pt), _d(ob),
           ctypes.c_double(sigma), _d(r), _d(jc), _d(ji), _d(jrc), _d(jp))
    return (r[:n].copy(), jc[: n * C].reshape(n, C).copy(), ji[: n * 6].reshape(n, 6).copy(),
            jrc[: n * 6].reshape(n, 6).copy(), jp[: n * 3].reshape(n, 3).copy())


def loss(name: str, a: float, s: float):
    out = np.zeros(2)
    lib().oracle_loss(LOSS_IDS[name], ctypes.c_double(a), ctypes.c_double(s), _d(out))
    return out


class OracleBA:
    """Holds one problem (duck-typed SoA, see opensfm_b200/ba_problem.py) on the C side."""

    def __init__(self, pb: Any):
        L = lib()
        c32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        self._keep = [
            c32(pb.cam_type), f64(pb.cam_params), c32(pb.cam_const), f64(pb.cam_prior),
            f64(pb.cam_prior_sigma), c32(pb.cam_prior_log), f64(pb.inst), c32(pb.inst_const),
            c32(pb.inst_has_prior), f64(pb.inst_prior_pos), f64(pb.inst_prior_std), f64(pb.rigcam),
            c32(pb.rigcam_const), c32(pb.shot_inst), c32(pb.shot_cam), c32(pb.shot_rc),
            c32(pb.shot_use_rc), f64(pb.points), c32(pb.point_const), c32(pb.obs_shot),
            c32(pb.obs_point), f64(pb.obs_xy), f64(pb.obs_sigma),
        ]
        k = self._keep
        if pb.loss_name not in LOSS_IDS:
            # bundle_adjuster.cc:427
            raise RuntimeError("ceres::LossFunction with name %s not found." % pb.loss_name)
        self.K, self.NI, self.NR = len(k[0]), len(k[6]) // 6 if k[6].ndim == 1 else k[6].shape[0], k[11].shape[0] if k[11].ndim == 2 else len(k[11]) // 6
        self.S, self.P, self.N = len(k[13]), k[17].shape[0], len(k[19])
        self.h = ctypes.c_void_p(L.oba_create(
            self.K, _i(k[0]), _d(k[1]), _i(k[2]), _d(k[3]), _d(k[4]), _i(k[5]),
            self.NI, _d(k[6]), _i(k[7]), _i(k[8]), _d(k[9]), _d(k[10]),
            self.NR, _d(k[11]), _i(k[12]),
            self.S, _i(k[13]), _i(k[14]), _i(k[15]), _i(k[16]),
            self.P, _d(k[17]), _i(k[18]),
            ctypes.c_int64(self.N), _i(k[19]), _i(k[20]), _d(k[21]), _d(k[22]),
            LOSS_IDS[pb.loss_name], ctypes.c_double(pb.loss_threshold)))
        self._set_secondary(pb)
        self.nc = L.oba_nc(self.h)
        self.npf = L.oba_npts_free(self.h)
        k2 = self._keep2
        # a free ext parameter with a finite lower bound makes the problem "constrained" (Ceres: is_constrained)
        self.constrained = bool(np.any(np.repeat(k2[2] == 0, k2[0]) & np.isfinite(k2[3]))) if len(k2[0]) else False
        self.n = self.nc + 3 * self.npf
        self.ncamp = len(k[1])

    def _set_secondary(self, pb: Any) -> None:
        """Ext blocks, side terms, point priors and rig-camera priors of the problem (duck-typed: the fields of
        opensfm_b200.ba_problem.BAProblem; absent fields = none)."""
        c32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        ext_size = c32(getattr(pb, "ext_size", np.zeros(0)))
        ext_values = f64(getattr(pb, "ext_values", np.zeros(0)))
        ext_const = c32(getattr(pb, "ext_const", np.zeros(0)))
        ext_lower = f64(getattr(pb, "ext_lower", np.zeros(0)))
        recs, consts = pb.packed_side_terms() if hasattr(pb, "packed_side_terms") else ([], np.zeros(0))
        ints = np.zeros((max(len(recs), 1), 21), dtype=np.int32)
        loss_a = np.ones(max(len(recs), 1))
        for t, (ty, nres, nb, kind, idx, loss, la, cofs, aux) in enumerate(recs):
            ints[t] = [ty, nres, nb] + list(kind) + list(idx) + [loss, cofs] + list(aux)
            loss_a[t] = la
        consts = f64(consts)
        pp_point = c32(getattr(pb, "pp_point", np.zeros(0)))
        pp_prior = f64(getattr(pb, "pp_prior", np.zeros((0, 3))))
        pp_sigma = f64(getattr(pb, "pp_sigma", np.zeros((0, 3))))
        pp_alt = c32(getattr(pb, "pp_alt", np.zeros(0)))
        rcp = getattr(pb, "rigcam_prior", None)
        rc_prior = f64(rcp if rcp is not None else np.zeros((1, 6)))
        rc_sigma = f64(pb.rigcam_prior_sigma if rcp is not None else np.ones((1, 6)))
        self.n_ext = int(ext_size.sum())
        self._keep2 = [ext_size, ext_values, ext_const, ext_lower, ints, loss_a, consts, pp_point, pp_prior, pp_sigma,
                       pp_alt, rc_prior, rc_sigma]
        lib().oba_set_secondary(self.h, len(ext_size), _i(ext_size), _d(ext_values), _i(ext_const), _d(ext_lower),
                                len(recs), _i(ints), _d(loss_a), len(consts), _d(consts), len(pp_point), _i(pp_point),
                                _d(pp_prior), _d(pp_sigma), _i(pp_alt), int(rcp is not None), _d(rc_prior), _d(rc_sigma))

    def __del__(self):
        try:
            lib().oba_destroy(self.h)
        except Exception:
            pass

    def get_ext(self):
        ext = np.zeros(self.n_ext)
        lib().oba_get_ext(self.h, _d(ext))
        return ext

    def get_params(self):
        cam = np.zeros(self.ncamp)
        inst = np.zeros((self.NI, 6))
        rc = np.zeros((self.NR, 6))
        pts = np.zeros((self.P, 3))
        lib().oba_get_params(self.h, _d(cam), _d(inst), _d(rc), _d(pts))
        return cam, inst, rc, pts, self.get_ext()

    def set_params(self, cam, inst, rc, pts, ext=None):
        lib().oba_set_params(self.h, _d(np.ascontiguousarray(cam)), _d(np.ascontiguousarray(inst)),
                             _d(np.ascontiguousarray(rc)), _d(np.ascontiguousarray(pts)))
        if ext is not None and len(ext):
            lib().oba_set_ext(self.h, _d(np.ascontiguousarray(ext)))

    def plus(self, delta):
        lib().oba_plus(self.h, _d(np.ascontiguousarray(delta)))

    def x_norm(self) -> float:
        return lib().oba_x_norm(self.h)

    def cost(self, want_reproj=False):
        if want_reproj:
            out = np.zeros((self.N, 3))
            c = lib().oba_cost(self.h, _d(out))
            return c, out
        return lib().oba_cost(self.h, None)

    def linearize(self) -> float:
        return lib().oba_linearize(self.h)

    def colnorm_gradient(self):
        cn = np.zeros(self.n)
        g = np.zeros(self.n)
        lib().oba_colnorm_gradient(self.h, _d(cn), _d(g))
        return cn, g

    def side_rows(self, pb: Any):
        """(cost, r, J) of the side terms at the current parameters: robustified rows packed per term like
        BAProblem.side_row_sizes (oracle_side_rows)."""
        nrow, nJ = pb.side_row_sizes()
        r, J = np.zeros(int(nrow.sum())), np.zeros(int(nJ.sum()))
        cost = lib().oracle_side_rows(self.h, _d(r), _d(J))
        return cost, r, J

    def set_scale(self, s):
        lib().oba_set_scale(self.h, _d(np.ascontiguousarray(s)))

    def schur(self, diag2):
        S = np.zeros((self.nc, self.nc))
        rhs = np.zeros(self.nc)
        lib().oba_schur(self.h, _d(diag2), _d(S), _d(rhs))
        return S, rhs

    def backsub(self, diag2, y):
        lib().oba_backsub(self.h, _d(diag2), _d(y))

    def model_cost_change(self, step) -> float:
        return lib().oba_model_cost_change(self.h, _d(step))


def solve(pb: Any, max_iterations: Optional[int] = None, verbose: bool = False,
          stop_after_iterations: Optional[int] = None) -> Dict[str, Any]:
    """Run the restated Ceres LM on problem `pb`.  Returns the solution and a summary.

    stop_after_iterations bounds the work for timing samples (bench cpu_baseline).
    """
    ba = OracleBA(pb)
    max_it = pb.max_iterations if max_iterations is None else max_iterations
    # Ceres defaults
    radius, max_radius, min_radius = 1e4, 1e16, 1e-32
    min_diag, max_diag = 1e-6, 1e32
    min_rel_decrease = 1e-3
    ftol, gtol, ptol = 1e-6, 1e-10, 1e-8
    decrease_factor = 2.0
    reuse_diagonal = False
    n_invalid = 0
    t0 = time.perf_counter()

    cost = ba.linearize()
    cn, g = ba.colnorm_gradient()
    scale = 1.0 / (1.0 + np.sqrt(cn))
    ba.set_scale(scale)
    x_norm = ba.x_norm()
    grad_max = float(np.max(np.abs(g))) if g.size else 0.0
    initial_cost = cost
    it = 0
    n_success = 0
    n_lin_solves = 0
    termination = "NO_CONVERGENCE"
    message = ""
    diag = None
    log = [(0, cost, 0.0, grad_max, 0.0, radius)]
    if grad_max <= gtol:
        termination, message = "CONVERGENCE", "Gradient tolerance reached."
    while termination == "NO_CONVERGENCE":
        if it >= max_it:
            message = "Maximum number of iterations reached."
            break
        if stop_after_iterations is not None and it >= stop_after_iterations:
            message = "stopped (bounded sample)"
            break
        if radius < min_radius:
            termination, message = "CONVERGENCE", "Minimum trust region radius reached."
            break
        it += 1
        if not reuse_diagonal:
            diag = np.clip(cn * scale * scale, min_diag, max_diag)
        diag2 = diag / radius  # (lm_diagonal)^2
        S, rhs = ba.schur(diag2)
        n_lin_solves += 1
        ok = True
        try:
            cf = scipy.linalg.cho_factor(S, lower=True, overwrite_a=True, check_finite=False)
            y = np.zeros(ba.n)
            y[: ba.nc] = scipy.linalg.cho_solve(cf, rhs, check_finite=False)
            ba.backsub(diag2, y)
            step = -y
            ok = bool(np.all(np.isfinite(step)))
        except np.linalg.LinAlgError:
            ok = False
        model_change = ba.model_cost_change(step) if ok else -1.0
        if not ok or model_change <= 0.0:
            n_invalid += 1
            if n_invalid >= 5:
                termination, message = "FAILURE", "Too many consecutive invalid steps."
                break
            radius *= 0.5
            reuse_diagonal = True
            log.append((it, cost, 0.0, grad_max, 0.0, radius))
            continue
        n_invalid = 0
        delta = step * scale
        saved = ba.get_params()
        if ba.constrained:
            # Ceres: bounds make the problem "constrained" and TrustRegionMinimizer::DoLineSearch runs a projected
            # Armijo search along the step before the candidate is evaluated (sufficient decrease 1e-4, at most 20
            # contractions).  Interpolation here is BISECTION (step *= 0.5); Ceres' default fits a
            # cubic -- the accepted step differs, the fixed points do not.  model_cost_change stays that of the
            # full step, as in Ceres.
            g0 = float(np.dot(g, delta))
            alpha, ok_ls = 1.0, False
            for _ in range(20):
                ba.set_params(*saved)
                ba.plus(alpha * delta)
                c = ba.cost()
                if np.isfinite(c) and c <= cost + 1e-4 * g0 * alpha:
                    ok_ls = True
                    break
                alpha *= 0.5
            if not ok_ls:
                alpha = 1.0
            delta = alpha * delta
            ba.set_params(*saved)
        ba.plus(delta)
        cand_cost = ba.cost()
        if ba.constrained:
            # Ceres: step_norm = |x - candidate_x|, i.e. the step actually taken after projection onto the bounds
            step_norm = float(np.sqrt(sum(((a - b) ** 2).sum() for a, b in zip(ba.get_params(), saved))))
        else:
            step_norm = float(np.linalg.norm(delta))
        if step_norm <= ptol * (x_norm + ptol):
            # Ceres leaves x at the pre-step value on parameter-tolerance exit
            ba.set_params(*saved)
            termination, message = "CONVERGENCE", "Parameter tolerance reached."
            break
        cost_change = cost - cand_cost
        if abs(cost_change) <= ftol * cost:
            # Ceres checks function tolerance before accepting the step: x stays at the previous point
            ba.set_params(*saved)
            termination, message = "CONVERGENCE", "Function tolerance reached."
            break
        rel = cost_change / model_change
        if rel > min_rel_decrease:
            cost = ba.linearize()
            cn, g = ba.colnorm_gradient()
            x_norm = ba.x_norm()
            grad_max = float(np.max(np.abs(g)))
            radius = min(max_radius, radius / max(1.0 / 3.0, 1.0 - (2.0 * rel - 1.0) ** 3))
            decrease_factor = 2.0
            reuse_diagonal = False
            n_success += 1
            log.append((it, cost, cost_change, grad_max, step_norm, radius))
            if grad_max <= gtol:
                termination, message = "CONVERGENCE", "Gradient tolerance reached."
                break
        else:
            ba.set_params(*saved)
            radius /= decrease_factor
            decrease_factor *= 2.0
            reuse_diagonal = True
            log.append((it, cost, cost_change, grad_max, step_norm, radius))
        if verbose:
            print("it %3d cost %.9e change %.3e |g| %.3e radius %.3e" % (it, cost, cost_change, grad_max, radius))
    run_time = time.perf_counter() - t0
    final_cost, reproj = ba.cost(want_reproj=True)
    cam, inst, rc, pts, ext = ba.get_params()
    return {
        "cam_params": cam, "inst": inst, "rigcam": rc, "points": pts, "ext_values": ext,
        "reprojection_errors": reproj,
        "initial_cost": initial_cost, "final_cost": final_cost,
        "iterations": it, "successful_steps": n_success, "linear_solves": n_lin_solves,
        "termination": termination, "message": message, "time_run": run_time, "log": log,
    }
