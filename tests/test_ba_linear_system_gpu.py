"""The engine's reduced camera system and PCG step, kernel path by kernel path, against the oracle.

Every scene captures LM iteration 1 (osfm_ba_capture_linear_system) and checks
  * scale, LM diagonal and gradient against OracleBA.colnorm_gradient (1e-12 relative);
  * the damped reduced system S and its rhs against OracleBA.schur fed with the engine's own scale and diagonal:
    |S_e - S_o|_ij <= TAU sqrt(S_o,ii S_o,jj), |rhs_e - rhs_o|_i <= TAU |rhs_o|_inf, every entry the oracle fills is
    stored, and the stored S_e (upper and lower blocks expanded from their own storage) is exactly symmetric;
  * the PCG solution: |S_e y - rhs_e| <= 1.5e-8 |rhs_e| (the engine's stopping bar), the same on the oracle's system
    within the margin the difference of the two systems allows, and no rescue by the classic PCG;
  * the camera and point step of a max_iterations=1 solve against the oracle's;
  * the kernel path the scene is named for.
The same scenes run on every fallback path (bundle.solve(fallbacks=...)), each compared against the oracle.

The segment chunk list, and with it ba_schur_pipe, ba_linearize_fused and ba_colnorm_grad_chunks, exists for camera
sides 9 wide with 2 residual rows only (whichever Schur kernel runs): wc < 9 needs a camera with fewer than 3
parameters, i.e. SPHERICAL (wc = 7, 3 residuals), so such problems run ba_schur_mma<0> and ba_colnorm_grad_seg<0>.
Scenes with FISHEYE624 or BROWN plus rig cameras (wc > 16) have no segment-eligible point at all and run the per-point
ba_schur only."""
import functools

import numpy as np
import pytest
import scipy.linalg

import ba_linear_system_scenes as scenes
from oracle import ba_lm as oracle
from opensfm_b200 import bundle

pytestmark = pytest.mark.gpu

PCG_BAR = 1.5e-8
# worst |S_e - S_o|_ij / sqrt(S_o,ii S_o,jj) and |rhs_e - rhs_o|_i / |rhs_o|_inf measured on every scene and every
# variant (H100, fp64 sums of at most ~100 terms in a different order): TAU is at most 100x that
TAU = 5e-12   # measured worst 1.3e-13 over all scenes and variants, H100


def _num_sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _oracle_system(pb, cap):
    ob = oracle.OracleBA(pb)
    cost = ob.linearize()
    cn, g = ob.colnorm_gradient()
    ob.set_scale(cap["scale"])
    S, rhs = ob.schur(cap["diag"] / cap["radius"])
    return ob, cost, cn, g, S, rhs


def measure(name, variant=""):
    """Capture iteration 1 of scene `name` with max_iterations=1 on the fallback paths of `variant` (a key of
    VARIANTS, "" for the default path) and compare with the oracle.  Returns the metrics; the asserts live in the
    callers."""
    pb = scenes.SCENES[name]()
    pb.max_iterations = 1
    res = bundle.solve(pb, capture_iteration=1, fallbacks=VARIANTS[variant] if variant else ())
    cap = res["capture"]
    ob, cost, cn, g, S_o, rhs_o = _oracle_system(pb, cap)
    nc, S_e, rhs_e, y = cap["nc"], cap["S"], cap["rhs"], cap["y"]
    m = {k: cap[k] for k in ("nc", "n", "wc", "nres", "nseg", "p_fast", "p_slow", "schur_kernel", "sp_nchunks",
                             "pcg_kernel", "pcg_rescued", "pcg_iterations")}
    m["name"], m["variant"] = name, variant
    m["n_oracle"] = ob.n
    # iteration 1 is linearised at the caller's parameters
    m["x_capture_err"] = max(float(np.max(np.abs(cap["x"][k] - np.asarray(getattr(pb, a)).reshape(cap["x"][k].shape))))
                             if cap["x"][k].size else 0.0
                             for k, a in (("cam_params", "cam_params"), ("inst", "inst"), ("points", "points"),
                                          ("ext_values", "ext_values")))
    scale_o = 1.0 / (1.0 + np.sqrt(cn))
    diag_o = np.clip(cn * scale_o * scale_o, 1e-6, 1e32)
    m["scale_err"] = float(np.max(np.abs(cap["scale"] - scale_o) / scale_o))
    m["diag_err"] = float(np.max(np.abs(cap["diag"] - diag_o) / diag_o))
    # |g_j| <= |J_j| |r~| and |r~|^2 <= 2 cost for every loss (rho' s <= rho): the scale of a gradient entry
    # (a free point without observations has an empty column: gradient exactly 0 on both sides)
    gscale = np.abs(g) + np.sqrt(cn * 2.0 * cost)
    gerr = np.abs(cap["grad"] - g)
    m["grad_err"] = float(np.max(np.where(gscale > 0, gerr / np.where(gscale > 0, gscale, 1.0), np.where(gerr > 0, np.inf, 0.0))))
    d = np.sqrt(np.diag(S_o))
    m["S_ratio"] = float(np.max(np.abs(S_e - S_o) / np.outer(d, d)))
    m["rhs_ratio"] = float(np.max(np.abs(rhs_e - rhs_o)) / np.max(np.abs(rhs_o)))
    m["missing_entries"] = int(np.count_nonzero((S_o != 0) & (S_e == 0)))
    m["asymmetric_entries"] = int(np.count_nonzero(S_e != S_e.T))
    m["pcg_res"] = float(np.linalg.norm(S_e @ y - rhs_e) / np.linalg.norm(rhs_e))
    res_o = np.linalg.norm(S_o @ y - rhs_o)
    # |S_o y - rhs_o| <= |S_e y - rhs_e| + |S_e - S_o|_F |y| + |rhs_e - rhs_o|  (triangle inequality)
    m["pcg_res_oracle"] = float(res_o / np.linalg.norm(rhs_e))
    m["pcg_res_oracle_bar"] = float((PCG_BAR * np.linalg.norm(rhs_e) + np.linalg.norm(S_e - S_o) * np.linalg.norm(y) +
                                     np.linalg.norm(rhs_e - rhs_o)) / np.linalg.norm(rhs_e))
    # step: |y_e - y_o| <= |S_o^-1| |S_o y_e - rhs_o|, propagated exactly to the parameters by the oracle's
    # back-substitution and update
    y_o = scipy.linalg.cho_solve(scipy.linalg.cho_factor(S_o), rhs_o)
    lam_min = float(scipy.linalg.eigvalsh(S_o, subset_by_index=[0, 0])[0])
    m["cond"] = float(scipy.linalg.eigvalsh(S_o, subset_by_index=[nc - 1, nc - 1])[0] / lam_min)
    m["y_err"] = float(np.linalg.norm(y - y_o))
    m["y_err_bar"] = float(1.01 * res_o / lam_min + 1e-14 * np.linalg.norm(y_o))

    def params_after(yc):
        b = oracle.OracleBA(pb)
        b.linearize()
        b.colnorm_gradient()
        b.set_scale(cap["scale"])
        full = np.zeros(b.n)
        full[:nc] = yc
        b.backsub(cap["diag"] / cap["radius"], full)
        b.plus(-full * cap["scale"])
        c, i, _, p, e = b.get_params()
        return np.concatenate([c, i.ravel(), p.ravel(), e])

    def dmax(a, b):
        return float(np.max(np.abs(a - b))) if a.size else 0.0

    def flat(r):
        return np.concatenate([r["cam_params"], r["inst"].ravel(), r["points"].ravel(), r["ext_values"]])

    x_e, x_o = params_after(y), params_after(y_o)
    x0 = np.concatenate([pb.cam_params, pb.inst.ravel(), pb.points.ravel(), pb.ext_values])
    ref = oracle.solve(pb, max_iterations=1)
    m["accepted"] = int(res["summary"]["successful_steps"])
    m["accepted_oracle"] = int(ref["successful_steps"])
    step = dmax(x_o, x0)
    got, want = flat(res), flat(ref)
    if name == "side_terms":
        # the ext-block columns (reconstruction scales) and the block of two instances that share no point, which
        # only side_enum_pairs puts into the structure
        K, NI = len(pb.cam_type), len(pb.inst)
        m["ext_cols"] = nc - (3 * K + 6 * NI)
        a, b = scenes.instances_sharing_no_point(pb)[0]
        ia, ib = 3 * K + 6 * a, 3 * K + 6 * b
        m["apart_block"] = float(np.max(np.abs(S_e[ia:ia + 6, ib:ib + 6])))
        m["apart_block_oracle"] = float(np.max(np.abs(S_o[ia:ia + 6, ib:ib + 6])))
    # engine parameters against the oracle's update of the engine's own y (back-substitution, update kernels)
    m["own_step_err"] = dmax(got, x_e) / step if m["accepted"] else dmax(got, x0)
    # engine against oracle.solve: the PCG error propagated exactly to the parameters, plus fp64 round-off
    m["step_err"] = dmax(got, want)
    m["step_err_bar"] = dmax(x_e, x_o) + 1e-10 * step
    return m


def check(m, tau=TAU):
    tag = "%s [%s]" % (m["name"], m["variant"] or "default")
    assert m["n"] == m["n_oracle"], tag
    assert m["x_capture_err"] == 0.0, (tag, m)
    assert m["scale_err"] <= 1e-12 and m["diag_err"] <= 1e-12 and m["grad_err"] <= 1e-12, (tag, m)
    assert m["S_ratio"] <= tau and m["rhs_ratio"] <= tau, (tag, m)
    assert m["missing_entries"] == 0 and m["asymmetric_entries"] == 0, (tag, m)
    assert m["pcg_res"] <= PCG_BAR, (tag, m)
    assert m["pcg_res_oracle"] <= m["pcg_res_oracle_bar"], (tag, m)
    assert not m["pcg_rescued"], (tag, m)
    assert m["y_err"] <= m["y_err_bar"], (tag, m)
    assert m["accepted"] == m["accepted_oracle"], (tag, m)
    assert m["own_step_err"] <= 1e-10, (tag, m)
    assert m["step_err"] <= m["step_err_bar"], (tag, m)


def _report(m):
    print("%-28s %-22s schur %-12s chunks %5d seg %5d slow %5d pcg %-18s its %4d res %.2e S %.2e rhs %.2e grad %.1e "
          "cond %.1e step %.1e/%.1e" % (
              m["name"], m["variant"] or "default", m["schur_kernel"], m["sp_nchunks"], m["nseg"], m["p_slow"],
              m["pcg_kernel"], m["pcg_iterations"], m["pcg_res"], m["S_ratio"], m["rhs_ratio"], m["grad_err"],
              m["cond"], m["step_err"], m["step_err_bar"]))


# what each scene must reach on the default path
EXPECT = {
    "pipe_many_chunks": dict(schur_kernel="pipe", wc=9, nres=2),
    "pipe_few_chunks": dict(schur_kernel="pipe", wc=9, nres=2),
    "c2_size": dict(schur_kernel="pipe", nc=450),
    "shared_intrinsics": dict(schur_kernel="pipe"),
    "constant_blocks": dict(schur_kernel="pipe"),
    "brown_simt_segments": dict(schur_kernel="simt_segment", wc=15),
    "rig_free_rigcam_priors": dict(schur_kernel="none", wc=21),
    "rig_segments": dict(schur_kernel="simt_segment", wc=15),
    "side_terms": dict(schur_kernel="pipe", wc=9),
    "spherical": dict(schur_kernel="mma", wc=7, nres=3),
    "all_ten_models": dict(schur_kernel="none", wc=22, nres=3),
    "point_priors_many_obs": dict(schur_kernel="none", wc=9),
    "camera_and_position_priors": dict(schur_kernel="pipe"),
    "cauchy_outliers": dict(schur_kernel="pipe"),
    "huber_outliers": dict(schur_kernel="pipe"),
    "duplicate_observations": dict(schur_kernel="pipe"),
    "fixed_instances": dict(schur_kernel="pipe", pcg_kernel="pipelined"),
    "pipe_long_runs": dict(schur_kernel="pipe", wc=9, nres=2, nseg=8, p_slow=0),
    "pipe_k_edge": dict(schur_kernel="pipe", wc=9, nres=2, p_fast=150, p_slow=150),
    "unobserved_and_idle": dict(schur_kernel="pipe", wc=9, nres=2, p_slow=20),
}


@pytest.mark.parametrize("name", sorted(scenes.SCENES))
def test_reduced_system_matches_oracle(name):
    m = measure(name)
    _report(m)
    for k, v in EXPECT[name].items():
        assert m[k] == v, (name, k, m)
    if "pcg_kernel" not in EXPECT[name]:
        assert m["pcg_kernel"] == "pipelined_deflated", m
    sms = _num_sms()
    if name == "pipe_many_chunks":
        assert m["sp_nchunks"] > sms and m["sp_nchunks"] > m["nseg"], m   # more chunks than SMs, multi-chunk segments
    if name == "pipe_few_chunks":
        assert 0 < m["sp_nchunks"] < sms, m
    if name in ("brown_simt_segments", "rig_segments"):
        assert m["p_fast"] > 0 and m["p_slow"] > 0, m   # points with 7 or more shots fall to the per-point ba_schur
    if name == "point_priors_many_obs":
        pb = scenes.SCENES[name]()
        assert np.bincount(pb.obs_point).max() > 16 and m["p_slow"] > 0, m
    if name == "constant_blocks":
        assert m["nseg"] > 0, m
    if name == "side_terms":
        # 8 free reconstruction scales; the relative motion / common position of instances that share no point fill
        # their block in the engine's S as in the oracle's
        assert m["ext_cols"] == 8 and m["apart_block"] > 0 and m["apart_block_oracle"] > 0, m
    check(m)


def test_iteration_two_uses_the_chunked_linearisation():
    """Iteration 2 (after an accepted step) computes column norms and gradient over the segment chunk list
    (ba_linearize_fused: the scene is all perspective).  The oracle
    is linearised at the parameters the engine linearised at (captured with the system), so the comparison is as
    exact as at iteration 1."""
    pb = scenes.SCENES["pipe_many_chunks"]()
    pb.max_iterations = 2
    res = bundle.solve(pb, capture_iteration=2)
    cap = res["capture"]
    assert cap["iteration"] == 2 and cap["schur_kernel"] == "pipe"
    assert res["summary"]["successful_steps"] >= 1
    x = cap["x"]
    assert np.max(np.abs(x["points"] - pb.points)) > 0   # the step of iteration 1 was taken
    pb1 = pb.copy()
    pb1.cam_params, pb1.inst, pb1.points = x["cam_params"], x["inst"], x["points"]
    ob = oracle.OracleBA(pb1)
    cost = ob.linearize()
    cn, g = ob.colnorm_gradient()
    gscale = np.abs(g) + np.sqrt(cn * 2.0 * cost)
    assert np.max(np.abs(cap["grad"] - g) / gscale) <= 1e-12
    # the diagonal of iteration 2 uses the scale of iteration 1 (Ceres computes the Jacobi scale once)
    d = np.clip(cn * cap["scale"] ** 2, 1e-6, 1e32)
    assert np.max(np.abs(cap["diag"] - d) / d) <= 1e-12
    ob.set_scale(cap["scale"])
    S_o, rhs_o = ob.schur(cap["diag"] / cap["radius"])
    dd = np.sqrt(np.diag(S_o))
    assert np.max(np.abs(cap["S"] - S_o) / np.outer(dd, dd)) <= TAU
    assert np.max(np.abs(cap["rhs"] - rhs_o)) <= TAU * np.max(np.abs(rhs_o))


# Every scene runs on every variant.  The path each variant forces follows from the default path of the scene: the
# persistent kernel gives way to the CTA-per-segment tensor-core kernel, the tensor-core kernels to the SIMT segment
# kernels, the segment kernels to the per-point kernel; the PCG variants replace the solver.
def _variant_path(variant, name):
    schur = EXPECT[name].get("schur_kernel")
    if variant == "cta_per_segment_schur":
        return dict(schur_kernel="mma" if schur == "pipe" else schur)
    if variant == "simt_segment_schur":
        return dict(schur_kernel="simt_segment" if schur in ("pipe", "mma") else schur)
    if variant == "per_point_schur":
        return dict(schur_kernel="none", p_fast=0)
    if variant == "undeflated_pcg":
        return dict(schur_kernel=schur, pcg_kernel="pipelined")
    if variant == "classic_pcg":
        return dict(schur_kernel=schur, pcg_kernel="classic_resident")
    return dict(schur_kernel=schur, pcg_kernel="classic_streamed")


VARIANTS = {
    "cta_per_segment_schur": ("cta_per_segment_schur",),
    "simt_segment_schur": ("simt_segment_schur",),
    "per_point_schur": ("per_point_schur",),
    "undeflated_pcg": ("undeflated_pcg",),
    "classic_pcg": ("classic_pcg",),
    "streamed_pcg": ("classic_pcg", "streamed_pcg"),
}


@functools.lru_cache(maxsize=None)
def _default_chunks(name):
    pb = scenes.SCENES[name]()
    pb.max_iterations = 1
    return bundle.solve(pb, capture_iteration=1)["capture"]["sp_nchunks"]


@pytest.mark.parametrize("name", sorted(scenes.SCENES))
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_kernel_variant_matches_oracle(variant, name):
    m = measure(name, variant)
    _report(m)
    for k, v in _variant_path(variant, name).items():
        assert m[k] == v, (variant, name, k, m)
    if variant in ("cta_per_segment_schur", "simt_segment_schur"):
        # the Schur variants replace the Schur kernel only: the chunk list (so the linearisation) is the default's,
        # and the 1e-12 checks of check() cover the chunk-list column norms on the variant
        want = _default_chunks(name)
        assert (want > 0) == (m["wc"] == 9 and m["nres"] == 2 and m["nseg"] > 0), (name, want, m)
        assert m["sp_nchunks"] == want, (variant, name, want, m)
    check(m)


def test_pooled_handle_returns_to_the_product_path():
    """A fallback solve leaves nothing behind on the pooled handle: the next solve without fallbacks, on the same
    handle, takes the persistent Schur kernel, the deflated pipelined PCG and the device-driven LM loop."""
    from opensfm_b200 import _lib

    pb = scenes.SCENES["pipe_few_chunks"]()
    pb.max_iterations = 1
    with _lib.pooled("ba") as first:
        pass
    forced = bundle.solve(pb, capture_iteration=1, fallbacks=("classic_pcg", "host_loop", "per_point_schur"))
    assert forced["capture"]["schur_kernel"] == "none" and forced["capture"]["pcg_kernel"] == "classic_resident"
    assert forced["summary"]["device_loop"] == 0
    cap = bundle.solve(pb, capture_iteration=1)["capture"]
    assert cap["schur_kernel"] == "pipe" and cap["pcg_kernel"] == "pipelined_deflated", cap
    assert bundle.solve(pb)["summary"]["device_loop"] == 1
    with _lib.pooled("ba") as last:
        assert last is first   # every solve above ran on this one handle
