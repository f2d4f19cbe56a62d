"""The LM loop driven by the device (one CUDA graph launch: a WHILE node around the iteration body, step control in
ba_lm_* kernels) against the same body driven by the host (the host_loop fallback path, which reads the LM state
after every decision).  Both must take the same steps: same iterations, successful steps, linear solves, PCG
iterations, termination and message; costs to 1e-9 relative and parameters to 1e-6 (the Schur atomics are unordered,
as in test_ba_pcg_path_gpu.py)."""
import numpy as np
import pytest

from opensfm_b200 import bundle, synthetic as syn

pytestmark = pytest.mark.gpu

KEYS = ("iterations", "successful_steps", "linear_solves", "pcg_iterations", "termination", "message", "initial_cost",
        "final_cost", "device_loop", "kernel_launches", "linearize_launches", "schur_launches")


def _both(pb):
    out = {}
    for name, fallbacks in (("device", ()), ("host", ("host_loop",))):
        r = bundle.solve(pb, fallbacks=fallbacks)
        out[name] = ({k: r["summary"][k] for k in KEYS}, {k: r[k] for k in ("cam_params", "inst", "points")})
    (sd, pd), (sh, ph) = out["device"], out["host"]
    print("device: %s\nhost:   %s" % (sd, sh))
    assert sd["device_loop"] == 1 and sh["device_loop"] == 0
    for k in ("iterations", "successful_steps", "linear_solves", "pcg_iterations", "termination", "message",
              "linearize_launches", "schur_launches"):
        assert sd[k] == sh[k], k
    for k in ("initial_cost", "final_cost"):
        assert abs(sd[k] - sh[k]) <= 1e-9 * abs(sh[k]), k
    for k in ("cam_params", "inst", "points"):
        a, b = np.asarray(pd[k], dtype=np.float64), np.asarray(ph[k], dtype=np.float64)
        assert np.abs(a - b).max(initial=0.0) <= 1e-6 * max(1.0, np.abs(b).max(initial=0.0)), k
    return sd, sh


def test_c4_device_loop_against_host_loop_fallback():
    pb = syn.scene_to_problem(syn.cube_scene(500, 200000, 1.0, seed=42, max_obs_per_point=10))
    sd, sh = _both(pb)
    # the graph's kernels are counted per execution: the same kernels as the host-driven loop, whose decisions
    # launch no kernels of their own
    assert sd["kernel_launches"] == sh["kernel_launches"]


def test_perturbed_ring_against_host_loop_fallback():
    pb = syn.scene_to_problem(syn.cube_scene(30, 4000, 1.0, seed=5), point_noise=0.05, position_noise=0.1,
                              rotation_noise=0.03)
    _both(pb)


def test_exact_start_against_host_loop_fallback():
    """Noise-free observations at the true parameters: the loop stops at its first step."""
    pb = syn.scene_to_problem(syn.cube_scene(12, 1500, 0.0, seed=3), perturb_seed=None)
    sd, _ = _both(pb)
    assert sd["iterations"] <= 1 and sd["termination"] == "CONVERGENCE"


def test_one_iteration_against_host_loop_fallback():
    pb = syn.scene_to_problem(syn.cube_scene(20, 3000, 1.0, seed=9), max_iterations=1)
    sd, _ = _both(pb)
    assert sd["iterations"] == 1 and sd["message"] == "Maximum number of iterations reached."


def test_constant_blocks_against_host_loop_fallback():
    pb = syn.scene_to_problem(syn.cube_scene(24, 3000, 1.0, seed=11), optimize_cameras=False)
    pb.inst_const[:3] = 1
    pb.point_const[::7] = 1
    _both(pb)
