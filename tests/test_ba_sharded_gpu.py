"""The sharded bundle adjustment (world > 1) on one GPU: `world` ranks as threads of one process behind the checking
all-reduce of tests/ba_ranks.py, on every reduced-system scene of tests/ba_linear_system_scenes.py.

What only the sharded path runs: points sharded by p % world == rank, the rank sums of column norms, gradient, cost
and per-rank gradient maxima, prior rows and side terms added by rank 0 only, the camera side of the step counted by
rank 0 only, point priors evaluated by the owning rank, structure discovery over the global observation list, the
gathers of points and reprojection errors, and the host-driven LM loop with the projected line search.

* max_iterations = 0: the gathers are exact (points bitwise the input, reprojection errors bitwise the world = 1 ones)
  and the initial cost matches world = 1 and the oracle (a prior row or side term added on every rank, or on none,
  changes it: `camera_and_position_priors` and `side_terms` start with non-zero prior and side residuals).
* The full solve matches world = 1 with the same loop driver (host_loop); the ranks agree with each other.
* Shards with no free point (all its points constant, or no point at all) take part in every all-reduce.
* Each fallback kernel path at world = 2 against world = 1 on the same path."""
import copy
import functools

import numpy as np
import pytest

import ba_linear_system_scenes as scenes
from ba_ranks import run_ranks
from oracle import ba_lm as oracle
from opensfm_b200 import _lib, bundle, synthetic as syn

pytestmark = pytest.mark.gpu

NAMES = list(scenes.SCENES)
WORLDS = [2, 3]
HOST_LOOP = ("host_loop",)   # the sharded solve always runs the host-driven LM loop
# the summary fields that describe the solve (the others are per-rank timings, kernel counts and the local size)
SOLVE_FIELDS = ("iterations", "successful_steps", "linear_solves", "pcg_iterations", "termination", "initial_cost",
                "final_cost", "message", "reduced_dim", "reduced_blocks", "reduced_nnz", "jac_planes", "device_loop")
CAMERA_SIDE = ("cam_params", "inst", "rigcam", "ext_values")
# a different summation order of the reduced system (test_kernel_variants_agree)
TOL_PARAM = 1e-8
# Scenes whose similarity gauge (rotation, translation, scale of the whole reconstruction) is free: no position prior
# holds it, and the sharded and the single-GPU iterates drift apart along it while the cost, the cameras and the
# reprojection errors agree.  Largest differences of three runs on an H100 (world 2 and 3), raw and after the
# least-squares similarity:
#   rig_free_rigcam_priors  instances 1.1e-6, points 2.5e-7; aligned instances 2.6e-10, points 4.5e-11;
#                           rig cameras 4.0e-8 (their translation scales with the reconstruction)
#   rig_segments            instances 2.6e-6, points 5.6e-6; aligned instances 1.8e-7, points 6.4e-8 -- over the
#                           points seen from two or more rig instances: 11 of its 300 points are seen from one or none,
#                           held along their ray by the LM damping only (aligned, those moved by 3.0e-6)
#   cauchy_outliers         instances 1.5e-5, points 9.6e-6; aligned instances 5.1e-11, points 9.9e-10
# There the points and instances are compared after the similarity (rig_segments to 1e-6), the rig cameras to 1e-6.
GAUGE_FREE = {"rig_free_rigcam_priors", "rig_segments", "cauchy_outliers"}
# rig_segments (thinned to 35 % of its observations): final costs up to 4.1e-9 apart, reprojection errors 4.3e-9
TOL_COST = {"rig_segments": 2e-8}
TOL_REPROJECTION = {"rig_segments": 5e-8}


@functools.lru_cache(maxsize=None)
def _scene(name):
    return scenes.SCENES[name]()


def _problem(name, **changes):
    pb = copy.deepcopy(_scene(name))
    for k, v in changes.items():
        setattr(pb, k, v)
    return pb


@functools.lru_cache(maxsize=None)
def _single(name, max_iterations=None, fallbacks=HOST_LOOP):
    pb = _problem(name) if max_iterations is None else _problem(name, max_iterations=max_iterations)
    return bundle.solve(pb, fallbacks=fallbacks)


def _check_ranks(pb, world, ranks):
    """Every rank returns the same solve: identical points, reprojection errors and summary (but for the local
    observation count, which is that of its shard), camera side to 1e-12 (each rank solves its own copy of the
    all-reduced system, and the side-term blocks are added with atomics after the exchange).  Returns that spread."""
    r0 = ranks[0]
    owner = np.asarray(pb.obs_point) % world
    for r, res in enumerate(ranks):
        s = res["summary"]
        assert s["device_loop"] == 0
        assert s["num_observations_local"] == int((owner == r).sum()), (r, s["num_observations_local"])
        assert {k: s[k] for k in SOLVE_FIELDS} == {k: r0["summary"][k] for k in SOLVE_FIELDS}, r
        assert res["points"].tobytes() == r0["points"].tobytes(), r
        assert res["reprojection_errors"].tobytes() == r0["reprojection_errors"].tobytes(), r
    spread = max([np.abs(res[k] - r0[k]).max(initial=0.0) for res in ranks[1:] for k in CAMERA_SIDE] + [0.0])
    assert spread <= 1e-12, spread
    return spread


def _similarity_aligned(one, got):
    """`got`'s points and rig instances moved by the similarity that maps its points and instance centres closest onto
    `one`'s (least squares, Umeyama): what is left differs outside the similarity gauge."""
    from scipy.spatial.transform import Rotation

    P = len(got["points"])
    A = np.vstack([got["points"], got["inst"][:, 3:]])
    B = np.vstack([one["points"], one["inst"][:, 3:]])
    A0, B0 = A - A.mean(0), B - B.mean(0)
    U, S, Vt = np.linalg.svd(B0.T @ A0)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    R = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / (A0 ** 2).sum()
    moved = s * A0 @ R.T + B.mean(0)
    # rotation angle between the moved and `one`'s camera-to-world rotations
    rot = Rotation.from_matrix(R) * Rotation.from_rotvec(got["inst"][:, :3])
    angle = (rot.inv() * Rotation.from_rotvec(one["inst"][:, :3])).magnitude()
    return moved[:P], moved[P:], angle


def _differences(pb, one, got):
    s1, s = one["summary"], got["summary"]
    d = {"cost": abs(s["final_cost"] - s1["final_cost"]) / s1["final_cost"]}
    for k in CAMERA_SIDE + ("points", "reprojection_errors"):
        d[k] = float(np.abs(got[k] - one[k]).max(initial=0.0))
    pts, centres, angle = _similarity_aligned(one, got)
    # points seen from two or more rig instances
    seen = np.zeros((len(pb.points), len(pb.inst)), dtype=bool)
    seen[np.asarray(pb.obs_point), np.asarray(pb.shot_inst)[np.asarray(pb.obs_shot)]] = True
    fixed = seen.sum(1) >= 2
    d["points_aligned"] = float(np.abs(pts[fixed] - one["points"][fixed]).max(initial=0.0))
    d["inst_aligned"] = float(max(np.abs(centres - one["inst"][:, 3:]).max(initial=0.0), angle.max(initial=0.0)))
    return d


def _check_against_single(label, pb, one, ranks, spread, name=None):
    s1, s = one["summary"], ranks[0]["summary"]
    d = _differences(pb, one, ranks[0])
    print("%s: %d iterations (%s), final cost rel %.1e, cameras %.1e, instances %.1e, rig cameras %.1e, ext %.1e, "
          "points %.1e, reprojection errors %.1e; after the similarity: instances %.1e, points %.1e; ranks' camera side "
          "%.1e" % (label, s["iterations"], s["termination"], d["cost"], d["cam_params"], d["inst"], d["rigcam"],
                    d["ext_values"], d["points"], d["reprojection_errors"], d["inst_aligned"], d["points_aligned"], spread))
    assert (s["iterations"], s["termination"]) == (s1["iterations"], s1["termination"]), (s, s1)
    assert d["cost"] <= TOL_COST.get(name, 1e-9), d
    assert d["reprojection_errors"] < TOL_REPROJECTION.get(name, TOL_PARAM), d
    if name in GAUGE_FREE:
        compared = {"cam_params": TOL_PARAM, "ext_values": TOL_PARAM, "rigcam": 1e-6, "inst_aligned": TOL_PARAM,
                    "points_aligned": TOL_PARAM}
        if name == "rig_segments":
            compared.update(inst_aligned=1e-6, points_aligned=1e-6)
    else:
        compared = {k: TOL_PARAM for k in CAMERA_SIDE + ("points",)}
    for k, tol in compared.items():
        assert d[k] < tol, (k, d)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", NAMES)
def test_sharded_start_is_exact(name, world):
    """No LM step: the gathers return the input points and the world = 1 reprojection errors bit for bit (one rank
    writes each value, the others add zeros); the initial cost is the world = 1 and the oracle's one."""
    pb = _problem(name, max_iterations=0)
    one = _single(name, 0)
    ranks = run_ranks(pb, world)
    _check_ranks(pb, world, ranks)
    c1 = one["summary"]["initial_cost"]
    ref = oracle.OracleBA(pb).cost()
    points = np.ascontiguousarray(pb.points, dtype=np.float64).tobytes()
    for res in ranks:
        assert res["points"].tobytes() == points
        assert res["reprojection_errors"].tobytes() == one["reprojection_errors"].tobytes()
        c = res["summary"]["initial_cost"]
        assert abs(c - c1) <= 1e-12 * c1, (c, c1)
        assert abs(c - ref) <= 1e-9 * ref, (c, ref)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", NAMES)
def test_sharded_solve_matches_single_gpu(name, world):
    pb = _problem(name)
    ranks = run_ranks(pb, world)
    spread = _check_ranks(pb, world, ranks)
    _check_against_single("%s world=%d" % (name, world), pb, _single(name), ranks, spread, name)


def _point_only(num_cameras, num_points, shared_intrinsics=False, optimize_cameras=False):
    """Cube scene with constant instances (and constant cameras unless `optimize_cameras`)."""
    sc = syn.cube_scene(num_cameras, num_points, 1.0, with_descriptors=False)
    pb = syn.scene_to_problem(sc, shared_intrinsics=shared_intrinsics, optimize_cameras=optimize_cameras)
    pb.inst_const[:] = 1
    return pb


def _no_free_points_case(case):
    if case == "constant_shard":    # world 2: every point of rank 1 constant, only points free (nc = 0)
        pb = _point_only(8, 400)
        pb.point_const[1::2] = 1
        return pb, 2, 0
    if case == "empty_shard":       # world 3, two points: rank 2 holds no point and no observation (nc = 0)
        return _point_only(6, 2), 3, 0
    if case == "empty_shard_free_cameras":   # the same with the (shared) intrinsics free: nc = 3
        return _point_only(6, 2, shared_intrinsics=True, optimize_cameras=True), 3, 3
    raise ValueError(case)


@pytest.mark.parametrize("case", ["constant_shard", "empty_shard", "empty_shard_free_cameras"])
def test_shard_without_free_points(case):
    """A rank whose shard has no free point still takes every all-reduce of the others and leaves the LM loop with them
    (the "no free parameters" decision is the whole problem's, not the shard's)."""
    pb, world, nc = _no_free_points_case(case)
    assert len(pb.points) >= 2
    one = bundle.solve(copy.deepcopy(pb), fallbacks=HOST_LOOP)
    assert one["summary"]["reduced_dim"] == nc
    assert one["summary"]["iterations"] > 0, one["summary"]
    ranks = run_ranks(pb, world)
    spread = _check_ranks(pb, world, ranks)
    _check_against_single("%s world=%d" % (case, world), pb, one, ranks, spread)


KERNEL_PATHS = {"per_point_schur": ("per_point_schur",), "simt_segment_schur": ("simt_segment_schur",),
                "cta_per_segment_schur": ("cta_per_segment_schur",), "generic_linearize": ("generic_linearize",),
                "classic_pcg": ("classic_pcg",), "streamed_pcg": ("classic_pcg", "streamed_pcg"),
                "undeflated_pcg": ("undeflated_pcg",)}


@pytest.mark.parametrize("path", list(KERNEL_PATHS))
def test_sharded_kernel_path(path):
    """Each fallback kernel path at world = 2 against world = 1 on the same path."""
    fb = KERNEL_PATHS[path]
    pb = _problem("pipe_many_chunks")
    ranks = run_ranks(pb, 2, fallbacks=fb)
    spread = _check_ranks(pb, 2, ranks)
    _check_against_single("pipe_many_chunks world=2 %s" % path, pb, _single("pipe_many_chunks", None, fb + HOST_LOOP),
                          ranks, spread)


def test_sharded_pinned_inputs():
    """pinned_inputs=True (observations uploaded on a copy stream while run() sorts) gives the default result."""
    pb = _problem("pipe_few_chunks")
    ref = run_ranks(pb, 2)
    got = run_ranks(pb, 2, pinned_inputs=True)
    _check_ranks(pb, 2, got)
    assert got[0]["summary"]["iterations"] == ref[0]["summary"]["iterations"]
    c = ref[0]["summary"]["final_cost"]
    assert abs(got[0]["summary"]["final_cost"] - c) <= 1e-12 * c
    assert np.abs(got[0]["points"] - ref[0]["points"]).max() < 1e-9


def test_distributed_capture_raises_before_any_allreduce():
    calls = []
    with pytest.raises(ValueError, match="world == 1"):
        bundle.solve(_problem("pipe_few_chunks"), rank=0, world=2, allreduce=lambda ptr, count, strm: calls.append(count),
                     capture_iteration=1)
    assert calls == []


def test_single_gpu_solve_after_sharded_solve():
    """The pooled handles of a sharded solve, reused at world = 1, run the device-driven loop again and give the usual
    solve."""
    pb = _problem("pipe_few_chunks")
    ref = bundle.solve(copy.deepcopy(pb))
    assert ref["summary"]["device_loop"] == 1
    world = 3
    run_ranks(pb, world)
    held = [_lib.acquire("ba", 0) for _ in range(world)]   # the ranks' handles: the pool hands out the last released first
    try:
        for i, h in enumerate(held):
            _lib.release(h)
            got = bundle.solve(copy.deepcopy(pb))   # on h
            held[i] = _lib.acquire("ba", 0)
            assert held[i] is h
            s = got["summary"]
            assert s["device_loop"] == 1 and s["iterations"] == ref["summary"]["iterations"], s
            assert abs(s["final_cost"] - ref["summary"]["final_cost"]) <= 1e-12 * ref["summary"]["final_cost"]
            assert np.abs(got["points"] - ref["points"]).max() < 1e-9
    finally:
        for h in held:
            _lib.release(h)
