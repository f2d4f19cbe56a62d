"""The bundle adjustment on inputs in the order the product gives them, not the (shot, point)-sorted, scene-numbered
order of the synthetic scenes.

* The device layout (tests/ba_layout_reference.py): nseg, p_fast and p_slow of every reduced-system scene.
* Observation order: a seeded shuffle of the observation list gives the same device layout, so the same solve within
  the run-to-run spread of the fp64 atomics (final cost 1e-12 relative, points 1e-9, identical iteration count), and
  the reprojection errors, un-permuted, to 1e-12.
* Relabelled problems: points, shots, cameras, rig instances and rig cameras renumbered (the side terms' block
  references with them) and the observations shuffled.  The local point order, the reduced system's block order and
  with them the summation order change: the bars of test_kernel_variants_agree (identical iteration count, cost 1e-9,
  points and cameras 1e-8; the gauge-free scenes after the similarity, as in test_ba_sharded_gpu.py).
* Reprojection errors, observation by observation, against the oracle's evaluation at the returned parameters.
  This needs no solver tolerance: it holds for any solve, one that stops early included.
* Sharded ranks (tests/ba_ranks.py) on the relabelled, shuffled problems.
* Through the product API: a map whose shots, landmarks and observations were inserted in shuffled order, with GCP
  points; `reconstruction.bundle`, `bundle_local`, `remove_outliers`, and the duplicate-observation rule of
  BundleAdjuster::Run (bundle_adjuster.cc:551: the later observation of a (point, shot) pair keeps its error).
* Parameter blocks no residual uses (`unobserved_and_idle`): the free points no shot observes and the rig instance
  of a shot without observations.  Ceres removes such blocks from the program it solves (the Solver::Summary
  documentation: a parameter block is inactive if no residual block refers to it, and num_parameter_blocks_reduced
  counts the blocks left after the inactive and constant ones are removed), so they come back as given.  The engine
  and the oracle keep them in the reduced system with empty columns: Jacobi scale 1, LM diagonal 1e-6, gradient 0,
  no entry in the gauge-deflation vectors of the pipelined PCG, so their step is exactly 0 and they come back bit for
  bit too.  The one place they count is |x| in the parameter-tolerance test (Ceres leaves them out); the tests pin
  that adding them changes nothing else beyond the run-to-run spread."""
import copy
import dataclasses
import functools

import numpy as np
import pytest

import ba_layout_reference as layout_ref
import ba_linear_system_scenes as scenes
import test_ba_sharded_gpu as sharded
from ba_ranks import run_ranks
from test_reconstruction_bundle import CONFIG   # the opensfm/config.py defaults
from oracle import ba_lm as oracle
from opensfm_b200 import ba_problem as bp
from opensfm_b200 import bundle
from opensfm_b200 import map_types as M
from opensfm_b200 import reconstruction as orec
from opensfm_b200 import synthetic as syn
from opensfm_b200 import types as T

pytestmark = pytest.mark.gpu

# one scene per Schur path: pipe (runs cut at 64; k = 10 / 11 at wc = 9), SIMT segments, spherical (mma), per-point
# with point priors, rig cameras (per-point, wc = 21), side terms, duplicate observations, idle blocks
ORDER_SCENES = ["pipe_long_runs", "pipe_k_edge", "brown_simt_segments", "spherical", "point_priors_many_obs",
                "rig_position_priors", "side_terms", "duplicate_observations", "unobserved_and_idle"]
ERROR_BAR = 1e-12   # per-observation reprojection error against the oracle (absolute)
SHUFFLE_COST, SHUFFLE_POINTS = 1e-12, 1e-9


@functools.lru_cache(maxsize=None)
def _scene(name):
    if name == "c2":
        return syn.scene_to_problem(syn.cube_scene(50, 5000, 1.0, with_descriptors=False))
    if name == "rig_position_priors":
        # rig_free_rigcam_priors with a position prior on every instance: the gauge is held, so the run-to-run spread
        # stays within the shuffle bars (without them, points moved 9e-8 between two runs of the same input on an H100)
        pb = scenes.rig_with_priors()
        rng = np.random.RandomState(14)
        pb.inst_has_prior[:] = 1
        pb.inst_prior_pos = pb.inst[:, 3:] + rng.normal(0, 0.02, (len(pb.inst), 3))
        pb.inst_prior_std = np.full((len(pb.inst), 3), 0.05)
        return pb
    return scenes.SCENES[name]()


@functools.lru_cache(maxsize=None)
def _solve(name):
    return bundle.solve(copy.deepcopy(_scene(name)))


def _at(pb, res):
    q = pb.copy()
    q.cam_params, q.inst, q.rigcam = res["cam_params"].copy(), res["inst"].copy(), res["rigcam"].copy()
    q.points, q.ext_values = res["points"].copy(), res["ext_values"].copy()
    return q


def _oracle_errors(pb, res):
    """The oracle's unscaled reprojection errors at the parameters `res` returned, in `pb`'s observation order."""
    return oracle.OracleBA(_at(pb, res)).cost(want_reproj=True)[1]


def _check_errors(label, pb, res):
    """res["reprojection_errors"] row by row against the oracle: 2 residuals for every model but SPHERICAL (3), the
    third column exactly 0 elsewhere.  Returns the worst difference."""
    got, want = res["reprojection_errors"], _oracle_errors(pb, res)
    assert got.shape == want.shape == (len(pb.obs_shot), 3)
    sph = np.asarray(pb.cam_type)[np.asarray(pb.shot_cam)[pb.obs_shot]] == bp.SPHERICAL
    assert np.all(got[~sph, 2] == 0.0), label
    worst = float(np.abs(got - want).max(initial=0.0))
    print("%s: worst per-observation error difference %.2e (%d observations)" % (label, worst, len(got)))
    assert worst <= ERROR_BAR, (label, worst)
    return worst


def _shuffled(pb, seed):
    """pb with its observation list permuted; perm[j] = the original index of observation j."""
    perm = np.random.RandomState(seed).permutation(len(pb.obs_shot))
    q = pb.copy()
    q.obs_shot, q.obs_point = pb.obs_shot[perm].astype(np.int32), pb.obs_point[perm].astype(np.int32)
    q.obs_xy, q.obs_sigma = pb.obs_xy[perm].copy(), pb.obs_sigma[perm].copy()
    return q, perm


def _relabelled(pb, seed):
    """pb with points, shots, cameras, rig instances and rig cameras renumbered by seeded permutations (new index of
    old block i = new[kind][i]) and the observation list shuffled.  Returns (problem, new, obs_perm)."""
    rng = np.random.RandomState(seed)
    K, NI, NR, S, P = len(pb.cam_type), len(pb.inst), len(pb.rigcam), len(pb.shot_inst), len(pb.points)
    new = {k: rng.permutation(n) for k, n in (("cam", K), ("inst", NI), ("rc", NR), ("shot", S), ("pt", P))}
    old = {k: np.argsort(v) for k, v in new.items()}   # old[kind][new index] = old index
    q = pb.copy()
    off = pb.cam_off
    seg = lambda a: np.concatenate([a[off[k]:off[k + 1]] for k in old["cam"]])
    q.cam_type, q.cam_const = pb.cam_type[old["cam"]], pb.cam_const[old["cam"]]
    q.cam_params, q.cam_prior = seg(pb.cam_params), seg(pb.cam_prior)
    q.cam_prior_sigma, q.cam_prior_log = seg(pb.cam_prior_sigma), seg(pb.cam_prior_log)
    for a in ("inst", "inst_const", "inst_has_prior", "inst_prior_pos", "inst_prior_std"):
        setattr(q, a, getattr(pb, a)[old["inst"]].copy())
    q.rigcam, q.rigcam_const = pb.rigcam[old["rc"]].copy(), pb.rigcam_const[old["rc"]].copy()
    if pb.rigcam_prior is not None:
        q.rigcam_prior, q.rigcam_prior_sigma = pb.rigcam_prior[old["rc"]].copy(), pb.rigcam_prior_sigma[old["rc"]].copy()
    s = old["shot"]
    q.shot_inst = new["inst"][pb.shot_inst[s]].astype(np.int32)
    q.shot_cam = new["cam"][pb.shot_cam[s]].astype(np.int32)
    q.shot_rc = new["rc"][pb.shot_rc[s]].astype(np.int32)
    q.shot_use_rc = pb.shot_use_rc[s].copy()
    q.points, q.point_const = pb.points[old["pt"]].copy(), pb.point_const[old["pt"]].copy()
    q.pp_point = new["pt"][pb.pp_point].astype(np.int32)
    kind_map = {bp.SB_CAM: new["cam"], bp.SB_INST: new["inst"], bp.SB_RIGCAM: new["rc"]}
    q.side_terms = [dataclasses.replace(t, blocks=[(k, int(kind_map[k][i]) if k in kind_map else i) for k, i in t.blocks])
                    for t in pb.side_terms]
    perm = rng.permutation(len(pb.obs_shot))
    q.obs_shot = new["shot"][pb.obs_shot[perm]].astype(np.int32)
    q.obs_point = new["pt"][pb.obs_point[perm]].astype(np.int32)
    q.obs_xy, q.obs_sigma = pb.obs_xy[perm].copy(), pb.obs_sigma[perm].copy()
    return q, new, perm


def _mapped_back(pb, res, new, perm):
    """The result of the relabelled problem in pb's numbering and observation order."""
    qoff = np.concatenate([[0], np.cumsum([bp.camera_num_params(pb.cam_type[k]) for k in np.argsort(new["cam"])])])
    cam = np.concatenate([res["cam_params"][qoff[new["cam"][k]]:qoff[new["cam"][k] + 1]] for k in range(len(pb.cam_type))])
    rep = np.empty_like(res["reprojection_errors"])
    rep[perm] = res["reprojection_errors"]
    return {"cam_params": cam, "inst": res["inst"][new["inst"]], "rigcam": res["rigcam"][new["rc"]],
            "points": res["points"][new["pt"]], "ext_values": res["ext_values"], "reprojection_errors": rep,
            "summary": res["summary"]}


# --------------------------------------------------------------------------------------------------------------------
# the device layout against the host reference
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(scenes.SCENES))
def test_layout_matches_the_host_reference(name):
    pb = copy.deepcopy(_scene(name))
    pb.max_iterations = 1
    cap = bundle.solve(pb, capture_iteration=1)["capture"]
    want = layout_ref.problem_layout(pb)
    assert cap["wc"] == layout_ref.camera_side_width(pb), (name, cap["wc"])
    got = (cap["nseg"], cap["p_fast"], cap["p_slow"])
    assert got == (want.nseg, want.p_fast, want.p_slow), (name, got, want.group_sizes)
    if name == "pipe_long_runs":
        assert want.group_sizes == [271, 65, 64] and cap["nseg"] == 5 + 2 + 1
    if name == "pipe_k_edge":   # k = 10 on the segments, k = 11 on the per-point kernel
        k = np.bincount(pb.obs_point)
        assert np.array_equal(want.eligible, k == 10) and set(k.tolist()) == {10, 11}
    if name == "duplicate_observations":
        assert len(set(zip(pb.obs_shot.tolist(), pb.obs_point.tolist()))) < len(pb.obs_shot)


def test_layout_of_the_per_point_fallback():
    pb = copy.deepcopy(_scene("pipe_long_runs"))
    pb.max_iterations = 1
    cap = bundle.solve(pb, capture_iteration=1, fallbacks=("per_point_schur",))["capture"]
    want = layout_ref.problem_layout(pb, per_point_fallback=True)
    assert (cap["nseg"], cap["p_fast"], cap["p_slow"]) == (want.nseg, want.p_fast, want.p_slow) == (0, 0, 400)


# --------------------------------------------------------------------------------------------------------------------
# observation order, relabelled problems, errors against the oracle
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ORDER_SCENES + ["c2"])
def test_reprojection_errors_match_the_oracle_observation_by_observation(name):
    _check_errors(name, _scene(name), _solve(name))


@pytest.mark.parametrize("name", ORDER_SCENES)
def test_shuffled_observations_give_the_same_solve(name):
    pb = _scene(name)
    one = _solve(name)
    q, perm = _shuffled(pb, 1)
    got = bundle.solve(q)
    s1, s = one["summary"], got["summary"]
    cost = abs(s["final_cost"] - s1["final_cost"]) / s1["final_cost"]
    pts = float(np.abs(got["points"] - one["points"]).max())
    rep = float(np.abs(got["reprojection_errors"] - one["reprojection_errors"][perm]).max())
    print("%s shuffled: %d iterations, final cost rel %.1e, points %.1e, reprojection errors %.1e"
          % (name, s["iterations"], cost, pts, rep))
    assert (s["iterations"], s["termination"]) == (s1["iterations"], s1["termination"]), (s, s1)
    assert cost <= SHUFFLE_COST and pts < SHUFFLE_POINTS, (cost, pts)
    assert rep <= 1e-12, rep
    _check_errors(name + " shuffled", q, got)


@pytest.mark.parametrize("name", ORDER_SCENES)
def test_relabelled_problem_gives_the_same_solve(name):
    pb = _scene(name)
    q, new, perm = _relabelled(pb, 2)
    got = bundle.solve(q)
    _check_errors(name + " relabelled", q, got)
    back = _mapped_back(pb, got, new, perm)
    sharded._check_against_single("%s relabelled" % name, pb, _solve(name), [back], 0.0, name)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("name", ORDER_SCENES)
def test_sharded_relabelled_problem(name, world):
    """The ranks return points and reprojection errors in the caller's order of the relabelled, shuffled problem:
    the single-GPU result of that problem under the bars of test_ba_sharded_gpu.py, and the oracle's errors at the
    returned parameters."""
    q, _, _ = _relabelled(_scene(name), 3)
    ranks = run_ranks(q, world)
    spread = sharded._check_ranks(q, world, ranks)
    one = bundle.solve(copy.deepcopy(q), fallbacks=sharded.HOST_LOOP)
    sharded._check_against_single("%s relabelled world=%d" % (name, world), q, one, ranks, spread, name)
    _check_errors("%s relabelled world=%d" % (name, world), q, ranks[0])


# --------------------------------------------------------------------------------------------------------------------
# parameter blocks no residual uses
# --------------------------------------------------------------------------------------------------------------------
def test_unobserved_blocks_come_back_as_given():
    pb = _scene("unobserved_and_idle")
    res = _solve("unobserved_and_idle")
    seen = np.zeros(len(pb.points), dtype=bool)
    seen[pb.obs_point] = True
    idle_inst = np.setdiff1d(np.arange(len(pb.inst)), pb.shot_inst[pb.obs_shot])
    assert (~seen).sum() == 20 and idle_inst.tolist() == [3]
    assert res["summary"]["iterations"] > 1 and np.abs(res["points"][seen] - pb.points[seen]).max() > 1e-4
    assert res["points"][~seen].tobytes() == np.ascontiguousarray(pb.points[~seen]).tobytes()
    assert res["inst"][idle_inst].tobytes() == np.ascontiguousarray(pb.inst[idle_inst]).tobytes()
    # the oracle does the same
    ref = oracle.solve(pb)
    assert ref["points"][~seen].tobytes() == np.ascontiguousarray(pb.points[~seen]).tobytes()
    assert ref["inst"][idle_inst].tobytes() == np.ascontiguousarray(pb.inst[idle_inst]).tobytes()


def test_unobserved_blocks_change_nothing_else():
    """The scene without its 20 unobserved points (and, separately, without the idle shot and its instance) solves
    to the same result as with them, within the run-to-run spread."""
    pb, full = _scene("unobserved_and_idle"), _solve("unobserved_and_idle")
    seen = np.zeros(len(pb.points), dtype=bool)
    seen[pb.obs_point] = True
    # without the unobserved points
    q = pb.copy()
    q.points, q.point_const = pb.points[seen].copy(), pb.point_const[seen].copy()
    q.obs_point = (np.cumsum(seen) - 1)[pb.obs_point].astype(np.int32)
    got = bundle.solve(q)
    # without the idle shot (4) and its instance (3)
    r = pb.copy()
    keep_inst, keep_shot = np.arange(len(pb.inst)) != 3, np.arange(len(pb.shot_inst)) != 4
    for a in ("inst", "inst_const", "inst_has_prior", "inst_prior_pos", "inst_prior_std"):
        setattr(r, a, getattr(pb, a)[keep_inst].copy())
    for a in ("shot_inst", "shot_cam", "shot_rc", "shot_use_rc"):
        setattr(r, a, getattr(pb, a)[keep_shot].copy())
    r.shot_inst = (r.shot_inst - (r.shot_inst > 3)).astype(np.int32)
    r.obs_shot = (pb.obs_shot - (pb.obs_shot > 4)).astype(np.int32)
    got_r = bundle.solve(r)
    s1 = full["summary"]
    for label, res, pts, inst in (("without the unobserved points", got, full["points"][seen], full["inst"]),
                                  ("without the idle shot", got_r, full["points"], full["inst"][keep_inst])):
        s = res["summary"]
        cost = abs(s["final_cost"] - s1["final_cost"]) / s1["final_cost"]
        dp, di = float(np.abs(res["points"] - pts).max()), float(np.abs(res["inst"] - inst).max())
        rep = float(np.abs(res["reprojection_errors"] - full["reprojection_errors"]).max())
        print("%s: %d iterations (%d with), final cost rel %.1e, points %.1e, instances %.1e, errors %.1e"
              % (label, s["iterations"], s1["iterations"], cost, dp, di, rep))
        assert (s["iterations"], s["termination"]) == (s1["iterations"], s1["termination"]), label
        assert cost <= SHUFFLE_COST and dp < SHUFFLE_POINTS and di < SHUFFLE_POINTS and rep < SHUFFLE_POINTS, label


# --------------------------------------------------------------------------------------------------------------------
# through the product API
# --------------------------------------------------------------------------------------------------------------------


class _Topocentric:   # lla are topocentric metres here
    def to_topocentric(self, lat, lon, alt):
        return np.array([lat, lon, alt])


@pytest.fixture()
def adjusters(monkeypatch):
    """Every BundleAdjuster that runs, in order (reconstruction.* build theirs internally)."""
    seen = []
    run = bundle.BundleAdjuster.run

    def recording_run(self):
        run(self)
        seen.append(self)

    monkeypatch.setattr(bundle.BundleAdjuster, "run", recording_run)
    return seen


def _shuffled_map(gcp_shots):
    """A cube scene (one shared perspective camera) whose shots, landmarks and observations enter the map in shuffled
    order, 4 % of the observations moved by 0.02 (gross outliers), and three GCPs with lla seen from `gcp_shots`."""
    sc = syn.cube_scene(10, 400, 1.0, with_descriptors=False, max_obs_per_point=5)
    pb = syn.scene_to_problem(sc, shared_intrinsics=True)
    rng = np.random.RandomState(31)
    r = M.Reconstruction()
    r.reference = _Topocentric()
    cam = T.Camera.create_perspective(float(sc.cam_params[0][2]), float(sc.cam_params[0][0]), float(sc.cam_params[0][1]))
    cam.id = "1"
    r.add_camera(cam)
    for s in rng.permutation(len(pb.inst)):
        r.create_shot("shot%d" % s, "1", T.Pose.from_ba_params(pb.inst[s]))
    for p in rng.permutation(len(pb.points)):
        r.create_point("pt%d" % p, pb.points[p])
    xy = pb.obs_xy.copy()
    bad = rng.uniform(size=len(xy)) < 0.04
    xy[bad] += rng.choice([-0.02, 0.02], (int(bad.sum()), 2))
    for k in rng.permutation(len(pb.obs_shot)):
        r.add_observation("shot%d" % pb.obs_shot[k], "pt%d" % pb.obs_point[k],
                          M.Observation(xy[k, 0], xy[k, 1], pb.obs_sigma[k], feature=int(k)))
    gcps = []
    for g, x in enumerate([np.array([0.1, 0.2, -0.1]), np.array([-0.3, 0.1, 0.2]), np.array([0.2, -0.3, 0.3])]):
        pt = M.GroundControlPoint()
        pt.id = "g%d" % g
        pt.lla = {"latitude": x[0], "longitude": x[1], "altitude": x[2]}
        pt.has_altitude = bool(g % 2)
        for sid in gcp_shots:
            s = int(sid[4:])
            px = syn.project_perspective((sc.R_wc[s] @ (x - sc.origins[s]))[None, :], *sc.cam_params[s])[0]
            pt.add_observation(M.GroundControlPointObservation(sid, px))
        gcps.append(pt)
    return r, gcps


def _check_map_errors(label, r, ba, point_ids):
    """Every landmark.reprojection_errors[shot] is the oracle's error of that (shot, point) at the returned parameters;
    every observation of the problem has its entry.  Returns the oracle's errors by (point id, shot id)."""
    pb, res = ba.results()
    _check_errors(label, pb, res)
    want = _oracle_errors(pb, res)
    shot_ids = ba._order[3]
    by_pair = {}
    for k, (s, p) in enumerate(zip(pb.obs_shot.tolist(), pb.obs_point.tolist())):
        by_pair[(ba._pt_ids[p], shot_ids[s])] = want[k, :2]
    n = 0
    for pid in point_ids:
        errs = r.points[pid].reprojection_errors
        assert set(errs) == {s for (q, s) in by_pair if q == pid}, (label, pid)
        for sid, e in errs.items():
            assert e.shape == (2,) and np.abs(e - by_pair[(pid, sid)]).max() <= ERROR_BAR, (label, pid, sid)
            n += 1
    assert n > 0
    return by_pair


def _observation_order(ba):
    """(shot id, point id) of the solved problem's observations, in its order."""
    pb, _ = ba.results()
    shot_ids = ba._order[3]
    return [(shot_ids[s], ba._pt_ids[p]) for s, p in zip(pb.obs_shot.tolist(), pb.obs_point.tolist())]


def test_bundle_of_a_shuffled_map(adjusters):
    """reconstruction.bundle on the shuffled map: its observations in the map's order (shot by shot in insertion order,
    a shot's landmarks in its order, GCP points last, point by point), errors on the map equal to the oracle's, and
    remove_outliers removes exactly the observations whose oracle error exceeds the threshold."""
    r, gcps = _shuffled_map(["shot1", "shot4", "shot7"])
    cfg = dict(CONFIG, bundle_use_gps=False, align_method="naive")
    orec.bundle(r, dict(r.cameras.items()), dict(r.rig_cameras.items()), gcps, cfg)
    (ba,) = adjusters
    want_order = [(sid, lm.id) for sid, shot in r.shots.items() for lm in shot.get_valid_landmarks()]
    want_order += [(o.shot_id, "gcp-" + g.id) for g in gcps for o in g.observations]
    assert _observation_order(ba) == want_order
    by_pair = _check_map_errors("bundle", r, ba, list(r.points))

    before = {(pid, s.id) for pid, lm in r.points.items() for s in lm.get_observations()}
    thr = CONFIG["bundle_outlier_fixed_threshold"]
    norm = {k: float(np.hypot(*e)) for k, e in by_pair.items() if k in before}
    assert min(abs(v - thr) for v in norm.values()) > 1e-9   # no decision within round-off of the threshold
    outliers = {k for k, v in norm.items() if v > thr}
    assert 20 < len(outliers) < len(before) // 10
    expected = set(outliers)
    for pid in {p for p, _ in outliers}:   # landmarks left with fewer than 2 observations go with theirs
        rest = {k for k in before if k[0] == pid} - outliers
        if len(rest) < 2:
            expected |= rest
    assert orec.remove_outliers(r, cfg) == len(outliers)
    after = {(pid, s.id) for pid, lm in r.points.items() for s in lm.get_observations()}
    assert before - after == expected and after <= before


def test_bundle_local_of_a_shuffled_map(adjusters):
    """reconstruction.bundle_local: the interior shots' observations, then the boundary shots' ones (of interior
    points), then the GCP points'; errors on the map equal to the oracle's for every point of the local problem."""
    r, _ = _shuffled_map([])
    cfg = dict(CONFIG, bundle_use_gps=False, local_bundle_radius=2, local_bundle_min_common_points=5,
               local_bundle_max_shots=5)
    central = "shot0"
    interior, boundary = orec.shot_neighborhood_ids(r, central, 2, 5, 5)
    assert interior and boundary
    gcp_shots = sorted(interior)[:3]
    _, gcps = _shuffled_map(gcp_shots)
    pt_ids, _ = orec.bundle_local(r, dict(r.cameras.items()), dict(r.rig_cameras.items()), gcps, central, cfg)
    (ba,) = adjusters
    order = _observation_order(ba)
    rank = [2 if p.startswith("gcp-") else 0 if s in interior else 1 for s, p in order]
    assert rank == sorted(rank) and set(rank) == {0, 1, 2}, "interior, then boundary, then GCP observations"
    shots_seen = [s for s, p in order if not p.startswith("gcp-")]
    assert shots_seen == sorted(shots_seen, key=shots_seen.index), "shot by shot"
    _check_map_errors("bundle_local", r, ba, pt_ids)


def test_duplicate_observation_keeps_the_later_error():
    """A (point, shot) pair observed twice: both residuals enter the solve, and Point::reprojection_errors[shot]
    holds the error of the one that comes later in the caller's order (the map is overwritten,
    bundle_adjuster.cc:551)."""
    pb0 = _scene("duplicate_observations")
    ba = bundle.BundleAdjuster()
    off = pb0.cam_off
    for k in range(len(pb0.cam_type)):
        vals = pb0.cam_params[off[k]:off[k + 1]]
        ba.add_camera("c%d" % k, T.Camera("perspective", vals), T.Camera("perspective", vals), False)
    ba.add_rig_camera("rc", T.Pose(), T.Pose(), True)
    for i in range(len(pb0.inst)):
        ba.add_rig_instance("i%d" % i, T.Pose.from_ba_params(pb0.inst[i]), {"s%d" % i: "c%d" % i}, {"s%d" % i: "rc"}, False)
    ba.add_points_bulk(["p%d" % p for p in range(len(pb0.points))], pb0.points, False)
    q, _ = _shuffled(pb0, 4)
    ba.add_observations_bulk(["s%d" % s for s in q.obs_shot], ["p%d" % p for p in q.obs_point], q.obs_xy, q.obs_sigma)
    ba.set_point_projection_loss_function("SoftLOneLoss", 1.0)
    ba.run()
    pb, res = ba.results()
    want = _oracle_errors(pb, res)
    _check_errors("duplicates through BundleAdjuster", pb, res)
    last, first = {}, {}
    for k, (s, p) in enumerate(zip(pb.obs_shot.tolist(), pb.obs_point.tolist())):
        last[(p, s)] = want[k, :2]
        first.setdefault((p, s), want[k, :2])
    differ = [k for k in last if np.abs(last[k] - first[k]).max() > 1e-5]
    assert len(differ) >= 20
    for (p, s), e in last.items():
        got = ba.get_point("p%d" % p).reprojection_errors["s%d" % s]
        assert np.abs(got - e).max() <= ERROR_BAR, (p, s, got, e, first[(p, s)])
