"""The engine's side terms (opensfm_b200/csrc/ba_side.cuh) row by row and assembled, against the oracle and against the
independent mpmath restatement of the reference's functors (tests/side_terms_mp.py).

* Rows: one problem of many independent terms (random configurations of all 17 types and every named edge case of
  test_side_terms_cpu.py), captured at LM iteration 1: the robustified rows side_linearize wrote against the oracle's
  (same formula in fp64; nvcc contracts to FMA) and against mpmath at the CPU test's bounds; the columns of constant
  blocks are exactly 0.
* Assembled system: one small scene per type, the ReconstructionAlignment scene and the duplicate-instance scene;
  column norms (through the Jacobi scale), gradient, S and rhs against the oracle at the linear-system test's TAU and
  against the dense system of the mpmath rows."""
import math

import numpy as np
import pytest

import test_side_terms_cpu as cpu
from opensfm_b200 import ba_problem as bp
from opensfm_b200 import bundle
from test_ba_linear_system_gpu import TAU

pytestmark = pytest.mark.gpu

# engine rows against the oracle's: the same fp64 formula; FMA contraction and libdevice's sin / cos / atan2 differ
# from glibc's in the last bits
ORACLE_ROW_TOL = 1e-12
N_RANDOM_GPU = 12


def capture(pb):
    pb.max_iterations = 1
    return bundle.solve(pb, capture_iteration=1, compute_reprojection_errors=False)


def rows_problem():
    B = cpu.random_builder(sorted(cpu.TYPE_NAMES), N_RANDOM_GPU, seed=31)
    cpu.edge_cases(B)
    return B


def test_side_rows_match_oracle_and_mpmath():
    B = rows_problem()
    pb = B.problem()
    res = capture(pb)
    cap = res["capture"]
    got = cpu.split_rows(pb, cap["side_r"], cap["side_J"])
    _, r_o, J_o = cpu.oracle.OracleBA(pb).side_rows(pb)
    want_o = cpu.split_rows(pb, r_o, J_o)
    want_mp = cpu.mp_rows(pb)
    worst_o, worst_mp, bad = 0.0, 0.0, {}
    for name, g, o, (r, J, ok) in zip(B.names, got, want_o, want_mp):
        assert ok, name
        eo = max(cpu.row_errors(g, o))
        ej, er = cpu.row_errors(g, (r, J))
        worst_o, worst_mp = max(worst_o, eo), max(worst_mp, ej)
        if eo > ORACLE_ROW_TOL or ej > cpu.j_tol(name) or er > cpu.R_TOL:
            bad[name] = (eo, ej, er)
    print("rows: worst vs oracle %.2e, vs mpmath %.2e" % (worst_o, worst_mp))
    assert not bad, bad
    # every column of a constant block is exactly 0 (local layout, before folding)
    nrow, nJ = pb.side_row_sizes()
    jo = np.concatenate([[0], np.cumsum(nJ)])
    n_const = 0
    for k, t in enumerate(pb.side_terms):
        sizes = [pb.block_size(*b) for b in t.blocks]
        Jl = cap["side_J"][jo[k]:jo[k + 1]].reshape(t.nres, sum(sizes))
        c = 0
        for b, n in zip(t.blocks, sizes):
            if cpu.block_constant(pb, *b):
                n_const += 1
                assert np.all(Jl[:, c:c + n] == 0.0), (B.names[k], b)
            c += n
    assert n_const > 0


def test_largest_term_every_column():
    """Linear motion over three instances with three distinct free rig cameras: 36 columns, close to SIDE_MAX_PARAMS."""
    B = cpu.Builder()
    rng = np.random.RandomState(8)
    B.add("lm36", bp.linear_motion_term([B.add_inst(cpu.pose(rng)) for _ in range(3)],
                                        [B.add_rc(cpu.pose(rng, 0.5, 0.5)) for _ in range(3)], 0.4, 0.5, 0.5))
    pb = B.problem()
    cap = capture(pb)["capture"]
    assert len(cap["side_J"]) == 6 * 36
    (g,) = cpu.split_rows(pb, cap["side_r"], cap["side_J"])
    ((r, J, ok),) = cpu.mp_rows(pb)
    den = np.max(np.abs(J), axis=0)
    assert np.all(den > 0)
    assert np.max(np.abs(g[1] - J) / den) <= cpu.J_TOL


def test_all_constant_term_adds_no_cost():
    """A term whose blocks are all constant is dropped from the minimised cost, as ceres drops it."""
    costs = []
    for with_constant in (False, True):
        rng = np.random.RandomState(9)
        B = cpu.Builder()
        B.add("free", bp.relative_rotation_term(B.add_inst(cpu.pose(rng)), B.add_inst(cpu.pose(rng)), None, None,
                                                cpu.rotvec(rng), np.eye(3), bp.LOSS_NONE, 1.0))
        if with_constant:
            B.add("constant", bp.relative_rotation_term(B.add_inst(cpu.pose(rng), True), B.add_inst(cpu.pose(rng), True),
                                                        None, None, cpu.rotvec(rng), np.eye(3), bp.LOSS_NONE, 1.0))
        costs.append(capture(B.problem())["summary"]["initial_cost"])
    assert costs[0] > 0 and costs[1] == costs[0], costs


def test_zero_scale_relative_motion_nan_cost():
    """RelativeMotionError fails on a zero scale: the cost is NaN on the engine as on the oracle (whose rows of the term
    are 0, test_side_terms_cpu.py); like ceres after a failed first evaluation, the solve stops before an iteration."""
    B = cpu.Builder()
    rng = np.random.RandomState(4)
    s0 = B.add_ext(0.0, True, [0.0])
    B.add("zero_scale", bp.relative_motion_term(B.add_inst(cpu.pose(rng)), B.add_inst(cpu.pose(rng)), s0, s0,
                                                np.r_[cpu.rotvec(rng), 1, 0, 0, 1], np.eye(7), True, bp.LOSS_SOFTLONE, 1.0))
    pb = B.problem()
    pb.max_iterations = 1
    res = bundle.solve(pb, compute_reprojection_errors=False)
    cost_o, _, _ = cpu.oracle.OracleBA(pb).side_rows(pb)
    assert math.isnan(res["summary"]["initial_cost"]) and math.isnan(cost_o), res["summary"]
    assert res["summary"]["successful_steps"] == 0


@pytest.mark.parametrize("name", cpu.SYSTEM_SCENES)
def test_assembled_system_matches_oracle_and_mpmath(name):
    pb = cpu.system_scene(name)
    cap = capture(pb)["capture"]
    nc = cap["nc"]
    scale, diag, radius = cap["scale"], cap["diag"], cap["radius"]
    cn = (1.0 / scale - 1.0) ** 2   # scale = 1 / (1 + |J_j|)
    ob, cost, cn_o, g_o, _, _, scale_o, diag_o = cpu.oracle_system(pb)
    ob.set_scale(scale)
    S_o, rhs_o = ob.schur(diag / radius)
    # against the oracle, as tests/test_ba_linear_system_gpu.py checks every kernel path; the cancelling columns of
    # duplicate_instance hold fp64 round-off on both sides (the mpmath comparison below bounds them)
    dup = name == "duplicate_instance"
    assert np.max(np.abs(scale - scale_o) / scale_o) <= 1e-12 and np.max(np.abs(diag - diag_o) / diag_o) <= 1e-12
    gscale = np.abs(g_o) + np.sqrt(cn_o * 2.0 * cost)
    gscale = np.maximum(gscale, 1e-12 * np.max(gscale))
    assert np.max(np.abs(cap["grad"] - g_o) / gscale) <= (cpu.DUPLICATE_SYSTEM_TOL if dup else 1e-12), name
    d = np.sqrt(np.diag(S_o))
    assert np.max(np.abs(cap["S"] - S_o) / np.outer(d, d)) <= (cpu.DUPLICATE_SYSTEM_TOL if dup else TAU), name
    assert np.max(np.abs(cap["rhs"] - rhs_o)) <= TAU * np.max(np.abs(rhs_o)), name
    # against the dense system of the mpmath rows
    want = cpu.dense_system(pb, cpu.mp_rows(pb), nc, scale, diag, radius)
    errs = cpu.system_errors(cn, cap["grad"], cap["S"], cap["rhs"], want, cost)
    print("%s: colnorm %.1e grad %.1e S %.1e rhs %.1e" % ((name,) + errs))
    # the column norm comes back through 1 / (1 + |J_j|): relative error up to 2 eps (1 + |J_j|) / |J_j| more
    tol = cpu.mp_system_tol(name)
    assert max(errs[1:]) <= tol, (name, errs)
    cscale = np.maximum(want[0], 1e-24 * np.max(want[0]))
    slack = 4e-16 * (1.0 + np.sqrt(want[0])) ** 2 / cscale
    assert np.all(np.abs(cn - want[0]) / cscale <= tol + slack), (name, errs)
