"""The shared-memory plan of the pipelined PCG (opensfm_b200/csrc/ba_pcg_plan.h, compiled for the host by g++) on the
structure of bench.py's C4 scene: it must fit an H100's shared memory with room to spare, so that the flagship
workload runs the gauge-deflated pipelined solver rather than the classic one."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from opensfm_b200 import ba_problem as bp
from opensfm_b200 import synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpu_harness", "ba_pcg_plan_host.cpp")
LIB = os.path.join(HERE, "cpu_harness", "_build", "libba_pcg_plan_host.so")
HDR = os.path.join(HERE, "..", "opensfm_b200", "csrc", "ba_pcg_plan.h")

H100_SMS = 132
H100_SMEM_OPTIN = 232448     # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
PIPELINED_STATIC_SMEM = 3840  # static shared memory of pcg_pipelined, ptxas -v of the sm_90a build
RESERVE = 1024                # what BA::plan_pcg keeps back on top
AVAILABLE = H100_SMEM_OPTIN - PIPELINED_STATIC_SMEM - RESERVE


@pytest.fixture(scope="module")
def hp():
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-o", LIB, SRC])
    return ctypes.CDLL(LIB)


def plan(hp, b1, b2, blk_sz, row_ptr, row_col, G, available=AVAILABLE):
    i32 = lambda x: np.ascontiguousarray(x, dtype=np.int32)
    b1, b2, blk_sz, row_ptr, row_col = map(i32, (b1, b2, blk_sz, row_ptr, row_col))
    grp_lo = np.zeros(G + 1, np.int32)
    shared = np.zeros(len(b1), np.int8)
    out = np.zeros(7, np.int64)
    P = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    hp.hp_plan(len(b1), P(b1), P(b2), len(blk_sz), P(blk_sz), P(row_ptr), P(row_col), G, ctypes.c_longlong(available),
               P(grp_lo), P(shared), P(out))
    keys = ("fits", "total", "ent", "cols", "minv", "rows", "groups")
    return dict(zip(keys, out.tolist()), grp_lo=grp_lo, shared=shared.astype(bool))


def reduced_structure(pb):
    """Parameter blocks, preconditioner groups and the CSR block structure of S, by the rules of BA::discover_structure
    (cameras first, then rig instances; a camera is grouped with the rig instance of its only shot)."""
    K, NI, S = len(pb.cam_type), len(pb.inst), len(pb.shot_inst)
    cam_blk, inst_blk, blk_sz = -np.ones(K, int), -np.ones(NI, int), []
    for k in range(K):
        if not pb.cam_const[k]:
            cam_blk[k] = len(blk_sz)
            blk_sz.append(bp.camera_num_params(int(pb.cam_type[k])))
    for i in range(NI):
        if not pb.inst_const[i]:
            inst_blk[i] = len(blk_sz)
            blk_sz.append(6)
    nblk = len(blk_sz)
    shot_cam, shot_inst = np.asarray(pb.shot_cam), np.asarray(pb.shot_inst)
    # shot -> its blocks, shot <-> shot through common points, block <-> block through their shots
    rows, cols = [], []
    for s in range(S):
        for b in (cam_blk[shot_cam[s]], inst_blk[shot_inst[s]]):
            if b >= 0:
                rows.append(s)
                cols.append(b)
    shot_blk = sp.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(S, nblk))
    obs = sp.csr_matrix((np.ones(len(pb.obs_shot)), (np.asarray(pb.obs_shot), np.asarray(pb.obs_point))),
                        shape=(S, len(pb.points)))
    covis = (obs @ obs.T) > 0
    blocks = (shot_blk.T @ covis @ shot_blk).tocsr()
    blocks.sort_indices()
    users = [set() for _ in range(K)]
    for s in range(S):
        users[shot_cam[s]].add(shot_inst[s])
    inst_cams = [set() for _ in range(NI)]
    for s in range(S):
        inst_cams[shot_inst[s]].add(shot_cam[s])
    b1, b2, done = [], [], set()
    for k in range(K):
        if cam_blk[k] < 0:
            continue
        i = next(iter(users[k])) if len(users[k]) == 1 else -1
        if i >= 0 and inst_blk[i] >= 0 and inst_cams[i] == {k} and blk_sz[cam_blk[k]] + 6 <= 16:
            b1.append(cam_blk[k]); b2.append(inst_blk[i]); done.add(i)
        else:
            b1.append(cam_blk[k]); b2.append(-1)
    for i in range(NI):
        if inst_blk[i] >= 0 and i not in done:
            b1.append(inst_blk[i]); b2.append(-1)
    return b1, b2, blk_sz, blocks.indptr, blocks.indices


@pytest.fixture(scope="module")
def c4_scene():
    return syn.cube_scene(500, 200000, 1.0, seed=42, max_obs_per_point=10)   # bench.py's C4


@pytest.fixture(scope="module")
def c4(c4_scene):
    return syn.scene_to_problem(c4_scene)


def test_c4_pipelined_plan_fits_h100(hp, c4):
    b1, b2, blk_sz, row_ptr, row_col = reduced_structure(c4)
    assert len(b1) == 500 and all(b >= 0 for b in b2)
    p = plan(hp, b1, b2, blk_sz, row_ptr, row_col, H100_SMS)
    print("C4 pipelined plan on %d CTAs: %d B of %d B available; worst CTA %d entries, %d columns, %d rows, %d groups" % (
        H100_SMS, p["total"], AVAILABLE, p["ent"], p["cols"], p["rows"], p["groups"]))
    assert p["shared"].all()   # camera k serves only shot k: both block rows of every group store the same columns
    assert p["fits"] and p["total"] + 8192 <= AVAILABLE
    lo = p["grp_lo"]
    assert lo[0] == 0 and lo[-1] == len(b1) and (np.diff(lo) >= 1).all()   # contiguous, every CTA owns a group


def test_cut_balances_entries(hp, c4):
    """S dominates the footprint, so the min-max cut leaves no CTA more than one group's entries above the mean."""
    b1, b2, blk_sz, row_ptr, row_col = reduced_structure(c4)
    p = plan(hp, b1, b2, blk_sz, row_ptr, row_col, H100_SMS)
    total_ent = sum(blk_sz[b] * sum(blk_sz[c] for c in row_col[row_ptr[b]:row_ptr[b + 1]]) for b in range(len(blk_sz)))
    widest_group = max(sum(blk_sz[b] * sum(blk_sz[c] for c in row_col[row_ptr[b]:row_ptr[b + 1]]) for b in (g1, g2))
                       for g1, g2 in zip(b1, b2))
    assert p["ent"] <= total_ent / H100_SMS + widest_group


def test_different_column_lists_keep_two_lists(hp):
    # two groups of a 3-wide and a 6-wide block row; in group 0 the rows store the same block columns, in group 1
    # block row 3 also couples to block 0 (a prior or side term can do that), so its lists differ
    blk_sz = [3, 6, 3, 6]
    rows = [[0, 1, 2], [0, 1, 2], [0, 1, 2, 3], [0, 2, 3]]
    row_ptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
    row_col = np.concatenate(rows)
    p = plan(hp, [0, 2], [1, 3], blk_sz, row_ptr, row_col, 1)
    assert p["shared"].tolist() == [True, False]
    assert p["cols"] == 12 + (18 + 12)   # group 0: one list of 12 columns; group 1: 18 and 12
    assert p["ent"] == 9 * 12 + 3 * 18 + 6 * 12
    assert p["minv"] == 2 * 81 and p["rows"] == 18 and p["groups"] == 2


def test_shared_intrinsics_variant(hp, c4_scene):
    """C4 with one camera for all 500 shots: its 3-row group stores every column of S."""
    b1, b2, blk_sz, row_ptr, row_col = reduced_structure(syn.scene_to_problem(c4_scene, shared_intrinsics=True))
    assert len(b1) == 501 and all(b < 0 for b in b2)
    p = plan(hp, b1, b2, blk_sz, row_ptr, row_col, H100_SMS)
    print("shared-intrinsics C4 pipelined plan: fits %d, %d B of %d B; worst CTA %d entries, %d columns, %d groups" % (
        p["fits"], p["total"], AVAILABLE, p["ent"], p["cols"], p["groups"]))
    assert p["fits"]
