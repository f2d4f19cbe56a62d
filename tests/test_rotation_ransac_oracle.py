"""oracle/rotation_ransac_oracle.py on the CPU: its sample stream against the host's libstdc++ (g++-compiled harness
tests/cpu_harness/uniform_int_host.cpp) and numpy's mt19937, OpenSfM's known-answer test for the rotation-only
RANSAC, and hand-built pairs for the scoring, tie and 3-point rules."""
import os
import subprocess

import numpy as np
import pytest

import image_pair_cases as C
from oracle import rotation_ransac_oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpu_harness", "uniform_int_host.cpp")
EXE = os.path.join(HERE, "cpu_harness", "_build", "uniform_int_host")


@pytest.fixture(scope="module")
def harness():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < os.path.getmtime(SRC):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-o", EXE, SRC])
    return EXE


def test_generator_pin(harness):
    """The 10000th output of a default-seeded mt19937 is 4123659995 (C++ standard, [rand.predef])."""
    assert int(o.Mt19937().outputs(10000)[-1]) == 4123659995
    assert int(subprocess.check_output([harness, "pin"]).decode().strip()) == 4123659995


def test_stream_is_numpy_mt19937():
    raw = np.random.RandomState(42).randint(0, 2 ** 32, size=5000, dtype=np.uint32)
    assert np.array_equal(o.SampleStream.prefix(5000)[:5000], raw)


CASES = [(3, 3, 40), (4, 3, 40), (5, 3, 40), (7, 3, 30), (12, 12, 10), (13, 12, 10), (24, 12, 10), (50, 3, 60),
         (100, 12, 20), (737, 3, 50), (1000, 12, 20), (3000, 3, 40), (65537, 3, 20), (1 << 20, 12, 5),
         ((1 << 31) - 1, 3, 30), ((1 << 31) - 1, 12, 10), ((1 << 31) + 12345, 3, 10), ((1 << 32) - 5, 3, 10)]


def test_samples_match_libstdcxx(harness):
    """uniform_int_distribution<mt19937::result_type> with redraw of repeats, for small n (where every index repeats
    often), n = 2^31 - 1 and ranges near 2^32 (where Lemire's rejection is frequent)."""
    lines = "".join("%d %d %d\n" % c for c in CASES)
    out = subprocess.run([harness], input=lines, capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(out) == len(CASES)
    for (n, size, count), line in zip(CASES, out):
        want = [int(x) for x in line.split()]
        s = o.SampleStream()
        got = [v for _ in range(count) for v in o.sample(s, size, n)]
        assert got == want, (n, size)


def test_known_answer_relative_rotation():
    """test_robust.py's test_outliers_relative_rotation_ransac: 30 % outliers, the inlier count within 4 % of 70 %
    and the model within 8e-2 of the true rotation (Frobenius)."""
    for seed in range(20):
        b1, b2, rotation, threshold = C.robust_case(seed)
        r = o.ransac_rotation(b1, b2, threshold)
        assert np.isclose(r.ransac_inliers, 0.7 * len(b1), rtol=0.04), seed
        assert np.linalg.norm(rotation - r.lo_model, ord="fro") < 8e-2, seed


def test_pure_rotation_scores_zero():
    rng = np.random.RandomState(3)
    b1 = C.unit(np.column_stack([rng.uniform(-0.5, 0.5, (300, 2)), np.ones(300)]))
    R = C.rotation_about([0.3, -1.0, 0.2], 0.4)
    b2 = b1 @ R     # b2 = R^T b1: R b2 = b1
    r = o.ransac_rotation(b1, b2, 0.016)
    assert r.chord_inliers == 300 and r.score == 0
    assert np.abs(r.R - R).max() < 1e-12


@pytest.mark.parametrize("outliers", [90, 91, 150])
def test_known_outlier_count(outliers):
    """Rows off the rotation by more than the threshold are exactly the outliers, and the score is their count
    (0 below 30 %)."""
    n = 300
    rng = np.random.RandomState(outliers)
    b1 = C.unit(np.column_stack([rng.uniform(-0.5, 0.5, (n, 2)), np.ones(n)]))
    R = C.rotation_about([1.0, 0.2, 0.1], 0.3)
    b2 = b1 @ R
    bad = rng.permutation(n)[:outliers]
    b2[bad] = (C.unit(b1[bad] + rng.uniform(0.1, 0.3, (outliers, 3)) * np.where(rng.rand(outliers, 3) < 0.5, -1, 1))
               @ R)
    r = o.ransac_rotation(b1, b2, 0.016)
    assert r.chord_inliers == n - outliers
    assert set(np.nonzero(~r.chord_mask)[0].tolist()) == set(bad.tolist())
    assert r.score == (outliers if outliers >= 0.3 * n else 0)


def test_tie_replaces_best_and_runs_local_optimisation():
    """Two groups of rows, each exact under its own rotation, of equal size: a model of the second group ties the
    best one, replaces it and starts local optimisation, so the result is the rotation of the group hit last."""
    k = 40
    rng = np.random.RandomState(11)
    b1 = C.unit(np.column_stack([rng.uniform(-0.5, 0.5, (2 * k, 2)), np.ones(2 * k)]))
    RA, RB = C.rotation_about([0, 0, 1], 0.2), C.rotation_about([1, 0, 0], 1.2)
    group = np.arange(2 * k) % 2          # interleaved, so the samples mix the groups
    b2 = np.where(group[:, None] == 0, b1 @ RA, b1 @ RB)
    r = o.ransac_rotation(b1, b2, 0.016)
    ties = [i for i, (inl, best, replaced, lo) in enumerate(r.events) if inl == best and inl == k]
    assert ties, r.events
    for i in ties:
        assert r.events[i][2] and r.events[i][3]      # replaced, local optimisation ran
    # the group of the last model with k inliers is the result's
    last = max(i for i, e in enumerate(r.events) if e[0] == k)
    draws = np.array(r.draws)
    pos = 0
    groups = []
    for i, (inl, best, replaced, lo) in enumerate(r.events):
        groups.append(set(group[draws[pos:pos + 3]].tolist()))
        pos += 3
        if lo:
            # local optimisation samples from the k inliers of one group: skip them
            pos += o.LO_ITERATIONS * max(min(o.LO_SAMPLE_CLAMP, int(inl * 0.5)), 3)
    hit = [next(iter(groups[i])) for i, e in enumerate(r.events) if e[0] == k]
    assert set(hit) == {0, 1}, hit        # both groups tied the best model at some point
    want = RA if groups[last] == {0} else RB
    assert np.abs(r.R - want).max() < 1e-9
    assert r.ransac_inliers == k


def test_three_point_sample_is_proper_kabsch():
    """3 rows: the proper completion u3 = u1 x u2, v3 = v1 x v2 (the Kabsch rotation), exact for an exact rotation;
    4 or more rows: the orthogonal polar factor U V^T, negated if improper."""
    rng = np.random.RandomState(5)
    for trial in range(200):
        R = C.rotation_about(rng.randn(3), rng.uniform(0, np.pi))
        b1 = C.unit(rng.randn(3, 3))
        Q = o.rotation_between(b1, b1 @ R)     # b2 = R^T b1
        assert np.abs(Q - R).max() < 1e-12 and np.linalg.det(Q) > 0
        # against the SVD of the centred cross-covariance
        b2 = C.unit(rng.randn(3, 3))
        M = (b1 - b1.mean(0)).T @ (b2 - b2.mean(0))
        U, _, Vt = np.linalg.svd(M)
        K = U @ np.diag([1, 1, np.sign(np.linalg.det(U @ Vt))]) @ Vt
        assert np.abs(o.rotation_between(b1, b2) - K).max() < 1e-10
        b1, b2 = C.unit(rng.randn(6, 3)), C.unit(rng.randn(6, 3))
        M = (b1 - b1.mean(0)).T @ (b2 - b2.mean(0))
        U, _, Vt = np.linalg.svd(M)
        P = U @ Vt
        P = -P if np.linalg.det(P) < 0 else P
        assert np.abs(o.rotation_between(b1, b2) - P).max() < 1e-10


def test_fewer_than_three_rows_is_an_error():
    with pytest.raises(ValueError):
        o.ransac_rotation(np.eye(3)[:2], np.eye(3)[:2], 0.016)
