"""The host restatement of the bundle adjustment's point layout (tests/ba_layout_reference.py) on hand-built cases
whose segment counts are worked out by hand: the 64-point cut, the k * wc <= 96 limit at wc = 9 and wc = 7, constant
points, point priors and duplicate observations.  test_ba_input_order_gpu.py holds the device's counts to it."""
import numpy as np
import pytest

import ba_layout_reference as ref


def _runs(sizes, shot_lists, wc=9, const=None, prior=None):
    """sizes[i] points, each seen by exactly shot_lists[i]."""
    obs_shot, obs_point = [], []
    p = 0
    for n, shots in zip(sizes, shot_lists):
        for _ in range(n):
            for s in shots:
                obs_shot.append(s)
                obs_point.append(p)
            p += 1
    const = np.zeros(p, dtype=np.int32) if const is None else const
    prior = np.zeros(p, dtype=bool) if prior is None else prior
    return ref.layout(obs_shot, obs_point, const, prior, wc)


@pytest.mark.parametrize("n,nseg", [(1, 1), (63, 1), (64, 1), (65, 2), (128, 2), (129, 3), (300, 5)])
def test_one_run_is_cut_every_64_points(n, nseg):
    lay = _runs([n], [[0, 1, 2]])
    assert (lay.nseg, lay.p_fast, lay.p_slow, lay.n_fast) == (nseg, n, 0, 3 * n)


def test_runs_of_different_shot_lists_are_cut_separately():
    lay = _runs([64, 65, 129, 1], [[0, 1], [1, 2], [0, 1, 2], [2, 0]])
    # {0, 2} listed as [2, 0] is its own shot list; the cut does not carry over from one run to the next
    assert lay.nseg == 1 + 2 + 3 + 1 and lay.p_fast == 64 + 65 + 129 + 1
    assert lay.group_sizes == [129, 65, 64, 1]


def test_interleaved_points_of_one_shot_list_form_one_run():
    """Points of the same shot list need not be adjacent in the caller's order: 40 + 40 points of {0, 1, 2} with 30
    points of {0, 1} between them are one run of 80 (two segments) and one of 30."""
    obs_shot, obs_point = [], []
    lists = [[0, 1, 2]] * 40 + [[0, 1]] * 30 + [[0, 1, 2]] * 40
    for p, shots in enumerate(lists):
        for s in shots[::-1]:   # a point's observations in any order
            obs_shot.append(s)
            obs_point.append(p)
    lay = ref.layout(obs_shot, obs_point, np.zeros(110), np.zeros(110, dtype=bool), 9)
    assert lay.nseg == 3 and lay.group_sizes == [80, 30]


@pytest.mark.parametrize("k,eligible", [(10, True), (11, False)])
def test_k_limit_at_wc_9(k, eligible):
    """wc = 9 (a 3-parameter camera and the instance pose): 10 shots are 90 camera-side columns, 11 are 99 > 96."""
    lay = _runs([70], [list(range(k))], wc=9)
    assert lay.p_fast == (70 if eligible else 0) and lay.p_slow == (0 if eligible else 70)
    assert lay.nseg == (2 if eligible else 0) and lay.n_fast == (70 * k if eligible else 0)


@pytest.mark.parametrize("k,eligible", [(13, True), (14, False)])
def test_k_limit_at_wc_7(k, eligible):
    """wc = 7 (SPHERICAL: one camera parameter): 13 shots are 91 columns, 14 are 98 > 96."""
    lay = _runs([5], [list(range(k))], wc=7)
    assert lay.p_fast == (5 if eligible else 0) and lay.nseg == (1 if eligible else 0)


def test_wide_camera_sides_and_the_per_point_fallback_have_no_segment():
    assert _runs([10], [[0, 1]], wc=16).nseg == 1
    assert _runs([10], [[0, 1]], wc=17).nseg == 0   # wc > 16 (e.g. BROWN through a rig camera: 9 + 6 + 6)
    assert _runs([10], [list(range(16))], wc=6).p_fast == 10
    assert _runs([10], [list(range(17))], wc=5).p_fast == 0   # k > 16 whatever wc
    obs_shot, obs_point = [0, 1] * 10, np.repeat(np.arange(10), 2)
    lay = ref.layout(obs_shot, obs_point, np.zeros(10), np.zeros(10, dtype=bool), 9, per_point_fallback=True)
    assert (lay.p_fast, lay.p_slow, lay.nseg) == (0, 10, 0)


def test_constant_point_between_free_points_of_its_shot_list():
    """A constant point between two free points that share its shot list: the free points are one run, the constant
    one its own, whatever the caller's order (2 segments, not 1 and not 3)."""
    lay = _runs([1, 1, 1], [[0, 1, 2]] * 3, const=np.array([0, 1, 0]))
    assert (lay.nseg, lay.p_fast, lay.p_slow) == (2, 3, 0)
    assert lay.group_sizes == [2, 1]


def test_point_with_a_prior_is_off_the_segment_path():
    lay = _runs([3], [[0, 1]], prior=np.array([False, True, False]))
    assert (lay.nseg, lay.p_fast, lay.p_slow, lay.n_fast) == (1, 2, 1, 4)
    assert lay.eligible.tolist() == [True, False, True]


def test_duplicate_observation_makes_its_own_shot_list():
    """A point observed twice by shot 1 has the shot list (0, 1, 1, 2): k = 4, not the run of (0, 1, 2)."""
    obs_shot = [0, 1, 2] * 3 + [1]
    obs_point = [0, 0, 0, 1, 1, 1, 2, 2, 2, 1]
    lay = ref.layout(obs_shot, obs_point, np.zeros(3), np.zeros(3, dtype=bool), 9)
    assert (lay.nseg, lay.p_fast, lay.n_fast) == (2, 3, 10) and lay.group_sizes == [2, 1]
    # at wc = 9, a point of 10 shots with one of them twice has k = 11: off the segment path
    obs_shot = list(range(10)) + [3]
    lay = ref.layout(obs_shot, [0] * 11, np.zeros(1), np.zeros(1, dtype=bool), 9)
    assert (lay.p_fast, lay.p_slow) == (0, 1)


def test_unobserved_points_are_off_the_segment_path():
    lay = ref.layout([0, 1], [1, 1], np.zeros(3), np.zeros(3, dtype=bool), 9)
    assert lay.eligible.tolist() == [False, True, False] and (lay.p_fast, lay.p_slow, lay.nseg) == (1, 2, 1)
