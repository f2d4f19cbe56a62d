"""The checking all-reduce of tests/ba_ranks.py on host buffers (no GPU): sums in rank order with the same bits on every
rank, a count mismatch raising on every rank, and a rank that never arrives ending in a timeout instead of a hang."""
import ctypes
import time

import numpy as np
import pytest

from ba_ranks import RankFailure, run_threads


def _call(allreduce, buf):
    allreduce(buf.ctypes.data_as(ctypes.c_void_p).value, len(buf), 0)
    return buf


@pytest.mark.parametrize("world", [2, 3])
def test_sums_in_rank_order_on_every_rank(world):
    rng = np.random.RandomState(world)
    # per rank: a large term and a small one at slot 0 whose sum depends on the order of the additions
    # ((1e16 + 1) - 1e16 = 0 in fp64, 1e16 - 1e16 + 1 = 1), then random data, then a second call of another size
    first = [np.concatenate([[v], rng.standard_normal(17)]) for v in ([1e16, 1.0, -1e16][:world] if world == 3
                                                                      else [1e16, 1.0])]
    second = [rng.standard_normal(5) * 10.0 ** r for r in range(world)]

    def body(r, allreduce):
        return _call(allreduce, first[r].copy()).copy(), _call(allreduce, second[r].copy()).copy()

    out = run_threads(world, body, device=None, timeout=30.0)
    for want_in, k in ((first, 0), (second, 1)):
        want = want_in[0].copy()
        for b in want_in[1:]:
            want += b
        for r in range(world):
            assert out[r][k].tobytes() == want.tobytes(), (r, k)
    if world == 3:
        assert out[0][0][0] == 0.0   # (1e16 + 1) + (-1e16): rank order, not a pairwise or reversed order


def test_count_mismatch_raises_on_every_rank():
    world = 3

    def body(r, allreduce):
        _call(allreduce, np.ones(4))
        _call(allreduce, np.ones(6 if r == 1 else 3))   # rank 1 exchanges another buffer at call #1
        return "done"

    t0 = time.time()
    with pytest.raises(RankFailure) as e:
        run_threads(world, body, device=None, timeout=30.0)
    assert time.time() - t0 < 10.0
    msg = str(e.value)
    for r in range(world):
        assert "rank %d: RankFailure: all-reduce #1: the ranks' counts differ: rank 0: 3, rank 1: 6, rank 2: 3" % r in msg
    assert "first difference at #1" in msg


def test_missing_rank_times_out():
    world = 3

    def body(r, allreduce):
        if r == 2:
            time.sleep(3.0)   # arrives long after the others gave up
            return "late"
        return _call(allreduce, np.ones(2))

    t0 = time.time()
    with pytest.raises(RankFailure) as e:
        run_threads(world, body, device=None, timeout=0.5)
    assert time.time() - t0 < 10.0
    msg = str(e.value)
    # the first rank to time out says why; the other gives up with it
    assert "not every rank arrived within 0.5 s" in msg
    for r in (0, 1):
        assert "rank %d: RankFailure: all-reduce #0 (count 2) on rank %d: " % (r, r) in msg


def test_rank_that_leaves_early_fails_the_others():
    """A rank whose solve ends while the others still exchange (fewer all-reduces) fails them at once."""

    def body(r, allreduce):
        _call(allreduce, np.ones(2))
        if r == 0:
            _call(allreduce, np.ones(2))
        return r

    t0 = time.time()
    with pytest.raises(RankFailure) as e:
        run_threads(2, body, device=None, timeout=60.0)
    assert time.time() - t0 < 10.0
    assert "all-reduce #1 (count 2) on rank 0: rank(s) [1] had finished their solve" in str(e.value)
