"""oracle/tracks_oracle.py on hand-built match graphs with known answers (no GPU)."""
from oracle import tracks_oracle as to

ALL = ("a", "b", "c", "d")


def fs(*obs):
    return frozenset(obs)


def test_chain_through_three_images_is_one_track():
    matches = {("a", "b"): [(0, 5)], ("b", "c"): [(5, 7)]}
    part, common = to.tracks(ALL, matches, 2)
    assert part == {fs(("a", 0), ("b", 5), ("c", 7))}
    assert common == {("a", "b"): [(0, 5)], ("a", "c"): [(0, 7)], ("b", "c"): [(5, 7)]}


def test_two_features_of_one_image_joined_through_another_are_dropped():
    matches = {("a", "b"): [(0, 5), (1, 5), (2, 6)]}
    part, common = to.tracks(ALL, matches, 2)
    assert part == {fs(("a", 2), ("b", 6))}
    assert common == {("a", "b"): [(2, 6)]}


def test_pair_listed_in_both_orders():
    matches = {("a", "b"): [(0, 5), (1, 6)], ("b", "a"): [(5, 0), (7, 2)]}
    part, common = to.tracks(ALL, matches, 2)
    assert part == {fs(("a", 0), ("b", 5)), fs(("a", 1), ("b", 6)), fs(("a", 2), ("b", 7))}
    assert sorted(common[("a", "b")]) == [(0, 5), (1, 6), (2, 7)]
    assert list(common) == [("a", "b")]


def test_min_length():
    matches = {("a", "b"): [(0, 0), (1, 1)], ("b", "c"): [(1, 1)]}
    assert to.tracks(ALL, matches, 2)[0] == {fs(("a", 0), ("b", 0)), fs(("a", 1), ("b", 1), ("c", 1))}
    assert to.tracks(ALL, matches, 3)[0] == {fs(("a", 1), ("b", 1), ("c", 1))}
    assert to.tracks(ALL, matches, 4) == (set(), {})


def test_image_without_features_counts_but_yields_no_observation():
    matches = {("a", "x"): [(0, 3), (1, 4), (2, 4)], ("x", "b"): [(3, 9)]}
    # x has no feature file: it lengthens a-x-b to 3, kills the track where it is matched twice from a ...
    part, common = to.tracks(("a", "b"), matches, 3)
    assert part == {fs(("a", 0), ("b", 9))}
    assert common == {("a", "b"): [(0, 9)]}
    # ... and a track it leaves with one observation still exists, joining no pair
    part, common = to.tracks(("a", "b"), {("a", "x"): [(0, 3)]}, 2)
    assert part == {fs(("a", 0))}
    assert common == {}
    # a track only of such images does not exist
    assert to.tracks(("a",), {("x", "y"): [(0, 0)]}, 2) == (set(), {})


def test_self_match_kills_its_track():
    matches = {("a", "a"): [(0, 1)], ("a", "b"): [(0, 0), (2, 2)]}
    assert to.tracks(ALL, matches, 2)[0] == {fs(("a", 2), ("b", 2))}


def test_empty_matches():
    assert to.tracks(ALL, {}, 2) == (set(), {})
    assert to.tracks(ALL, {("a", "b"): []}, 2) == (set(), {})
