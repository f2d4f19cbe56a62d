"""compute_depthmaps on an in-memory UndistortedDataSet against the reference's own steps (opensfm/dense.py's
compute_depthmap, clean_depthmap and prune_depthmap) driven through the pydense mirror classes one shot at a time;
the cleaner mirror and raw maps uploaded with set_maps."""
import numpy as np
import pytest

import dense_fakes as F
from opensfm_b200 import dense as D
from oracle import dense_oracle as do

pytestmark = pytest.mark.gpu


def _reference_steps(data, tm, rec, seed):
    """opensfm/dense.py's compute_depthmaps with pydense = opensfm_b200.dense, one shot at a time."""
    cfg = data.config
    common = D.common_tracks_double_dict(tm)
    neighbors = {s.id: D.find_neighboring_images(s, common, rec, cfg["depthmap_num_neighbors"])
                 for s in rec.shots.values()}
    shots = [s for s in rec.shots.values() if len(neighbors[s.id]) > 1]
    view = {}
    for s in shots:
        for n in neighbors[s.id]:
            view.setdefault(n.id, D._load_view(data, n, cfg["depthmap_resolution"]))
    for s in shots:
        if data.raw_depthmap_exists(s.id):
            continue
        mind, maxd = D.compute_depth_range(tm, rec, s, cfg)
        de = D.DepthmapEstimator(seed=seed, key=D.shot_key(s.id))
        de.set_depth_range(mind, maxd, 100)
        de.set_patchmatch_iterations(cfg["depthmap_patchmatch_iterations"])
        de.set_patch_size(cfg["depthmap_patch_size"])
        de.set_min_patch_sd(cfg["depthmap_min_patch_sd"])
        for n in neighbors[s.id][:cfg["depthmap_num_matching_views"] + 1]:
            v = view[n.id]
            de.add_view(v.K, v.R, v.t, v.gray, v.mask)
        depth, plane, score, nghbr = de.compute_patch_match_sample()
        depth = depth * (depth < np.float64(maxd)) * (score > cfg["depthmap_min_correlation_score"])
        data.save_raw_depthmap(s.id, depth, plane, score, nghbr, [n.id for n in neighbors[s.id][1:]])
    for s in shots:
        dc = D.DepthmapCleaner()
        dc.set_same_depth_threshold(cfg["depthmap_same_depth_threshold"])
        dc.set_min_consistent_views(cfg["depthmap_min_consistent_views"])
        for n in neighbors[s.id]:
            if data.raw_depthmap_exists(n.id):
                v = view[n.id]
                dc.add_view(v.K, v.R, v.t, data.load_raw_depthmap(n.id)[0])
        raw = data.load_raw_depthmap(s.id)
        data.save_clean_depthmap(s.id, dc.clean(), raw[1], raw[2])
    for s in shots:
        dp = D.DepthmapPruner()
        dp.set_same_depth_threshold(cfg["depthmap_same_depth_threshold"])
        for n in neighbors[s.id]:
            depth, plane, _ = data.load_clean_depthmap(n.id)
            v = view[n.id]
            dp.add_view(v.K, v.R, v.t, depth, plane, v.color, v.labels)
        data.save_pruned_depthmap(s.id, *dp.prune())
    data.save_point_cloud(*D.merge_depthmaps(data, rec), filename="merged.ply")


def test_compute_depthmaps_equals_reference_steps(tmp_path):
    rec, tm, images = F.scene(5)
    want = F.DataSet(images, str(tmp_path))
    got = F.DataSet(images, str(tmp_path))
    # a raw map computed earlier, for the second shot, is reused by both
    pre = F.DataSet(images, str(tmp_path))
    _reference_steps(pre, tm, rec, seed=9)
    for d in (want, got):
        d.raw["s1"] = pre.raw["s1"]
    _reference_steps(want, tm, rec, seed=3)
    D.compute_depthmaps(got, tm, rec, seed=3)
    assert "s5" not in got.raw and "s5" not in got.pruned          # the lone shot has no neighbour: skipped
    assert set(got.raw) == set(want.raw) == {"s0", "s1", "s2", "s3", "s4"}
    for sid in want.raw:
        for a, b in zip(got.raw[sid], want.raw[sid]):
            assert np.array_equal(np.asarray(a), np.asarray(b)), sid
        for a, b in zip(got.clean[sid], want.clean[sid]):
            assert np.array_equal(a, b), sid
        for a, b in zip(got.pruned[sid], want.pruned[sid]):
            assert np.array_equal(a, b), sid
    assert np.array_equal(got.raw["s1"][0], pre.raw["s1"][0])
    for a, b in zip(got.clouds["merged.ply"][0], want.clouds["merged.ply"][0]):
        assert np.array_equal(a, b)
    assert len(got.clouds["merged.ply"][0][0]) > 1000
    assert (tmp_path / "s0.raw.npz.ply").exists() and (tmp_path / "s0.clean.npz.ply").exists()


def test_cleaner_mirror_and_uploaded_raw_maps_equal_oracle():
    rec, tm, images = F.scene(4, 64, 48)
    data = F.DataSet(images, "")
    views = [D._load_view(data, s, 640) for s in list(rec.shots.values())[:4]]
    rng = np.random.RandomState(2)
    depths = [rng.uniform(4, 9, (48, 64)).astype(np.float32) for _ in range(4)]
    depths[0][::3] = 0
    want = {m: do.clean([v.K for v in views], [v.R for v in views], [v.t for v in views], depths, 0.05, m)
            for m in (1, 2, 3)}
    for m in (1, 2, 3):
        dc = D.DepthmapCleaner()
        dc.set_same_depth_threshold(0.05)
        dc.set_min_consistent_views(m)
        for v, d in zip(views, depths):
            dc.add_view(v.K, v.R, v.t, d)
        assert np.array_equal(dc.clean(), want[m]), m
    for v, d in zip(views, depths):
        v.raw_depth, v.plane = d, np.zeros((48, 64, 3), np.float32)
    with D.Engine(views) as E:
        got = E.clean([[0, 1, 2, 3], [2, 0]], 0.05, 2)
    assert np.array_equal(got[0], want[2])
    v2 = [views[2], views[0]]
    assert np.array_equal(got[1], do.clean([v.K for v in v2], [v.R for v in v2], [v.t for v in v2],
                                           [depths[2], depths[0]], 0.05, 2))
