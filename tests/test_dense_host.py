"""The dense driver's host helpers on the CPU: the reference's test_dense.py cases, and find_neighboring_images /
compute_depth_range against direct loop restatements of opensfm/dense.py."""
import numpy as np

from opensfm_b200 import dense as D
import dense_fakes as F


def test_angle_between_points():
    assert np.allclose(D.angle_between_points([0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]), np.pi / 2)
    assert np.allclose(D.angle_between_points([10.0, 15.0, 20.0], [10.0, 16.0, 20.0], [10.0, 16.0, 21.0]), np.pi / 4)


def test_depthmap_to_ply():
    height, width = 2, 3
    shot = F.Shot("shot1", F.Camera(width, height, 0.8), F.Pose(np.eye(3), np.zeros(3)))
    ply = D.depthmap_to_ply(shot, np.ones((height, width)), np.zeros((height, width, 3)))
    assert len(ply.splitlines()) == 16


def _angle_loop(origin, p1, p2):
    a0, a1, a2 = p1[0] - origin[0], p1[1] - origin[1], p1[2] - origin[2]
    b0, b1, b2 = p2[0] - origin[0], p2[1] - origin[1], p2[2] - origin[2]
    dot = a0 * b0 + a1 * b1 + a2 * b2
    la = a0 * a0 + a1 * a1 + a2 * a2
    lb = b0 * b0 + b1 * b1 + b2 * b2
    return np.arccos(dot / np.sqrt(la * lb))


def _neighbors_loop(shot, common_tracks, reconstruction, num_neighbors):
    ns = []
    C1 = shot.pose.get_origin()
    for other_id, tracks in common_tracks.get(shot.id, {}).items():
        if other_id not in reconstruction.shots:
            continue
        other = reconstruction.shots[other_id]
        score = 0
        C2 = other.pose.get_origin()
        for track in tracks:
            if track in reconstruction.points:
                theta = _angle_loop(reconstruction.points[track].coordinates, C1, C2)
                if np.pi / 60 < theta < np.pi / 6:
                    score += 1
        if score > 20:
            ns.append((other, score))
    ns.sort(key=lambda ns: ns[1], reverse=True)
    return [shot] + [n for n, s in ns[:num_neighbors]]


def _range_loop(tm, rec, shot, config):
    depths = [shot.pose.transform(rec.points[t].coordinates)[2] for t in tm.get_shot_observations(shot.id)
              if t in rec.points]
    mind, maxd = np.percentile(depths, 10) * 0.9, np.percentile(depths, 90) * 1.1
    return config["depthmap_min_depth"] or mind, config["depthmap_max_depth"] or maxd


def test_neighbors_and_depth_range_against_loops():
    rec, tm, _ = F.scene(7, seed=4)
    rec.points.pop("t5")                                      # a track that is not reconstructed
    common = D.common_tracks_double_dict(tm)
    assert common["s7"] == {} and set(common["s0"]) == {"s%d" % k for k in range(1, 7)}
    for num in (1, 3, 10):
        for shot in rec.shots.values():
            assert [s.id for s in D.find_neighboring_images(shot, common, rec, num)] == [
                s.id for s in _neighbors_loop(shot, common, rec, num)]
    for shot in list(rec.shots.values())[:7]:
        for cfg in (F.CONFIG, dict(F.CONFIG, depthmap_min_depth=1.5, depthmap_max_depth=30.0)):
            got, want = D.compute_depth_range(tm, rec, shot, cfg), _range_loop(tm, rec, shot, cfg)
            assert np.allclose(got, want, rtol=1e-13, atol=0)
