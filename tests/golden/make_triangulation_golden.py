"""Fixture of the reference's known-answer tests for track triangulation (opensfm/test/test_triangulation.py:7-102,
138-173), written out as data:

    python tests/golden/make_triangulation_golden.py      # writes tests/golden/triangulation_known_answers.json

Each track case is a spherical camera, two shots (world-to-camera angle-axis rotation and translation), the track's
normalised image points in each shot, TrackTriangulator.triangulate's options and the expected outcome; each
bearing case is the rays and options of TriangulateBearingsMidpoint and its expected outcome."""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
OPTIONS = {"reproj_threshold": 0.01, "min_ray_angle_degrees": 2.0, "iterations": 10}


def track_case(name, im2_translation, min_depth, expected_point):
    return {
        "name": name,
        "camera": {"projection_type": "spherical", "width": 800, "height": 400},
        "shots": {"im1": {"rotation": [0.0, 0.0, 0.0], "translation": [0.0, 0.0, 0.0]},
                  "im2": {"rotation": [0.0, 0.0, 0.0], "translation": im2_translation}},
        "observations": {"im1": [0.0, 0.0], "im2": [-0.1, 0.0]},
        "options": dict(OPTIONS, min_depth=min_depth),
        "expected_point": expected_point,
        "expected_observations": 2 if expected_point is not None else 0,
    }


def bearing_case(name, o2, expected):
    return {"name": name, "centers": [[0.0, 0.0, 0.0], o2], "bearings": [[0.0, 0.0, 1.0], [-1.0, 0.0, 1.0]],
            "max_reprojection": 0.01, "min_ray_angle_degrees": 2.0, "min_depth": 0.001, "expected": expected}


if __name__ == "__main__":
    cases = {
        "tracks": [track_case("spherical", [-1.0, 0.0, 0.0], 0.001, [0.0, 0.0, 1.3763819204711]),
                   track_case("coincident_camera_origins", [0.0, 0.0, 0.0], 0.0001, None)],
        # bearings are normalised by the test (unit_vector)
        "bearings_midpoint": [bearing_case("midpoint", [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]),
                              bearing_case("midpoint_coincident_camera_origins", [0.0, 0.0, 0.0], None)],
    }
    with open(os.path.join(HERE, "triangulation_known_answers.json"), "w") as f:
        json.dump(cases, f, indent=1)
        f.write("\n")
