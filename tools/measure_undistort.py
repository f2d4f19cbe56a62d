"""Undistortion cost per image: device ms by CUDA events (upload, kernel, download) of `undistort_image` for a
4000x3000 RGB uint8 image of each undistortable model and for the six 640x640 faces of an 8000x4000 panorama (the
reference's default depthmap_resolution); the host's cv2.remap over the same maps (mapping excluded) and the host's
cv2.resize of the panorama; JPEG decode and encode of the 4000x3000 image with cv2; the card's name and power limit.

    python tools/measure_undistort.py [--repeats 5]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import cv2  # noqa: E402

import undistort_cases as uc  # noqa: E402
from opensfm_b200 import _lib  # noqa: E402
from opensfm_b200 import undistort as GU  # noqa: E402


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "not measured"
    return name, out


def device_ms():
    """upload, kernel and download ms of the last call on the pooled handle (the one the call released)."""
    a, b, c = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
    with _lib.pooled("undistort", 0) as h:
        _lib.check(h.L.osfm_undistort_last_device_ms(h.h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)))
    return a.value, b.value, c.value


def timed(fn, repeats):
    """median wall ms of fn() and the median device (upload, kernel, download) ms after it"""
    fn()
    walls, devs = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        walls.append(1e3 * (time.perf_counter() - t0))
        devs.append(device_ms())
    return float(np.median(walls)), [float(np.median([d[k] for d in devs])) for k in range(3)]


def host_ms(fn, repeats):
    fn()
    out = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        out.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    rng = np.random.RandomState(0)
    # a smooth image, so the JPEG sizes are those of a photograph rather than of noise
    y, x = np.mgrid[0:3000, 0:4000]
    image = np.dstack([(127 + 100 * np.sin(x / 37.0 + k) * np.cos(y / 53.0 - k)).astype(np.uint8) for k in range(3)])
    image = np.ascontiguousarray(image + rng.randint(0, 8, image.shape).astype(np.uint8))
    name, power = card()
    res = {"card": name, "power_limit": power, "cv2_threads": cv2.getNumThreads(), "models": {}}
    for model in uc.MODELS:
        shot, subs = uc.shot_pair(model, "mild", 4000, 3000)
        wall, (up, kern, down) = timed(lambda: GU.undistort_image(shot, subs, image, cv2.INTER_AREA, 100000),
                                       a.repeats)
        maps = GU.compute_camera_mapping(shot.camera, subs[0].camera, 4000, 3000)
        remap = host_ms(lambda: cv2.remap(image, *maps, cv2.INTER_AREA), a.repeats)
        res["models"][model] = {"kernel_ms": kern, "h2d_ms": up, "d2h_ms": down, "wall_ms": wall,
                                "host_cv2_remap_ms": remap}
    shot, subs = uc.panorama(640)
    pano = np.ascontiguousarray(cv2.resize(image, (8000, 4000), interpolation=cv2.INTER_LINEAR))
    wall, (up, kern, down) = timed(lambda: GU.undistort_image(shot, subs, pano, cv2.INTER_AREA, 100000), a.repeats)
    small = cv2.resize(pano, (2560, 1280), interpolation=cv2.INTER_AREA)
    fmaps = [GU.panorama_face_mapping(shot, f, 2560, 1280) for f in subs]
    remap = host_ms(lambda: [cv2.remap(small, *m, cv2.INTER_LINEAR, borderMode=cv2.BORDER_WRAP) for m in fmaps],
                    a.repeats)
    resize = host_ms(lambda: cv2.resize(pano, (2560, 1280), interpolation=cv2.INTER_AREA), a.repeats)
    res["panorama_8000x4000_six_faces"] = {"kernel_ms": kern, "h2d_ms": up, "d2h_ms": down, "wall_ms": wall,
                                           "host_cv2_remap_ms": remap, "host_cv2_resize_ms": resize}
    ok, jpg = cv2.imencode(".jpg", image)
    res["host_jpeg_4000x3000"] = {"decode_ms": host_ms(lambda: cv2.imdecode(jpg, cv2.IMREAD_UNCHANGED), a.repeats),
                                  "encode_ms": host_ms(lambda: cv2.imencode(".jpg", image), a.repeats),
                                  "bytes": int(len(jpg))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
