"""Undistortion on the GPU: camera and face maps against the fp64 oracle (oracle/undistort_oracle.py), the sampler
against live cv2.remap bit for bit, undistort_image against cv2.remap over the GPU's own maps followed by the
reference's scale_image, the batched driver against per-shot calls, and the limits."""
import cv2
import numpy as np
import pytest

import undistort_cases as uc
from opensfm_b200 import _lib
from opensfm_b200 import undistort as GU
from opensfm_b200.types import camera_type_id, camera_values
from oracle import undistort_oracle as uo
from test_undistort_oracle import LAYOUTS, adversarial_maps, random_image

pytestmark = pytest.mark.gpu

SIZES = [(4000, 3000), (641, 479), (480, 640), (1, 1), (2, 1)]


def scale_image(image, max_size):
    """opensfm/undistort.py:224-232."""
    height, width = image.shape[:2]
    factor = max_size / float(max(height, width))
    if factor >= 1:
        return image
    width = int(round(width * factor))
    height = int(round(height * factor))
    return cv2.resize(image, (width, height), interpolation=cv2.INTER_NEAREST)


def compare_maps(got, want, what):
    """Within 2 f32 ulp; returns the number of coordinates whose rint(32 x) differs."""
    flips = 0
    for g, w in zip(got, want):
        assert g.shape == w.shape and g.dtype == np.float32
        tol = 2 * np.spacing(np.maximum(np.abs(g), np.abs(w)))
        assert np.all(np.abs(g.astype(np.float64) - w) <= tol), (what, float(np.abs(g.astype(np.float64) - w).max()))
        flips += int((uo.cv_round(g * np.float32(32)) != uo.cv_round(w * np.float32(32))).sum())
    print("%s: %d of %d fixed-point coordinates flipped" % (what, flips, 2 * got[0].size))
    assert flips <= 1e-5 * got[0].size, (what, flips)
    return flips


@pytest.mark.parametrize("model", uc.MODELS)
@pytest.mark.parametrize("strength", ["mild", "strong"])
def test_camera_maps_match_the_oracle(model, strength):
    cam = uc.camera(model, strength)
    to = uc.undistorted_camera(cam)
    for w, h in SIZES:
        got = GU.compute_camera_mapping(cam, to, w, h)
        want = uo.camera_mapping(camera_type_id(cam), camera_values(cam), to.focal, w, h)
        compare_maps(got, want, "%s %s %dx%d" % (model, strength, w, h))


@pytest.mark.parametrize("face_size", [1, 2, 479, 640])
def test_face_maps_match_the_oracle(face_size):
    shot, faces = uc.panorama(face_size)
    pw, ph = 4 * face_size, 2 * face_size
    for face in faces:
        got = GU.panorama_face_mapping(shot, face, pw, ph)
        want = uo.face_mapping(face_size, GU.face_rotation(shot, face), pw, ph)
        compare_maps(got, want, "%s %d" % (face.id, face_size))
    # an 8000x4000 panorama sampled directly
    got = GU.panorama_face_mapping(shot, faces[1], 8000, 4000)
    compare_maps(got, uo.face_mapping(face_size, GU.face_rotation(shot, faces[1]), 8000, 4000), "8000x4000 face")


@pytest.mark.parametrize("dtype,ch", LAYOUTS)
@pytest.mark.parametrize("interp", [cv2.INTER_LINEAR, cv2.INTER_AREA, cv2.INTER_NEAREST])
@pytest.mark.parametrize("border", [cv2.BORDER_CONSTANT, cv2.BORDER_WRAP])
def test_remap_equals_cv2(dtype, ch, interp, border):
    for (w, h), seed in (((41, 29), 0), ((1, 1), 1), ((2, 1), 2)):
        img = random_image(dtype, ch, w, h, seed=seed)
        mx, my = adversarial_maps(w, h, seed=seed)
        got = GU.remap(img, mx, my, interp, border)
        want = cv2.remap(img, mx, my, interp, borderMode=border)
        assert got.shape == want.shape and got.dtype == want.dtype
        assert np.array_equal(got, want), ((w, h), int((got != want).sum()))


def _camera_reference(shot, subs, image, interp, max_size):
    to = subs[0].camera
    h, w = image.shape[:2]
    return {subs[0].id: scale_image(cv2.remap(image, *GU.compute_camera_mapping(shot.camera, to, w, h), interp),
                                    max_size)}


def _panorama_reference(shot, subs, image, interp, max_size):
    s = subs[0].camera.width
    pano = cv2.resize(image, (4 * s, 2 * s), interpolation=interp)
    mint = cv2.INTER_LINEAR if interp == cv2.INTER_AREA else interp
    return {f.id: scale_image(cv2.remap(pano, *GU.panorama_face_mapping(shot, f, 4 * s, 2 * s), mint,
                                        borderMode=cv2.BORDER_WRAP), max_size) for f in subs}


def _assert_same(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].shape == want[k].shape and got[k].dtype == want[k].dtype, k
        assert np.array_equal(got[k], want[k]), (k, int((got[k] != want[k]).sum()))


@pytest.mark.parametrize("model", uc.MODELS)
def test_undistort_image_equals_remap_over_the_gpus_maps(model):
    rng = np.random.RandomState(3)
    for (w, h), strength in (((641, 479), "strong"), ((480, 640), "mild")):
        shot, subs = uc.shot_pair(model, strength, w, h)
        image = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        mask = (rng.rand(h, w) > 0.3).astype(np.uint8)
        seg = rng.randint(0, 20, (h, w)).astype(np.uint8)
        for max_size in (10000, 640, 333, 1):
            _assert_same(GU.undistort_image(shot, subs, image, cv2.INTER_AREA, max_size),
                         _camera_reference(shot, subs, image, cv2.INTER_AREA, max_size))
            for arr in (mask, seg):
                _assert_same(GU.undistort_image(shot, subs, arr, cv2.INTER_NEAREST, max_size),
                             _camera_reference(shot, subs, arr, cv2.INTER_NEAREST, max_size))


def test_undistort_image_of_a_panorama_equals_the_references_render():
    rng = np.random.RandomState(4)
    shot, subs = uc.panorama(160)
    image = rng.randint(0, 256, (1000, 2000, 3)).astype(np.uint8)
    mask = (rng.rand(1000, 2000) > 0.5).astype(np.uint8)
    for max_size in (10000, 100):
        _assert_same(GU.undistort_image(shot, subs, image, cv2.INTER_AREA, max_size),
                     _panorama_reference(shot, subs, image, cv2.INTER_AREA, max_size))
        _assert_same(GU.undistort_image(shot, subs, mask, cv2.INTER_NEAREST, max_size),
                     _panorama_reference(shot, subs, mask, cv2.INTER_NEAREST, max_size))
    # the face renderer itself, in every interpolation and border
    pano = cv2.resize(image, (640, 320), interpolation=cv2.INTER_AREA)
    for interp in (cv2.INTER_LINEAR, cv2.INTER_NEAREST):
        for border in (cv2.BORDER_WRAP, cv2.BORDER_CONSTANT):
            got = GU.render_perspective_view_of_a_panorama(pano, shot, subs[4], interp, border)
            want = cv2.remap(pano, *GU.panorama_face_mapping(shot, subs[4], 640, 320), interp, borderMode=border)
            assert np.array_equal(got, want)


def _dataset(max_size=500):
    rng = np.random.RandomState(6)
    pairs, images, masks, segs = [], {}, {}, {}
    for k in range(11):
        model = uc.MODELS[k % len(uc.MODELS)]
        w, h = (120 + 7 * k, 90 + 5 * k) if k % 3 else (90 + 5 * k, 120 + 7 * k)
        shot, subs = uc.shot_pair(model, "strong" if k % 2 else "mild", w, h, sid="s%d" % k)
        pairs.append((shot, subs))
        dtype = np.uint16 if k == 4 else np.uint8
        images[shot.id] = random_image(dtype, 3 if k % 4 else 4, w, h, seed=10 + k)
        if k % 3 != 1:
            masks[shot.id] = (rng.rand(h, w) > 0.4).astype(np.uint8)
        if k % 2 == 0:
            segs[shot.id] = rng.randint(0, 9, (h, w)).astype(np.uint8)
    shot, subs = uc.panorama(64, sid="p0")
    pairs.append((shot, subs))
    images[shot.id] = random_image(np.uint8, 3, 600, 300, seed=99)
    masks[shot.id] = (rng.rand(300, 600) > 0.5).astype(np.uint8)
    return dict(pairs), uc.DataSet(images, masks, segs, max_size=max_size)


def test_driver_saves_what_undistort_image_returns():
    shots, data = _dataset()
    want = {}
    for shot, subs in shots.items():
        for kind, arr, interp in (("image", data.images.get(shot.id), cv2.INTER_AREA),
                                  ("mask", data.masks.get(shot.id), cv2.INTER_NEAREST),
                                  ("segmentation", data.segmentations.get(shot.id), cv2.INTER_NEAREST)):
            for k, v in GU.undistort_image(shot, subs, arr, interp, data.config["undistorted_image_max_size"]).items():
                want[(kind, k)] = v
    small = uc.UndistortedDataSet()
    GU.undistort_images(data, small, shots, batch_size=2)
    big = uc.UndistortedDataSet()
    GU.undistort_images(data, big, list(shots.items()), batch_size=1000)
    assert len(want) == 11 + 6 + 7 + 6 + 6   # images, panorama faces, masks, panorama mask faces, segmentations
    for got in (small.saved, big.saved):
        assert sorted(got) == sorted(want)
        for k in want:
            assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), k
    # and each saved image is the reference's for its shot
    s3 = [s for s in shots if s.id == "s3"][0]
    ref = _camera_reference(s3, shots[s3], data.images["s3"], cv2.INTER_AREA, 500)
    assert np.array_equal(small.saved[("image", "s3.jpg")], ref["s3.jpg"])


def test_limits():
    shot, subs = uc.shot_pair("fisheye62", "strong", 8000, 6000)
    big = np.random.RandomState(1).randint(0, 65536, (6000, 8000, 3)).astype(np.uint16)
    got = GU.undistort_image(shot, subs, big, cv2.INTER_AREA, 100000)[subs[0].id]
    want = cv2.remap(big, *GU.compute_camera_mapping(shot.camera, subs[0].camera, 8000, 6000), cv2.INTER_AREA)
    assert np.array_equal(got, want)
    del big, got, want
    launches = _lib.load().osfm_kernel_launch_count()
    for bad in (np.zeros((60, 80), np.float32), np.zeros((60, 80, 2), np.uint8)):
        with pytest.raises(NotImplementedError, match="float32|shape"):
            GU.undistort_image(*uc.shot_pair("brown", "mild", 80, 60), bad, cv2.INTER_AREA, 100)
    assert _lib.load().osfm_kernel_launch_count() == launches
    with pytest.raises(NotImplementedError, match="Undistort not implemented for projection type: radial"):
        radial = uc.Camera.create_radial(0.5, 1.0, [0, 0], [0.1, 0.0])
        GU.undistort_image(uc.Shot("r", radial), subs, np.zeros((6, 8), np.uint8), cv2.INTER_AREA, 100)
    for model in uc.MODELS:
        shot, subs = uc.shot_pair(model, "strong", 1, 1)
        img = np.array([[[7, 8, 9]]], np.uint8)
        for interp in (cv2.INTER_AREA, cv2.INTER_NEAREST):
            _assert_same(GU.undistort_image(shot, subs, img, interp, 10),
                         _camera_reference(shot, subs, img, interp, 10))
