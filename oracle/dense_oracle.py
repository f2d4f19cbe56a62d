"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product.

ctypes binding of oracle/dense_oracle.cpp, the raster-order restatement of pydense's DepthmapEstimator,
DepthmapCleaner and DepthmapPruner (opensfm/src/dense/src/depthmap.cc), one reference shot per call.  Its rules,
and where it departs from the reference (the seeded generator), are stated at the top of the C++ file.  The
reference itself cannot be compiled without the OpenCV C++ headers, so the restatement is checked against the
reference's own unit tests (tests/test_dense_oracle.py), not against a compiled reference.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import c_double, c_float, c_int, c_uint32, c_void_p

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "dense_oracle.cpp")
_LIB_PATH = os.path.join(_HERE, "_build", "libdense_oracle.so")
# no -march: contraction to FMA must stay off for the comparison with the engine (compiled with -fmad=false)
CXXFLAGS = ["-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-fno-fast-math"]

_lib = None


def build(force: bool = False) -> str:
    """Compile oracle/_build/libdense_oracle.so (g++, a few seconds)."""
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_SRC) > os.path.getmtime(_LIB_PATH):
        os.makedirs(os.path.dirname(_LIB_PATH), exist_ok=True)
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-o", _LIB_PATH, _SRC])
    return _LIB_PATH


def _load():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build())
        L.dn_estimate.restype = c_int
        L.dn_estimate.argtypes = [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                  c_int, c_int, c_int, c_float, c_double, c_double, c_void_p, c_uint32, c_uint32,
                                  c_void_p, c_void_p, c_void_p, c_void_p]
        L.dn_clean.restype = None
        L.dn_clean.argtypes = [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int,
                               c_void_p]
        L.dn_prune.restype = ctypes.c_longlong
        L.dn_prune.argtypes = [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p]
        L.dn_median5.argtypes = [c_void_p, c_int, c_int, c_void_p]
        L.dn_homography.argtypes = [c_void_p] * 6
        L.dn_plane_from_depth_normal.argtypes = [c_float, c_float, c_void_p, c_float, c_void_p, c_void_p]
        L.dn_depth_of_plane.restype = c_float
        L.dn_depth_of_plane.argtypes = [c_double, c_double, c_void_p, c_void_p]
        L.dn_backproject.argtypes = [c_double, c_double, c_double, c_void_p, c_void_p, c_void_p, c_void_p]
        L.dn_project.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
        L.dn_ncc.restype = c_float
        L.dn_ncc.argtypes = [c_int, c_void_p, c_void_p, c_void_p]
        L.dn_log.restype = c_double
        L.dn_log.argtypes = [c_double]
        L.dn_exp.restype = c_double
        L.dn_exp.argtypes = [c_double]
        L.dn_normal.restype = c_float
        L.dn_normal.argtypes = [c_uint32] * 5
        L.dn_philox.argtypes = [c_uint32] * 6 + [c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(c_void_p)


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def _ptr_array(arrays):
    return (c_void_p * len(arrays))(*[a.ctypes.data for a in arrays])


METHODS = {"BRUTE_FORCE": 0, "PATCH_MATCH": 1, "PATCH_MATCH_SAMPLE": 2}


def estimate(Ks, Rs, ts, images, mask, method, patch_size=7, num_depth_planes=50, iterations=3,
             min_patch_variance=25.0, min_depth=0.0, max_depth=0.0, weights=None, seed=0, key=0):
    """One reference (view 0) against views 1..n-1: (depth, plane, score, nghbr), ungated, as pydense returns them.
    K^-1, Q and a come from opensfm_b200.dense.view_terms, the same numpy code the engine's host side runs."""
    from opensfm_b200 import dense as D

    L = _load()
    n = len(images)
    images = [_c(im, np.uint8) for im in images]
    size = _c([(im.shape[1], im.shape[0]) for im in images], np.int32)
    Kinv, Q, a = D.view_terms(Ks, Rs, ts)
    K = _c(Ks, np.float64)
    w = D.bilateral_weights() if weights is None else _c(weights, np.float32)
    h, wd = images[0].shape
    depth = np.zeros((h, wd), np.float32)
    plane = np.zeros((h, wd, 3), np.float32)
    score = np.zeros((h, wd), np.float32)
    nghbr = np.zeros((h, wd), np.int32)
    keep = _ptr_array(images)
    mask = _c(mask, np.uint8)
    Kinv0 = _c(Kinv[0], np.float64)
    if L.dn_estimate(n, _p(size), keep, _p(mask), _p(K), _p(Kinv0), _p(Q), _p(a), METHODS.get(method, method),
                  patch_size, num_depth_planes, iterations, float(np.float32(min_patch_variance)), min_depth,
                  max_depth, _p(w), seed, key, _p(depth), _p(plane), _p(score), _p(nghbr)) != 0:
        raise ValueError("patch size %d: PatchMatch needs a border around every pixel" % patch_size)
    return depth, plane, score, nghbr


def clean(Ks, Rs, ts, depths, same_depth_threshold=0.01, min_consistent_views=2):
    from opensfm_b200 import dense as D

    L = _load()
    depths = [_c(d, np.float32) for d in depths]
    size = _c([(d.shape[1], d.shape[0]) for d in depths], np.int32)
    Kinv, _, _ = D.view_terms(Ks, Rs, ts)
    out = np.zeros(depths[0].shape, np.float32)
    L.dn_clean(len(depths), _p(size), _ptr_array(depths), _p(_c(Ks, np.float64)), _p(Kinv), _p(_c(Rs, np.float64)),
               _p(_c(ts, np.float64)), same_depth_threshold, min_consistent_views, _p(out))
    return out


def prune(Ks, Rs, ts, depths, planes, color0, labels0, same_depth_threshold=0.01):
    from opensfm_b200 import dense as D

    L = _load()
    depths = [_c(d, np.float32) for d in depths]
    planes = [_c(p, np.float32) for p in planes]
    size = _c([(d.shape[1], d.shape[0]) for d in depths], np.int32)
    Kinv, _, _ = D.view_terms(Ks, Rs, ts)
    npx = depths[0].size
    pts, nrm = np.zeros((npx, 3), np.float32), np.zeros((npx, 3), np.float32)
    col, lab = np.zeros((npx, 3), np.uint8), np.zeros(npx, np.uint8)
    c = L.dn_prune(len(depths), _p(size), _ptr_array(depths), _ptr_array(planes), _p(_c(color0, np.uint8)),
                   _p(_c(labels0, np.uint8)), _p(_c(Ks, np.float64)), _p(Kinv), _p(_c(Rs, np.float64)),
                   _p(_c(ts, np.float64)), same_depth_threshold, _p(pts), _p(nrm), _p(col), _p(lab))
    return pts[:c], nrm[:c], col[:c], lab[:c]


def median5(depth):
    L = _load()
    d = _c(depth, np.float32)
    out = np.zeros_like(d)
    L.dn_median5(_p(d), d.shape[1], d.shape[0], _p(out))
    return out


def homography(K1inv, Q, a, K2, plane):
    """PlaneInducedHomographyBaked, as the estimator's score uses it (f32, row-major)."""
    out = np.zeros(9, np.float32)
    _load().dn_homography(_p(_c(K1inv, np.float64)), _p(_c(Q, np.float64)), _p(_c(a, np.float64)),
                          _p(_c(K2, np.float64)), _p(_c(plane, np.float32)), _p(out))
    return out.reshape(3, 3)


def plane_from_depth_normal(x, y, Kinv, depth, normal):
    out = np.zeros(3, np.float32)
    _load().dn_plane_from_depth_normal(x, y, _p(_c(Kinv, np.float64)), depth, _p(_c(normal, np.float32)), _p(out))
    return out


def depth_of_plane(x, y, Kinv, plane):
    return _load().dn_depth_of_plane(x, y, _p(_c(Kinv, np.float64)), _p(_c(plane, np.float32)))


def backproject(x, y, depth, Kinv, R, t):
    out = np.zeros(3)
    _load().dn_backproject(x, y, depth, _p(_c(Kinv, np.float64)), _p(_c(R, np.float64)), _p(_c(t, np.float64)),
                           _p(out))
    return out


def project(X, K, R, t):
    out = np.zeros(3)
    _load().dn_project(_p(_c(X, np.float64)), _p(_c(K, np.float64)), _p(_c(R, np.float64)), _p(_c(t, np.float64)),
                       _p(out))
    return out


def ncc(x, y, w):
    x, y, w = _c(x, np.float32), _c(y, np.float32), _c(w, np.float32)
    return _load().dn_ncc(len(x), _p(x), _p(y), _p(w))


def log(x):
    return _load().dn_log(x)


def exp(x):
    return _load().dn_exp(x)


def normal(pixel, pass_, draw, k0, k1):
    return _load().dn_normal(pixel, pass_, draw, k0, k1)


def philox(c, k):
    out = np.zeros(4, np.uint32)
    _load().dn_philox(*[int(v) for v in c], *[int(v) for v in k], _p(out))
    return out
