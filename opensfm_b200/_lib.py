"""ctypes binding of the C ABI declared in include/opensfm_b200.h.

There is no CPU fallback: if the shared library is missing or no CUDA device is
present, calls raise.  (The library is built in-tree by `__graft_entry__.build()`.)
"""
from __future__ import annotations

import contextlib
import ctypes
import os
import threading
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_uint, c_uint8, c_void_p
from typing import Dict, Iterator, List, Optional, Tuple

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libopensfm_b200.so")

OSFM_OK = 0
PROJECTION_TYPES = dict(PERSPECTIVE=0, BROWN=1, FISHEYE=2, FISHEYE_OPENCV=3, FISHEYE62=4, FISHEYE624=5,
                        SPHERICAL=6, DUAL=7, RADIAL=8, SIMPLE_RADIAL=9)
LOSS_IDS = {"TrivialLoss": 0, "HuberLoss": 1, "SoftLOneLoss": 2, "CauchyLoss": 3, "ArctanLoss": 4}
LOSS_TUKEY = 5  # side terms only (common position)
SIDE_TYPES = dict(UP_VECTOR=0, PAN=1, TILT=2, ROLL=3, RELATIVE_MOTION=4, RELATIVE_ROTATION=5, COMMON_POSITION=6,
                  LINEAR_MOTION=7, TRANSLATION_PRIOR=8, PARAMETER_BARRIER=9, STD_DEVIATION=10, POSITION_PRIOR=11)
SB_CAM, SB_INST, SB_RIGCAM, SB_EXT = 0, 1, 2, 3


class SideTerm(ctypes.Structure):
    """osfm_side_term (include/opensfm_b200.h)."""
    _fields_ = [("type", c_int32), ("nres", c_int32), ("nblocks", c_int32), ("kind", c_int32 * 6), ("idx", c_int32 * 6),
                ("loss", c_int32), ("loss_a", c_double), ("cofs", c_int32), ("aux", c_int32 * 4)]


class BASummary(ctypes.Structure):
    _fields_ = [
        ("iterations", c_int), ("successful_steps", c_int), ("linear_solves", c_int), ("pcg_iterations", c_int),
        ("termination", c_int), ("initial_cost", c_double), ("final_cost", c_double), ("time_run_s", c_double),
        ("time_device_ms", c_double), ("time_linearize_ms", c_double), ("linearize_launches", c_int64),
        ("time_schur_ms", c_double), ("schur_launches", c_int64), ("time_pcg_ms", c_double),
        ("time_backsub_ms", c_double), ("num_observations_local", c_int64), ("reduced_dim", c_int),
        ("reduced_blocks", c_int), ("reduced_nnz", c_int64), ("jac_planes", c_int), ("kernel_launches", c_int64), ("message", ctypes.c_char * 128),
        ("device_loop", c_int),
    ]


class BACapture(ctypes.Structure):
    """osfm_ba_capture (include/opensfm_b200.h)."""
    _fields_ = [("iteration", c_int), ("nc", c_int), ("n", c_int), ("wc", c_int), ("nres", c_int), ("radius", c_double),
                ("nseg", c_int), ("p_fast", c_int), ("p_slow", c_int), ("schur_kernel", c_int), ("sp_nchunks", c_int),
                ("pcg_kernel", c_int), ("pcg_rescued", c_int), ("pcg_iterations", c_int), ("pcg_rr", c_double)]


SCHUR_KERNELS = {0: "none", 1: "pipe", 2: "mma", 3: "simt_segment"}
PCG_KERNELS = {1: "pipelined_deflated", 2: "pipelined", 3: "classic_resident", 4: "classic_streamed"}
COVARIANCE_STATUS = {0: "ok", 1: "solver_failure", 2: "point_rank_deficient", 3: "camera_rank_deficient",
                     4: "non_finite"}
# OSFM_BA_FALLBACK_* bits of osfm_ba_set_fallbacks by name: kernel paths a solve can be made to take (tests, A/B runs)
BA_FALLBACKS = {"per_point_schur": 1, "simt_segment_schur": 2, "cta_per_segment_schur": 4, "generic_linearize": 8,
                "classic_pcg": 16, "streamed_pcg": 32, "undeflated_pcg": 64, "host_loop": 128}

ALLREDUCE_FN = ctypes.CFUNCTYPE(c_int, c_void_p, c_int64, c_void_p, c_void_p)

# name -> (restype, argtypes); every symbol include/opensfm_b200.h declares
SIGNATURES = {
    "osfm_last_error": (c_char_p, []),
    "osfm_version": (c_int, []),
    "osfm_kernel_launch_count": (c_int64, []),
    "osfm_matcher_create": (c_int, [c_int, POINTER(c_void_p)]),
    "osfm_matcher_destroy": (c_int, [c_void_p]),
    "osfm_bf_match_f32": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_double, c_void_p, c_int, c_void_p]),
    "osfm_bf_match_u8": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_double, c_void_p, c_int, c_void_p]),
    "osfm_matcher_add_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(c_int)]),
    "osfm_matcher_add_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(c_int)]),
    "osfm_matcher_add_batch_f32": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "osfm_matcher_add_batch_u8": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "osfm_matcher_add_u8_l2": (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(c_int)]),
    "osfm_matcher_add_batch_u8_l2": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "osfm_matcher_remove": (c_int, [c_void_p, c_int]),
    "osfm_matcher_clear": (c_int, [c_void_p]),
    "osfm_matcher_match_pairs_async": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_double, c_int]),
    "osfm_matcher_set_bearings": (c_int, [c_void_p, c_int, c_void_p]),
    "osfm_matcher_match_pairs_guided_async": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_double, c_double,
                                                       c_int]),
    "osfm_matcher_get_epipolar_masks": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "osfm_matcher_sync": (c_int, [c_void_p]),
    "osfm_matcher_fetch": (c_int, [c_void_p, c_void_p, c_int64]),
    "osfm_matcher_fetch_pairs": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, POINTER(c_int64)]),
    "osfm_matcher_last_device_ms": (c_int, [c_void_p, POINTER(c_float), POINTER(c_float)]),
    "osfm_matcher_set_kernel": (c_int, [c_void_p, c_int]),
    "osfm_matcher_last_kernel": (c_int, [c_void_p]),
    "osfm_matcher_device_bytes": (c_int, [c_void_p, POINTER(c_int64), POINTER(c_int64)]),
    "osfm_match_words": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_float,
                                  c_int, c_void_p]),
    "osfm_vlad_distances": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "osfm_matcher_vlad_compute": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "osfm_matcher_vlad_get": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "osfm_matcher_vlad_select": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                         c_void_p, c_void_p]),
    "osfm_matcher_bow_words": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                       c_void_p]),
    "osfm_bow_map_to_words": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "osfm_matcher_bow_histograms": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "osfm_matcher_bow_get": (c_int, [c_void_p, c_int, c_void_p]),
    "osfm_bow_histogram": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "osfm_matcher_bow_select": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                        c_void_p, c_void_p]),
    "osfm_bow_distances": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "osfm_ba_create": (c_int, [c_int, POINTER(c_void_p)]),
    "osfm_ba_destroy": (c_int, [c_void_p]),
    "osfm_camera_num_params": (c_int, [c_int]),
    "osfm_ba_set_cameras": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_ba_set_rig_instances": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_ba_set_rig_cameras": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "osfm_ba_set_shots": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_ba_set_points": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "osfm_ba_set_observations": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_ba_set_observations_async": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_ba_set_rig_camera_priors": (c_int, [c_void_p, c_void_p, c_void_p]),
    "osfm_ba_set_point_priors": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_ba_set_ext_blocks": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_ba_get_ext_blocks": (c_int, [c_void_p, c_void_p]),
    "osfm_ba_set_side_terms": (c_int, [c_void_p, c_int, c_void_p, c_int64, c_void_p]),
    "osfm_ba_set_options": (c_int, [c_void_p, c_int, c_double, c_int, c_char_p, c_int]),
    "osfm_ba_set_distributed": (c_int, [c_void_p, c_int, c_int, ALLREDUCE_FN, c_void_p]),
    "osfm_nccl_unique_id": (c_int, [c_void_p]),
    "osfm_ba_set_nccl": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "osfm_ba_set_stream": (c_int, [c_void_p, c_void_p]),
    "osfm_ba_run": (c_int, [c_void_p]),
    "osfm_ba_get_summary": (c_int, [c_void_p, POINTER(BASummary)]),
    "osfm_ba_get_cameras": (c_int, [c_void_p, c_void_p]),
    "osfm_ba_get_rig_instances": (c_int, [c_void_p, c_void_p]),
    "osfm_ba_get_rig_cameras": (c_int, [c_void_p, c_void_p]),
    "osfm_ba_get_points": (c_int, [c_void_p, c_void_p]),
    "osfm_ba_get_reprojection_errors": (c_int, [c_void_p, c_void_p]),
    "osfm_ba_eval_observation": (c_int, [c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                         c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int)]),
    "osfm_ba_capture_linear_system": (c_int, [c_void_p, c_int]),
    "osfm_ba_set_fallbacks": (c_int, [c_void_p, c_uint]),
    "osfm_ba_get_captured_system": (c_int, [c_void_p, POINTER(BACapture), c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_void_p]),
    "osfm_ba_get_captured_parameters": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_ba_get_captured_side_rows": (c_int, [c_void_p, c_void_p, c_void_p]),
    "osfm_ba_set_compute_covariances": (c_int, [c_void_p, c_int]),
    "osfm_ba_get_covariances": (c_int, [c_void_p, POINTER(c_int), POINTER(c_int), c_void_p]),
    "osfm_ba_get_covariance_timing": (c_int, [c_void_p, POINTER(c_double), POINTER(c_double)]),
    "osfm_tracks_create": (c_int, [c_int, POINTER(c_void_p)]),
    "osfm_tracks_destroy": (c_int, [c_void_p]),
    "osfm_tracks_build": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_int, POINTER(c_int64), POINTER(c_int64)]),
    "osfm_tracks_get": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_tracks_common": (c_int, [c_void_p, POINTER(c_int64), POINTER(c_int64)]),
    "osfm_tracks_get_common": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_tracks_last_device_ms": (c_int, [c_void_p, POINTER(c_float), POINTER(c_float)]),
    "osfm_tracks_triangulate": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_int64,
                                        c_void_p, c_double, c_double, c_double, c_int, c_void_p, c_void_p]),
    "osfm_tracks_last_triangulate_ms": (c_int, [c_void_p, POINTER(c_float)]),
    "osfm_rotransac_create": (c_int, [c_int, POINTER(c_void_p)]),
    "osfm_rotransac_destroy": (c_int, [c_void_p]),
    "osfm_rotransac_run": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_double, c_int,
                                   c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_rotransac_last_device_ms": (c_int, [c_void_p, POINTER(c_float)]),
    "osfm_rotransac_set_stream_prefix": (c_int, [c_void_p, c_int64]),
    "osfm_rotransac_set_trace": (c_int, [c_void_p, c_int]),
    "osfm_rotransac_get_trace": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_resect_create": (c_int, [c_int, POINTER(c_void_p)]),
    "osfm_resect_destroy": (c_int, [c_void_p]),
    "osfm_resect_run": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                                c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_resect_last_device_ms": (c_int, [c_void_p, POINTER(c_float)]),
    "osfm_resect_set_stream_prefix": (c_int, [c_void_p, c_int64]),
    "osfm_resect_set_trace": (c_int, [c_void_p, c_int]),
    "osfm_resect_get_trace": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_relpose_create": (c_int, [c_int, POINTER(c_void_p)]),
    "osfm_relpose_destroy": (c_int, [c_void_p]),
    "osfm_relpose_run": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_double, c_int,
                                 c_void_p, c_void_p, c_void_p]),
    "osfm_relpose_two_view": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_double,
                                      c_int, c_int, c_int, c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "osfm_relpose_robust_match": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                                          c_double, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_relpose_last_device_ms": (c_int, [c_void_p, POINTER(c_float)]),
    "osfm_relpose_last_stage_ms": (c_int, [c_void_p, POINTER(c_float), POINTER(c_float)]),
    "osfm_relpose_set_stream_prefix": (c_int, [c_void_p, c_int64]),
    "osfm_relpose_set_trace": (c_int, [c_void_p, c_int]),
    "osfm_relpose_get_trace": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_dense_create": (c_int, [c_int, POINTER(c_void_p)]),
    "osfm_dense_destroy": (c_int, [c_void_p]),
    "osfm_dense_set_views": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p]),
    "osfm_dense_set_maps": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "osfm_dense_estimate": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_uint, c_double, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_dense_clean": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_float, c_int, c_void_p]),
    "osfm_dense_prune": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_float, c_void_p]),
    "osfm_dense_get_pruned": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_dense_last_device_ms": (c_int, [c_void_p, POINTER(c_float), POINTER(c_float), POINTER(c_float)]),
    "osfm_undistort_create": (c_int, [c_int, POINTER(c_void_p)]),
    "osfm_undistort_destroy": (c_int, [c_void_p]),
    "osfm_undistort_camera_maps": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "osfm_undistort_face_maps": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "osfm_undistort_remap": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                     c_int, c_int, c_void_p]),
    "osfm_undistort_run": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "osfm_undistort_last_device_ms": (c_int, [c_void_p, POINTER(c_float), POINTER(c_float), POINTER(c_float)]),
}

_lib = None


def load() -> ctypes.CDLL:
    """Load the CUDA library.  Raises if it has not been built (no silent fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "opensfm_b200: %s is missing; run `python -c 'import __graft_entry__ as g; g.build()'`. "
                "There is no CPU fallback." % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(code: int) -> None:
    if code != OSFM_OK:
        msg = load().osfm_last_error().decode("utf-8", "replace")
        if code == 2:
            raise ValueError(msg)
        raise RuntimeError(msg)


def ptr(a: Optional[np.ndarray]) -> Optional[ctypes.c_void_p]:
    """The data pointer of a C-contiguous array, or None for None."""
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


class Handle:
    """One engine object of the C ABI, `osfm_<kind>_create(device)` .. `osfm_<kind>_destroy`, with kind one of "ba",
    "matcher", "tracks", "rotransac", "resect", "relpose", "dense" and "undistort".  It keeps its stream and device workspaces between calls.  The
    library serialises calls on one handle, so callers that should not wait for one another use handles of their own."""

    def __init__(self, kind: str, device: int = 0):
        self.kind, self.device, self.L = kind, int(device), load()
        self.h = ctypes.c_void_p()
        check(getattr(self.L, "osfm_%s_create" % kind)(self.device, ctypes.byref(self.h)))

    def __del__(self):
        try:
            getattr(self.L, "osfm_%s_destroy" % self.kind)(self.h)
        except Exception:
            pass


# Released handles by (kind, device).  A caller that asks again gets the handle it released last, so one thread
# calling repeatedly reuses the same stream, HBM workspaces and, for bundle adjustment, NCCL communicator.
_pool_lock = threading.Lock()
_pool: Dict[Tuple[str, int], List[Handle]] = {}


def acquire(kind: str, device: int = 0) -> Handle:
    """A handle of `kind` on `device` that is the caller's alone until it calls release()."""
    with _pool_lock:
        free = _pool.get((kind, int(device)))
        if free:
            return free.pop()
    return Handle(kind, device)


def release(handle: Handle) -> None:
    with _pool_lock:
        _pool.setdefault((handle.kind, handle.device), []).append(handle)


@contextlib.contextmanager
def pooled(kind: str, device: int = 0) -> Iterator[Handle]:
    """acquire() for the duration of a `with` block, released however the block ends."""
    h = acquire(kind, device)
    try:
        yield h
    finally:
        release(h)
