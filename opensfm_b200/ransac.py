"""What the batched RANSAC engines share on the host (rotation_ransac, resection, relative_pose): the handle and its
test hooks, the check of a batch's row layout, and the packing of per-pair bearing arrays.

A batch is a table (or two) and, per row, the entry it names in each; problem p owns rows [start[p], start[p + 1]).
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence

import numpy as np

from . import _lib
from ._lib import ptr


class Engine:
    """An osfm_<kind> handle ("rotransac", "resect" or "relpose"): one stream, its workspaces and the sample stream
    kept on the device; a new handle, or `handle` when given."""

    kind = ""

    def __init__(self, device: int = 0, handle: Optional[_lib.Handle] = None):
        self.handle = handle if handle is not None else _lib.Handle(self.kind, device)
        self.h, self.L, self.device = self.handle.h, self.handle.L, self.handle.device
        self._trace_cap = 0
        self._num_problems = 0

    def _call(self, name: str, *args) -> None:
        _lib.check(getattr(self.L, "osfm_%s_%s" % (self.kind, name))(self.h, *args))

    def set_stream_prefix(self, length: int) -> None:
        """How many generator outputs the device keeps (a test hook: problems that use them all continue from the
        saved generator state)."""
        self._call("set_stream_prefix", int(length))

    def set_trace(self, capacity: int) -> None:
        """Record up to `capacity` drawn sample indices per problem in the following runs (0: off)."""
        self._call("set_trace", int(capacity))
        self._trace_cap = int(capacity)

    def trace(self):
        """(drawn indices per problem as a list of arrays, how many were drawn, generator outputs consumed per
        problem) of the last run."""
        P, cap = self._num_problems, self._trace_cap
        count = np.zeros(P, dtype=np.int32)
        used = np.zeros(P, dtype=np.int64)
        idx = np.zeros(P * cap, dtype=np.int32)
        self._call("get_trace", ptr(count), ptr(used), ptr(idx))
        idx = idx.reshape(P, cap)
        return [idx[p, :min(int(count[p]), cap)] for p in range(P)], count, used

    def _device_ms(self) -> float:
        """Device time of the last run."""
        ms = ctypes.c_float(0)
        self._call("last_device_ms", ctypes.byref(ms))
        return float(ms.value)


def batch_rows(start: np.ndarray, rows_a: np.ndarray, rows_b: np.ndarray,
               names: Sequence[str] = ("pair_start", "row_a", "row_b")):
    """(start, rows_a, rows_b) as contiguous int64 arrays, checked to describe the same rows; `names` name them in
    the error."""
    start = np.ascontiguousarray(start, dtype=np.int64)
    rows_a = np.ascontiguousarray(rows_a, dtype=np.int64)
    rows_b = np.ascontiguousarray(rows_b, dtype=np.int64)
    if len(start) < 1 or start[-1] != len(rows_a) or len(rows_a) != len(rows_b):
        raise ValueError("%s must end at the number of rows, and %s / %s must match in length" % tuple(names))
    return start, rows_a, rows_b


def pack_pairs(b1_list: Sequence[np.ndarray], b2_list: Sequence[np.ndarray]):
    """(bearing table, pair_start, row_a, row_b) of per-pair arrays: the first images' rows, then the second's."""
    if len(b1_list) != len(b2_list) or any(len(a) != len(b) for a, b in zip(b1_list, b2_list)):
        raise ValueError("every pair needs as many second bearings as first bearings")
    n = np.array([len(b) for b in b1_list], dtype=np.int64)
    pair_start = np.zeros(len(n) + 1, dtype=np.int64)
    np.cumsum(n, out=pair_start[1:])
    R = int(pair_start[-1])
    if R == 0:
        return np.zeros((0, 3)), pair_start, np.zeros(0, np.int64), np.zeros(0, np.int64)
    bearings = np.concatenate([np.asarray(b, np.float64).reshape(-1, 3) for b in b1_list] +
                              [np.asarray(b, np.float64).reshape(-1, 3) for b in b2_list])
    rows = np.arange(R, dtype=np.int64)
    return bearings, pair_start, rows, rows + R
