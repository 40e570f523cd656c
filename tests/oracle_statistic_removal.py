"""ctypes binding of oracle/statistic_removal_oracle.cc: PCL's StatisticalOutlierRemoval as StatisticRemoval computes it
(product mode: libnabo's neighbours over widened coordinates, exactly rounded sums) and as PCL runs it (literal mode:
neighbours ranked by float d2, serial double sums).  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import numpy as np

import oracle_lib as O

_lib = None

PRODUCT, LITERAL = 0, 1


class Result(NamedTuple):
    out: np.ndarray          # (m, 5) float32 kept records
    inliers: np.ndarray      # (m,) int32
    distances: np.ndarray    # (n,) float32
    stats: tuple             # mean, stddev, threshold, valid


def lib():
    global _lib
    if _lib is None:
        _lib = O.lib()
        _lib.sm_oracle_statistic_removal.restype = C.c_int
        _lib.sm_oracle_statistic_removal.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_int32,
                                                     C.c_void_p, C.POINTER(C.c_int64), C.c_void_p, C.c_void_p,
                                                     C.c_void_p]
    return _lib


def statistic_removal(records, mean_k=30, std_mul=1.0, mode=PRODUCT):
    """records: (n, >= 5) float32 rows -> Result; raises ValueError for rejected arguments, RuntimeError for the
    CHECK case (1..mean_k finite points)."""
    pts = np.ascontiguousarray(np.asarray(records, dtype=np.float32))
    n, cols = pts.shape
    out = np.empty((max(n, 1), 5), np.float32)
    inl = np.empty(max(n, 1), np.int32)
    dist = np.empty(max(n, 1), np.float32)
    stats = np.empty(4, np.float64)
    m = C.c_int64(0)
    rc = lib().sm_oracle_statistic_removal(pts.ctypes.data, n, 4 * cols, int(mean_k), float(std_mul), int(mode),
                                           out.ctypes.data, C.byref(m), inl.ctypes.data, dist.ctypes.data,
                                           stats.ctypes.data)
    if rc == -1:
        raise ValueError("sm_oracle_statistic_removal rejected the arguments")
    if rc == -5:
        raise RuntimeError("CHECK: between 1 and mean_k finite points")
    k = m.value
    return Result(out[:k].copy(), inl[:k].copy(), dist[:n].copy(), tuple(float(v) for v in stats))
