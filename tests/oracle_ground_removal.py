"""ctypes binding of oracle/ground_removal_oracle.cc: the reference's GroundRemoval (v1) restated literally in C++ with
its std::map.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import numpy as np

import oracle_lib as O

_lib = None


class Result(NamedTuple):
    out: np.ndarray          # (m, 5) float32 emitted records, in the map's order
    index: np.ndarray        # (m,) int32 their input indices
    inliers: np.ndarray      # ascending int32
    outliers: np.ndarray     # ascending int32


def lib():
    global _lib
    if _lib is None:
        _lib = O.lib()
        _lib.sm_oracle_ground_removal.restype = C.c_int
        _lib.sm_oracle_ground_removal.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_float,
                                                  C.c_void_p, C.POINTER(C.c_int64), C.c_void_p, C.c_void_p,
                                                  C.POINTER(C.c_int64), C.c_void_p, C.POINTER(C.c_int64)]
    return _lib


def ground_removal(records, min_point_num_in_voxel=10, leaf_size=0.8, height_threshold=0.15):
    """records: (n, >= 5) float32 rows -> Result"""
    pts = np.ascontiguousarray(np.asarray(records, dtype=np.float32))
    n, cols = pts.shape
    out = np.empty((max(n, 1), 5), np.float32)
    index, inl, outl = (np.empty(max(n, 1), np.int32) for _ in range(3))
    m, ni, no = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    rc = lib().sm_oracle_ground_removal(pts.ctypes.data, n, 4 * cols, int(min_point_num_in_voxel),
                                        float(leaf_size), float(height_threshold), out.ctypes.data, C.byref(m),
                                        index.ctypes.data, inl.ctypes.data, C.byref(ni), outl.ctypes.data,
                                        C.byref(no))
    if rc != 0:
        raise ValueError("sm_oracle_ground_removal rejected the arguments")
    return Result(out[:m.value].copy(), index[:m.value].copy(), inl[:ni.value].copy(), outl[:no.value].copy())
