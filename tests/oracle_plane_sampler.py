"""ctypes binding of oracle/plane_sampler_oracle.cc: the reference's RandomSamplerWithPlaneDetect and PlaneDetector,
with PCL's RANSAC plane fit, restated literally in C++.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import numpy as np

import oracle_lib as O

_lib = None

# one voxel of the trace: int32 status, iterations, best, final_count; float32 coef[4]
TRACE = np.dtype([("status", "<i4"), ("iterations", "<i4"), ("best", "<i4"), ("final_count", "<i4"),
                  ("coef", "<f4", (4,))])
RAW_WORDS = 3 * 1000 * 51


class Result(NamedTuple):
    keep: np.ndarray         # (n,) bool
    plane: np.ndarray        # ascending int32, the sorted output of Detect
    traces: np.ndarray       # TRACE per voxel in map order (empty when Detect does not run)

    @property
    def inliers(self):
        return np.flatnonzero(self.keep).astype(np.int32)

    @property
    def outliers(self):
        return np.flatnonzero(~self.keep).astype(np.int32)


def lib():
    global _lib
    if _lib is None:
        _lib = O.lib()
        _lib.sm_oracle_plane_sampler.restype = C.c_int
        _lib.sm_oracle_plane_sampler.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_float, C.c_float, C.c_uint64,
                                                 C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p,
                                                 C.POINTER(C.c_int64)]
        _lib.sm_oracle_plane_sampler_raw_stream.restype = C.c_int
        _lib.sm_oracle_plane_sampler_raw_stream.argtypes = [C.c_void_p, C.c_int64]
        _lib.sm_oracle_plane_sampler_keep_loop.restype = C.c_int
        _lib.sm_oracle_plane_sampler_keep_loop.argtypes = [C.c_float, C.c_int64, C.c_void_p]
        _lib.sm_oracle_plane_sampler_piece.restype = C.c_int
        _lib.sm_oracle_plane_sampler_piece.argtypes = [C.c_int32, C.c_void_p, C.c_void_p]
    return _lib


def raw_stream(n=RAW_WORDS):
    out = np.empty(n, np.uint32)
    assert lib().sm_oracle_plane_sampler_raw_stream(out.ctypes.data, n) == 0
    return out


def keep_loop(rate, k):
    """keep[j] = the loop's decision for non-plane point j + 1"""
    out = np.empty(max(k, 1), np.uint8)
    assert lib().sm_oracle_plane_sampler_keep_loop(float(rate), k, out.ctypes.data) == 0
    return out[:k].astype(bool)


def piece(op, values):
    inp = np.ascontiguousarray(values, np.float32)
    out = np.zeros(4, np.float32)
    assert lib().sm_oracle_plane_sampler_piece(op, inp.ctypes.data, out.ctypes.data) == 0
    return out


def plane_sampler(records, rate=1.0, leaf_size=0.8, min_point_num_in_voxel=10):
    """records: (n, >= 3) float32 rows; rate, leaf_size and min_point_num_in_voxel as after the setters -> Result"""
    pts = np.ascontiguousarray(np.asarray(records, dtype=np.float32))
    n, cols = pts.shape
    keep = np.zeros(max(n, 1), np.uint8)
    plane = np.empty(max(n, 1), np.int32)
    traces = np.zeros(max(n, 1), TRACE)
    npl, nv = C.c_int64(0), C.c_int64(0)
    rc = lib().sm_oracle_plane_sampler(pts.ctypes.data, n, 4 * cols, float(rate), float(leaf_size),
                                       int(min_point_num_in_voxel) % (1 << 64), keep.ctypes.data, plane.ctypes.data,
                                       C.byref(npl), traces.ctypes.data, C.byref(nv))
    if rc != 0:
        raise ValueError("sm_oracle_plane_sampler rejected the arguments")
    return Result(keep[:n].astype(bool), plane[:npl.value].copy(), traces[:nv.value].copy())


def clamp_rate(rate):
    """SetSamplingRate on a float"""
    r = np.float32(rate)
    if float(r) > 1.0:
        return np.float32(1.0)
    if float(r) < 1e-6:
        return np.float32(1e-6)
    return r
