"""ctypes binding of oracle/unordered_map_oracle.cc: VoxelGrid's std::unordered_map from this toolchain's libstdc++
itself, its literal iteration order (as first-member indices), bucket_count() after every distinct insert and the
reference's voxel hash; and the library's own schedule and hash hooks.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O


def _fn(name, restype, argtypes):
    f = getattr(O.lib(), name)
    f.restype, f.argtypes = restype, argtypes
    return f


def order_points(points, voxel_size):
    """the input index of each voxel's first member, in the container's iteration order; `points` (N, >= 3)
    float32 records, every one inserted (pass finite points only)"""
    p = np.ascontiguousarray(np.asarray(points, np.float32))
    out = np.zeros(len(p), np.int64)
    f = _fn("sm_oracle_voxel_unordered_order", C.c_int64, [C.c_void_p, C.c_int64, C.c_int64, C.c_float, C.c_void_p])
    m = f(p.ctypes.data, len(p), p.shape[1] if len(p) else 5, voxel_size, out.ctypes.data)
    assert m >= 0
    return out[:m]


def order_keys(keys):
    """the same over int32 keys (N, 3): the first index of every distinct key in iteration order"""
    k = np.ascontiguousarray(np.asarray(keys, np.int32).reshape(-1, 3))
    out = np.zeros(len(k), np.int64)
    f = _fn("sm_oracle_unordered_order_keys", C.c_int64, [C.c_void_p, C.c_int64, C.c_void_p])
    m = f(k.ctypes.data, len(k), out.ctypes.data)
    return out[:m]


def bucket_counts(m):
    """bucket_count() after each of m distinct inserts into a default-constructed map"""
    out = np.zeros(m, np.uint64)
    assert _fn("sm_oracle_unordered_bucket_counts", C.c_int, [C.c_int64, C.c_void_p])(m, out.ctypes.data) == 0
    return out


def key_hash(keys):
    """Key3Hash (common/eigen_hash.h) of int32 keys (N, 3)"""
    k = np.ascontiguousarray(np.asarray(keys, np.int32).reshape(-1, 3))
    out = np.zeros(len(k), np.uint64)
    assert _fn("sm_oracle_key3_hash", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p])(k.ctypes.data, len(k),
                                                                                    out.ctypes.data) == 0
    return out


# ---- the library's host hooks -----------------------------------------------------------------------------------------
def library_bucket_counts(m):
    from staticmapping_b200 import _lib
    out = np.zeros(m, np.uint64)
    assert _lib.lib().sm_debug_voxel_bucket_counts_host(m, out.ctypes.data) == 0
    return out


def library_hash(keys):
    from staticmapping_b200 import _lib
    k = np.ascontiguousarray(np.asarray(keys, np.int32).reshape(-1, 3))
    out = np.zeros(len(k), np.uint64)
    assert _lib.lib().sm_debug_voxel_hash_host(k.ctypes.data, len(k), out.ctypes.data) == 0
    return out
