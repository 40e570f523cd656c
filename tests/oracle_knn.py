"""ctypes binding of oracle/knn_oracle.cc: libnabo's k-NN (KDTREE_LINEAR_HEAP) for general k, epsilon, maxRadius
and option flags on the tree of the oracle's Knn1.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O

_lib = None

ALLOW_SELF_MATCH = 1
SORT_RESULTS = 2


def lib():
    global _lib
    if _lib is None:
        _lib = O.lib()
        _lib.sm_oracle_knn.restype = C.c_int
        _lib.sm_oracle_knn.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_double,
                                       C.c_double, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
    return _lib


def knn(target, query, k, epsilon=0.0, max_radius=float("inf"), flags=ALLOW_SELF_MATCH, bucket_size=8):
    """-> (ids int32 (n_query, k), d2 float64 (n_query, k)); raises ValueError where the call is rejected."""
    t = np.ascontiguousarray(np.asarray(target, dtype=np.float64).reshape(-1, 3))
    q = np.ascontiguousarray(np.asarray(query, dtype=np.float64).reshape(-1, 3))
    ids = np.empty((q.shape[0], max(int(k), 1)), dtype=np.int32)
    d2 = np.empty((q.shape[0], max(int(k), 1)), dtype=np.float64)
    rc = lib().sm_oracle_knn(t.ctypes.data, t.shape[0], q.ctypes.data, q.shape[0], int(k), float(epsilon),
                             float(max_radius), int(flags), int(bucket_size), ids.ctypes.data, d2.ctypes.data)
    if rc != 0:
        raise ValueError(f"sm_oracle_knn rejected the call ({rc})")
    return ids, d2
