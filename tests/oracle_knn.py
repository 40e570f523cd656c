"""ctypes binding of tests/cpp/knn_oracle.cc: libnabo's k-NN (KDTREE_LINEAR_HEAP) for general k, epsilon, maxRadius
and option flags on the tree of the oracle's Knn1.  TEST INFRASTRUCTURE.  The library is compiled on first use into a
per-user temporary directory (keyed by the source's hash), so a read-only tree works."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "tests", "cpp", "knn_oracle.cc")
_lib = None

ALLOW_SELF_MATCH = 1
SORT_RESULTS = 2


def lib():
    global _lib
    if _lib is None:
        with open(_SRC, "rb") as f:
            h = hashlib.sha256(f.read()).hexdigest()[:16]
        out_dir = os.path.join(tempfile.gettempdir(), f"sm_knn_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        so = os.path.join(out_dir, f"libsm_knn_oracle_{h}.so")
        if not os.path.exists(so):
            cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
            tmp = so + f".{os.getpid()}.tmp"
            # the flags of oracle/Makefile: no FMA contraction, so the arithmetic is the written one
            subprocess.check_call([cxx, "-O2", "-fopenmp", "-fPIC", "-std=c++17", "-ffp-contract=off",
                                   "-shared", _SRC, "-o", tmp])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
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
