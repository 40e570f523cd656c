"""ctypes binding of oracle/nth_element_oracle.cc: std::nth_element's own permutations, BuildNormals' index array in
the literal order, and keys that exhaust introselect's depth limit.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O


def _fn(name, argtypes):
    f = getattr(O.lib(), name)
    f.restype, f.argtypes = C.c_int, argtypes
    return f


def nth_element_perm(keys, nth):
    """the index array std::nth_element(idx, idx + nth, idx + n) leaves from iota, comparing keys[a] < keys[b]"""
    k = np.ascontiguousarray(keys, np.float64)
    out = np.zeros(len(k), np.int32)
    f = _fn("sm_oracle_nth_element_perm", [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p])
    assert f(k.ctypes.data, len(k), nth, out.ctypes.data) == 0
    return out


def normals_perm(points):
    """BuildNormals' index array after the whole recursion, every node split by std::nth_element"""
    p = np.ascontiguousarray(np.asarray(points, np.float64))
    out = np.zeros(len(p), np.int32)
    f = _fn("sm_oracle_normals_nth_perm", [C.c_void_p, C.c_int64, C.c_void_p])
    assert f(p.ctypes.data, len(p), out.ctypes.data) == 0
    return out


def adversary(n, nth):
    """keys of n items on which std::nth_element(nth) meets McIlroy's adversary's answers, so it runs to its depth
    limit on large enough n"""
    out = np.zeros(n, np.float64)
    f = _fn("sm_oracle_nth_element_adversary", [C.c_int64, C.c_int64, C.c_void_p])
    assert f(n, nth, out.ctypes.data) == 0
    return out
