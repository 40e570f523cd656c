"""ctypes binding of oracle/lum_oracle.cc: MultiviewRegistratorLumPcl's LUM alignment on the CPU, as the GPU computes
it (product mode) and as PCL's float arithmetic runs it (literal mode).  The handle mirrors sm_lum_*: the graph lives
on it across AlignAll calls.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O

PRODUCT, LITERAL = 0, 1
TRACE_EDGE = 67   # s, t, finite pairs, 15 sums, D[6], s^2, cinv[36], cinvd[6]

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = O.lib()
        vp, i64 = C.c_void_p, C.c_int64
        _lib.sm_oracle_lum_create.restype = vp
        _lib.sm_oracle_lum_create.argtypes = [C.c_int32]
        _lib.sm_oracle_lum_destroy.restype = None
        _lib.sm_oracle_lum_destroy.argtypes = [vp]
        _lib.sm_oracle_lum_add_cloud.argtypes = [vp, vp, i64, i64, vp]
        _lib.sm_oracle_lum_align_all.argtypes = [vp, vp, i64, C.POINTER(i64)]
        _lib.sm_oracle_lum_poses.argtypes = [vp, vp, i64, C.POINTER(i64)]
        _lib.sm_oracle_lum_correspondences.argtypes = [vp, C.c_int32, C.c_int32, vp, i64, C.POINTER(i64)]
        _lib.sm_oracle_lum_trace.argtypes = [vp, C.c_int32]
        _lib.sm_oracle_lum_trace_get.argtypes = [vp, i64, C.POINTER(C.c_int32), C.POINTER(C.c_int32), vp, vp, vp,
                                                 C.POINTER(C.c_double)]
    return _lib


class Trace:
    """One LUM iteration: the vertex count, per edge (s, t, pairs, sums[15], D[6], ss, cinv[36], cinvd[6]) as float32
    rows, X, the poses after the update and the sum of the pose changes' norms."""

    def __init__(self, n, edges, X, poses, total):
        self.n, self.edges, self.X, self.poses, self.sum = n, edges, X, poses, total


def read_trace(get, h):
    """All recorded iterations through get(h, it, nv, ne, edges, X, poses, sum) (the oracle's or the library's)."""
    nv, ne, s = C.c_int32(0), C.c_int32(0), C.c_double(0)
    assert get(h, -1, C.byref(nv), C.byref(ne), None, None, None, C.byref(s)) == 0
    out = []
    for it in range(ne.value):
        assert get(h, it, C.byref(nv), C.byref(ne), None, None, None, C.byref(s)) == 0
        n, e = nv.value, ne.value
        edges = np.zeros((e, TRACE_EDGE), np.float32)
        X = np.zeros(6 * (n - 1), np.float64)
        poses = np.zeros((n, 6), np.float32)
        assert get(h, it, C.byref(nv), C.byref(ne), edges.ctypes.data, X.ctypes.data, poses.ctypes.data,
                   C.byref(s)) == 0
        out.append(Trace(n, edges, X, poses, s.value))
    return out


class Lum:
    """The oracle's MultiviewRegistratorLumPcl.  AlignAll returns the output records, or raises ValueError where the
    library returns SM_ERR_BAD_ARGUMENT."""

    def __init__(self, mode=PRODUCT):
        self._l = lib()
        self._h = self._l.sm_oracle_lum_create(mode)
        self.cols = 3

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.sm_oracle_lum_destroy(self._h)
            self._h = None

    def AddNewCloud(self, cloud, pose):
        pts = np.ascontiguousarray(np.asarray(cloud, np.float32))
        T = np.ascontiguousarray(np.asarray(pose, np.float32).reshape(4, 4).T)
        if self._l.sm_oracle_lum_add_cloud(self._h, pts.ctypes.data, pts.shape[0], 4 * pts.shape[1],
                                           T.ctypes.data) != 0:
            raise ValueError("sm_oracle_lum_add_cloud rejected the cloud")
        self.cols = pts.shape[1]

    def align_all(self, n_out):
        out = np.zeros((max(n_out, 1), self.cols), np.float32)
        m = C.c_int64(0)
        if self._l.sm_oracle_lum_align_all(self._h, out.ctypes.data, out.shape[0], C.byref(m)) != 0:
            raise ValueError("sm_oracle_lum_align_all rejected the graph")
        return out[:m.value]

    def Poses(self):
        n = C.c_int64(0)
        self._l.sm_oracle_lum_poses(self._h, None, 0, C.byref(n))
        out = np.zeros((n.value, 6), np.float32)
        self._l.sm_oracle_lum_poses(self._h, out.ctypes.data, n.value, C.byref(n))
        return out

    def correspondences(self, j, i):
        n = C.c_int64(0)
        assert self._l.sm_oracle_lum_correspondences(self._h, j, i, None, 0, C.byref(n)) == 0
        out = np.zeros((n.value, 2), np.int32)
        if n.value:
            assert self._l.sm_oracle_lum_correspondences(self._h, j, i, out.ctypes.data, n.value, C.byref(n)) == 0
        return out

    def trace(self, enable=True):
        self._l.sm_oracle_lum_trace(self._h, 1 if enable else 0)

    def traced(self):
        return read_trace(self._l.sm_oracle_lum_trace_get, self._h)
