"""ctypes binding of oracle/pm_surface_normals_oracle.cc: libpointmatcher's SamplingSurfaceNormalDataPointsFilter
(knn 7) with its eigenvector leaf, and the IcpUsingPointMatcher stand-in's chain (oracle_lib.icp_pm_equivalent) with
either reference filter of sm_set_pm_surface_normals, composed from libsm_oracle.so's pieces.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O


def pm_surface_normal_leaf(members_f32):
    """The eigenvector leaf on 1..7 float members in member order -> (kept, mean (3,) f32, covariance (3,3) f32,
    normal (3,) f32 or None when dropped)."""
    m = O._fcloud(members_f32)
    mean = np.zeros(3, np.float32); cov = np.zeros(9, np.float32); nrm = np.zeros(3, np.float32)
    f = O.lib().sm_oracle_pm_surface_normal_leaf
    f.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    r = f(m.ctypes.data, m.shape[0], mean.ctypes.data, cov.ctypes.data, nrm.ctypes.data)
    assert r >= 0
    return bool(r), mean, cov.reshape(3, 3), (nrm if r else None)


def pm_surface_normals(points_f32):
    """The whole filter with the eigenvector leaf -> (means (M,3) f32, normals (M,3) f32, smallest member index (M,)
    int64), in ascending order of that index."""
    p = O._fcloud(points_f32)
    n = p.shape[0]
    means = np.zeros((n, 3), np.float32); nrm = np.zeros((n, 3), np.float32); idx = np.zeros(n, np.int64)
    f = O.lib().sm_oracle_pm_surface_normals
    f.restype = C.c_int64
    f.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    m = f(p.ctypes.data, n, means.ctypes.data, nrm.ctypes.data, idx.ctypes.data)
    return means[:m].copy(), nrm[:m].copy(), idx[:m].copy()


def pm_reference_filter(target_f32, normals="least_squares"):
    """The type-1 reference filter in either mode of sm_set_pm_surface_normals -> (points, normals) as double (M,3):
    "least_squares" = CalculateNormals on the widened cloud, "eigenvector" = pm_surface_normals widened."""
    tgt = np.asarray(target_f32, dtype=np.float32)
    if normals == "least_squares":
        return O.calculate_normals(tgt.astype(np.float64))
    if normals == "eigenvector":
        tp, tn, _ = pm_surface_normals(tgt)
        return tp.astype(np.float64), tn.astype(np.float64)
    raise ValueError(normals)


def icp_pm_equivalent(source_f32, target_f32, guess=None, prob=0.9, seed=1, max_iteration=150,
                      accept_min_score=0.6, normals="least_squares"):
    """oracle_lib.icp_pm_equivalent (the stand-in's chain: reference filter, hash subsample of the reading,
    IcpFast::Align capped at 150 iterations, the score pass, Align() false below 0.6) with the reference filter of
    `normals`; "least_squares" gives oracle_lib's result."""
    src = np.asarray(source_f32, dtype=np.float32)
    tgt = np.asarray(target_f32, dtype=np.float32)
    tp, tn = pm_reference_filter(tgt, normals)
    keep = O.pm_keep_mask(src.shape[0], prob, seed)
    o = O.icp_fast_align(src[keep].astype(np.float64), tp, tn, guess, max_iteration=max_iteration)
    o["icp_fast_score"] = o["score"]
    o["n_source"] = int(keep.sum())
    o["n_target"] = int(tp.shape[0])
    _, d2 = O.knn1(tgt.astype(np.float64), O.pm_moved(src, o["result"]), epsilon=3.16)
    v, _, kept = O.pm_score_trim(d2)
    if kept:
        o["score"] = float(np.exp(-(np.sqrt(v[:kept]).sum() / kept)))
        o["score_kept"] = kept
    o["ok"] = o["score"] >= float(np.float32(accept_min_score))
    return o
