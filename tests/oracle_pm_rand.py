"""ctypes binding of oracle/pm_rand_oracle.cc: glibc's rand() stream taken from glibc's own random_r on a private TYPE_3
state, libpointmatcher's RandomSamplingDataPointsFilter drawn from it, and the IcpUsingPointMatcher stand-in's chain
(oracle_lib.icp_pm_equivalent) with that reading filter, composed from libsm_oracle.so's pieces.  TEST
INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O


def glibc_rand(seed, position, count):
    """Draws position .. position + count - 1 of glibc's rand() stream after srand(seed) -> int64 array."""
    out = np.zeros(count, np.int32)
    f = O.lib().sm_oracle_glibc_rand
    f.argtypes = [C.c_uint32, C.c_int64, C.c_int64, C.c_void_p]
    assert f(seed & 0xFFFFFFFF, position, count, out.ctypes.data) == 0
    return out.astype(np.int64)


def pm_rand_mask(n, prob=0.9, seed=1, position=0):
    """RandomSamplingDataPointsFilter over n points with glibc's rand() stream at `position` after srand(seed): point i
    is kept iff (float)rand() / (float)RAND_MAX < prob."""
    keep = np.zeros(n, np.uint8)
    f = O.lib().sm_oracle_pm_rand_mask
    f.restype = C.c_int64
    f.argtypes = [C.c_uint32, C.c_int64, C.c_float, C.c_int64, C.c_void_p]
    assert f(seed & 0xFFFFFFFF, position, prob, n, keep.ctypes.data) >= 0
    return keep.astype(bool)


def icp_pm_equivalent(source_f32, target_f32, guess=None, prob=0.9, seed=1, max_iteration=150,
                      accept_min_score=0.6, position=0):
    """oracle_lib.icp_pm_equivalent (the stand-in's chain: CalculateNormals on the target, the reading's subsample,
    IcpFast::Align capped at 150 iterations, the score pass, Align() false below 0.6) with the reading subsampled by
    glibc's rand() stream at `position` after srand(seed) (pm_rand_mask) instead of the counter hash."""
    src = np.asarray(source_f32, dtype=np.float32)
    tgt = np.asarray(target_f32, dtype=np.float32)
    tp, tn = O.calculate_normals(tgt.astype(np.float64))
    keep = pm_rand_mask(src.shape[0], prob, seed, position)
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
