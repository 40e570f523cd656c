"""PCL's StatisticalOutlierRemoval (setMeanK(K), setStddevMulThresh(std_mul)) restated in numpy / scipy, independently of
the product and of oracle/statistic_removal_oracle.cc.  TEST INFRASTRUCTURE.

Neighbours are ranked by a key over all finite points: `rank="float"` is FLANN's L2_Simple<float> d2 (what PCL ranks
by), `rank="double"` the d2 of the coordinates widened to double in libnabo's operation order (what the GPU ranks by).
Small clouds are searched by brute force; larger ones take scipy's cKDTree candidates, re-ranked by the key, and a
query whose candidates leave too small a margin to the first point left out is searched by brute force.  Per point the
mean of sqrt((double)float d2) over neighbours 1..K; the two sums of the statistics are math.fsum's (the exact sum
rounded once)."""
from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np

F32, F64 = np.float32, np.float64
BRUTE_MAX = 4096          # finite points up to which every query is searched by brute force
MARGIN = {"float": 1e-6, "double": 1e-9}   # relative gap a key may be off the cKDTree's squared distance


class Result(NamedTuple):
    kept: np.ndarray         # (n,) bool
    distances: np.ndarray    # (n,) float32
    stats: tuple             # mean, stddev, threshold, valid


def _float_d2(q, p):
    """L2_Simple<float>: q (r, 3), p (r, c, 3) float32 -> (r, c) float32, ((0 + dx*dx) + dy*dy) + dz*dz"""
    d = (q[:, None, :] - p).astype(F32)
    return ((F32(0) + d[..., 0] * d[..., 0]) + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _double_d2(q, p):
    d = q[:, None, :].astype(F64) - p.astype(F64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _key(rank, q, p):
    return _float_d2(q, p) if rank == "float" else _double_d2(q, p)


def _brute(P, rows, K, rank):
    out = np.empty((len(rows), K + 1), np.int64)
    for a in range(0, len(rows), 512):
        r = rows[a:a + 512]
        key = _key(rank, P[r], P[None, :, :])
        out[a:a + 512] = np.argsort(key, axis=1, kind="stable")[:, :K + 1]
    return out


def neighbours(P, K, rank="float"):
    """P: (nf, 3) float32 finite points -> (nf, K + 1) indices in list order, entry 0 included"""
    nf = len(P)
    if nf <= BRUTE_MAX:
        return _brute(P, np.arange(nf), K, rank)
    from scipy.spatial import cKDTree
    kc = min(nf, K + 1 + 8)
    d, idx = cKDTree(P.astype(F64)).query(P.astype(F64), k=kc)
    key = _key(rank, P, P[idx])
    order = np.argsort(key, axis=1, kind="stable")
    nb = np.take_along_axis(idx, order[:, :K + 1], axis=1)
    sel = np.take_along_axis(key, order[:, K:K + 1], axis=1)[:, 0].astype(F64)
    last = d[:, -1] ** 2
    bad = np.flatnonzero(~((sel == 0) | (sel <= last * (1 - MARGIN[rank]))))
    if bad.size:
        nb[bad] = _brute(P, bad, K, rank)
    return nb


def statistic_removal(records, K=30, std_mul=1.0, rank="float"):
    """records: (n, >= 3) float32 -> Result; raises RuntimeError for 1..K finite points (PCL's CHECK case)"""
    xyz = np.asarray(records, F32)[:, :3]
    n = len(xyz)
    finite = np.flatnonzero(np.all(np.isfinite(xyz), axis=1))
    nf = len(finite)
    if 1 <= nf <= K:
        raise RuntimeError("CHECK: between 1 and K finite points")
    dist = np.zeros(n, F32)
    if nf:
        P = np.ascontiguousarray(xyz[finite])
        nb = neighbours(P, K, rank)
        d2 = _float_d2(P, P[nb[:, 1:]])                    # (nf, K) float32, entries 1..K
        s = np.zeros(nf, F64)
        for j in range(K):
            s = s + np.sqrt(d2[:, j].astype(F64))
        dist[finite] = (s / F64(K)).astype(F32)
    total = F64(math.fsum(dist.astype(F64).tolist()))
    sq_total = F64(math.fsum((dist * dist).astype(F64).tolist()))
    valid = F64(nf)
    with np.errstate(all="ignore"):
        mean = total / valid
        variance = (sq_total - total * total / valid) / (valid - F64(1))
        stddev = np.sqrt(variance)
        threshold = mean + F64(F32(std_mul)) * stddev
    kept = ~(dist.astype(F64) > threshold)
    return Result(kept, dist, (float(mean), float(stddev), float(threshold), float(valid)))
