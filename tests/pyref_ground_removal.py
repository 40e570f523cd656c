"""GroundRemoval (v1) in numpy, written from the definition in include/sm_b200.h independently of the C++ oracle: float32
division, explicit truncation with the INT_MIN rule, a stable lexsort on (ix, iy, iz) and per-voxel reductions.
TEST INFRASTRUCTURE."""
import numpy as np

import oracle_ground_removal as OG

F32 = np.float32
INT_MIN = -(1 << 31)


def voxel_index(xyz, leaf_size):
    """(n, 3) int64: trunc(float32(coord / leaf_size)), INT_MIN for NaN or outside (-2^31 - 1, 2^31)"""
    with np.errstate(all="ignore"):
        q = (np.asarray(xyz, F32) / F32(leaf_size)).astype(np.float64)
        ok = (q > -2147483649.0) & (q < 2147483648.0)
        return np.where(ok, np.trunc(np.where(ok, q, 0.0)), INT_MIN).astype(np.int64)


def voxel_status(z, iz, min_points, height_threshold):
    """one voxel's fate from its z values (any order): 0 skipped, 1 ground, 2 kept"""
    z = np.asarray(z, F32)
    if len(z) < min_points:
        return 0
    if iz > 0:
        return 2
    finite_or_inf = z[~np.isnan(z)]
    max_z = max(F32(-1e9), finite_or_inf.max()) if len(finite_or_inf) else F32(-1e9)
    min_z = min(F32(1e9), finite_or_inf.min()) if len(finite_or_inf) else F32(1e9)
    delta = F32(max_z) - F32(min_z)
    return 1 if (delta >= 0 and delta <= F32(height_threshold)) else 2


def ground_removal(records, min_point_num_in_voxel=10, leaf_size=0.8, height_threshold=0.15):
    rec = np.ascontiguousarray(np.asarray(records, F32)[:, :5])
    n = len(rec)
    if n == 0:
        e = np.zeros(0, np.int32)
        return OG.Result(np.zeros((0, 5), F32), e, e, e)
    idx = voxel_index(rec[:, :3], leaf_size)
    order = np.lexsort((idx[:, 2], idx[:, 1], idx[:, 0]))          # stable: a voxel keeps its input order
    s = idx[order]
    heads = np.flatnonzero(np.r_[True, np.any(s[1:] != s[:-1], axis=1)])
    ends = np.r_[heads[1:], n]
    z = rec[order, 2]
    # per-voxel max / min over the non-NaN z, against the loop's initial -1e9 / 1e9
    with np.errstate(invalid="ignore"):
        zmax = np.maximum.reduceat(np.where(np.isnan(z), -np.inf, z).astype(F32), heads)
        zmin = np.minimum.reduceat(np.where(np.isnan(z), np.inf, z).astype(F32), heads)
    zmax = np.maximum(zmax, F32(-1e9)).astype(F32)
    zmin = np.minimum(zmin, F32(1e9)).astype(F32)
    count = ends - heads
    delta = (zmax - zmin).astype(F32)
    ground = (s[heads, 2] <= 0) & (delta >= 0) & (delta <= F32(height_threshold))
    status = np.where(count < min_point_num_in_voxel, 0, np.where(ground, 1, 2))
    per_sorted = np.repeat(status, count)
    emitted = order[per_sorted == 2]
    return OG.Result(rec[emitted].copy(), emitted.astype(np.int32), np.sort(emitted).astype(np.int32),
                     np.sort(order[per_sorted == 1]).astype(np.int32))
