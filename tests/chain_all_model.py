"""Whole filter chains with GroundRemoval, StatisticRemoval and VoxelGrid among their stages (the chain option
all_filters, include/sm_b200.h), composed stage by stage with the scan indices carried, twice: from the C++
restatements (oracle_filters, oracle_ground_removal, oracle_statistic_removal, oracle_lib's VoxelGrid) and from the
numpy ones (pyref_filters, pyref_ground_removal, pyref_statistic_removal and the VoxelGrid below).  A chain is
[(name, {xml name: value}), ...]; a stage reads the previous stage's records in their order.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import math

import numpy as np

import oracle_filters as OF
import oracle_ground_removal as OG
import oracle_lib as O
import oracle_statistic_removal as OS
import pyref_filters as PF
import pyref_ground_removal as PG
import pyref_statistic_removal as PR

F32, F64 = np.float32, np.float64
NEW = ("GroundRemoval", "StatisticRemoval", "VoxelGrid")
GR_DEFAULT = dict(min_point_num_in_voxel=10, leaf_size=0.8, height_threshold=0.15)
SR_DEFAULT = dict(point_num_meank=30, std_mul=1.0)
VG_DEFAULT = dict(voxel_size=0.1)


class CheckFailed(RuntimeError):
    """a stage CHECK-fails (StatisticRemoval with 1..K finite points)"""


def voxel_keys(records, voxel_size):
    """(kept, keys): VoxelGrid's voxel of every record, lround(float32(coordinate / voxel_size)) halves away from zero;
    kept is False where a quotient is NaN, inf or not below 9e18 in magnitude (the point is dropped)"""
    with np.errstate(all="ignore"):
        q = (np.asarray(records, F32)[:, :3] / F32(voxel_size)).astype(F64)
        kept = np.all(np.abs(q) < 9.0e18, axis=1)
        q = np.where(kept[:, None], q, 0.0)
        return kept, np.where(q >= 0, np.floor(q + 0.5), np.ceil(q - 0.5)).astype(np.int64)


def voxel_first_members(records, voxel_size):
    """the position of each voxel's first member, voxels in ascending (ix, iy, iz)"""
    kept, keys = voxel_keys(records, voxel_size)
    rows = np.flatnonzero(kept)
    _, first = np.unique(keys[rows], axis=0, return_index=True)
    return rows[first]


def _params(defaults, params):
    p = dict(defaults)
    for k, v in (params or {}).items():
        if k not in p:
            raise KeyError(k)
        p[k] = v
    return p


# ---- the C++ restatements -------------------------------------------------------------------------------------------
def oracle_stage(name, params, rec, index, seed=1):
    """one stage on records `rec` with scan indices `index` -> (records, scan indices)"""
    if name == "GroundRemoval":
        r = OG.ground_removal(rec, **_params(GR_DEFAULT, params))
        return r.out, index[r.index]
    if name == "StatisticRemoval":
        p = _params(SR_DEFAULT, params)
        try:
            r = OS.statistic_removal(rec, p["point_num_meank"], p["std_mul"], OS.PRODUCT)
        except RuntimeError as e:
            raise CheckFailed(str(e)) from None
        return r.out, index[r.inliers]
    if name == "VoxelGrid":
        voxel = _params(VG_DEFAULT, params)["voxel_size"]
        kept, _ = voxel_keys(rec, voxel)
        m, out = O.voxel_grid_filter(np.ascontiguousarray(rec[kept]), voxel)   # the oracle leaves lround(NaN) undefined
        first = voxel_first_members(rec, voxel)
        assert m == len(first)
        return out, index[first]
    keep = OF.filter_flags(name, params, rec, index, seed).astype(bool)
    return np.ascontiguousarray(rec[keep]), index[keep]


# ---- the numpy restatements -----------------------------------------------------------------------------------------
def pyref_voxel_grid(rec, voxel_size):
    """VoxelGrid::Filter in plain Python: a dict of voxels in input order, double sums in input order, means cast to
    float, factor 0, voxels in ascending (ix, iy, iz); -> (records, first member of each voxel)"""
    q = np.asarray(rec, F32)[:, :3] / F32(voxel_size) if len(rec) else np.zeros((0, 3), F32)
    voxels = {}
    for i in range(len(rec)):
        key = []
        for v in q[i].tolist():
            if not (abs(v) < 9.0e18):
                break
            key.append(int(math.copysign(math.floor(abs(v) + 0.5), v)))
        if len(key) < 3:
            continue
        acc = voxels.setdefault(tuple(key), [i, 0, 0.0, 0.0, 0.0, 0.0])
        acc[1] += 1
        for c in range(4):
            acc[2 + c] += float(rec[i, c])
    out = np.zeros((len(voxels), 5), F32)
    first = np.zeros(len(voxels), np.int64)
    for j, key in enumerate(sorted(voxels)):
        acc = voxels[key]
        first[j] = acc[0]
        out[j, :4] = [F32(s / acc[1]) for s in acc[2:]]
    return out, first


def pyref_stage(name, params, rec, index, seed=1):
    if name == "GroundRemoval":
        r = PG.ground_removal(rec, **_params(GR_DEFAULT, params))
        return r.out, index[r.index]
    if name == "StatisticRemoval":
        p = _params(SR_DEFAULT, params)
        try:
            keep = PR.statistic_removal(rec, p["point_num_meank"], p["std_mul"], rank="double").kept
        except RuntimeError as e:
            raise CheckFailed(str(e)) from None
        return np.ascontiguousarray(rec[keep]), index[keep]
    if name == "VoxelGrid":
        out, first = pyref_voxel_grid(rec, _params(VG_DEFAULT, params)["voxel_size"])
        return out, index[first]
    keep = PF.filter_flags(name, params, rec, index, seed)
    return np.ascontiguousarray(rec[keep]), index[keep]


def chain(filters, cloud, seed=1, stage=oracle_stage):
    """Factory::Filter with the option on -> (records of the last stage, their scan indices in emission order); an
    empty cloud ends the chain"""
    r = np.ascontiguousarray(np.asarray(cloud, F32)[:, :5])
    index = np.arange(len(r), dtype=np.int32)
    for name, params in filters:
        if len(r) == 0:
            break
        r, index = stage(name, params, r, index, seed)
        r, index = np.ascontiguousarray(r, F32), np.asarray(index, np.int32)
    return r, index
