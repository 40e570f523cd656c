"""A step-by-step numpy model of the epoch-sort formulation SM_VOXEL_ORDER_UNORDERED_MAP runs on the GPU
(csrc/voxel_filter.cu): per rehash epoch e (from c_e distinct keys on, B_e buckets, n_e keys at its end), every voxel
present takes v = its position before the epoch for t < c_e, v = t otherwise; a bucket's run key is n_e - 1 - min v
over the bucket, a voxel's within-run key n_e - 1 - v; the list after the epoch is ascending (run key, within-run key).
TEST INFRASTRUCTURE."""
from __future__ import annotations

import numpy as np

import chain_all_model as CM


def epochs_of(bucket_counts):
    """[(c_e, B_e)] from bucket_count() after each distinct insert"""
    bc = np.asarray(bucket_counts, np.uint64)
    if len(bc) == 0:
        return []
    starts = np.flatnonzero(np.r_[True, bc[1:] != bc[:-1]])
    return [(int(c), int(bc[c])) for c in starts]


def epoch_positions(hashes, epochs):
    """hashes: uint64 by insertion rank -> the list position of every rank present after each epoch"""
    h = np.asarray(hashes, np.uint64)
    m = len(h)
    pos = np.zeros(0, np.int64)
    out = []
    for e, (c, buckets) in enumerate(epochs):
        ne = epochs[e + 1][0] if e + 1 < len(epochs) else m
        t = np.arange(ne, dtype=np.int64)
        v = t.copy()
        v[:c] = pos[:c]
        b = (h[:ne] % np.uint64(buckets)).astype(np.int64)
        table = np.full(buckets, np.iinfo(np.int64).max, np.int64)
        np.minimum.at(table, b, v)
        bits = max(1, int(ne - 1).bit_length())
        key = ((ne - 1 - table[b]).astype(np.uint64) << np.uint64(bits)) | (ne - 1 - v).astype(np.uint64)
        assert len(np.unique(key)) == ne                      # one position per voxel
        pos = np.empty(ne, np.int64)
        pos[np.argsort(key, kind="stable")] = t
        out.append(pos)
    return out


def ranks_of_keys(keys):
    """(first index of every distinct key in insertion order, the keys in that order)"""
    k = np.asarray(keys).reshape(-1, 3)
    _, first = np.unique(k, axis=0, return_index=True)
    first = np.sort(first)
    return first, k[first]


def order_keys(keys, hash_fn, schedule_fn):
    """the iteration order (first indices) the formulation gives for int keys (N, 3)"""
    first, distinct = ranks_of_keys(keys)
    if len(first) == 0:
        return first
    steps = epoch_positions(hash_fn(distinct.astype(np.int32)), epochs_of(schedule_fn(len(first))))
    return first[np.argsort(steps[-1])]


def order_points(records, voxel_size, hash_fn, schedule_fn):
    """the same for a cloud: the points VoxelGrid keeps (finite quotients), keyed as the filter keys them"""
    kept, keys = CM.voxel_keys(records, voxel_size)
    rows = np.flatnonzero(kept)
    return rows[order_keys(keys[rows].astype(np.int64).astype(np.int32), hash_fn, schedule_fn)]
