"""SM_VOXEL_ORDER_UNORDERED_MAP without a GPU: the library's rehash schedule and hash against libstdc++'s own
std::unordered_map (oracle/unordered_map_oracle.cc), and the literal iteration order against two restatements, the
linked-list rules (pyref_unordered_map) and the epoch-sort formulation the GPU runs (voxel_order_model)."""
import numpy as np
import pytest

import chain_all_model as CM
import oracle_unordered_map as U
import pyref_unordered_map as P
import scenes
import voxel_order_model as M

INT_MIN, INT_MAX = -(2 ** 31), 2 ** 31 - 1


def model_order(keys):
    return M.order_keys(keys, U.library_hash, U.library_bucket_counts)


def pyref_order(keys):
    first, distinct = M.ranks_of_keys(keys)
    return first[P.iteration_order(U.library_hash(distinct.astype(np.int32)), U.library_bucket_counts(len(first)))]


def distinct_keys(count, seed, span=1 << 20):
    """count distinct int32 keys in random order"""
    rng = np.random.default_rng(seed)
    k = np.unique(rng.integers(-span, span, (count + count // 4 + 16, 3)), axis=0)
    assert len(k) >= count
    return k[rng.permutation(len(k))[:count]].astype(np.int32)


def thresholds(limit):
    counts = U.library_bucket_counts(limit)
    return [c for c, _ in M.epochs_of(counts)]


# ---- the schedule and the hash ----------------------------------------------------------------------------------------
def test_bucket_schedule_is_the_containers():
    m = 3_000_000
    assert np.array_equal(U.library_bucket_counts(m), U.bucket_counts(m))
    # 13 buckets from the first insert on; the 14th key rehashes to 29
    assert M.epochs_of(U.library_bucket_counts(20)) == [(0, 13), (13, 29)]


def test_bucket_schedule_is_cached_consistently():
    # a smaller m after a larger one reads the cached prefix
    assert np.array_equal(U.library_bucket_counts(1000), U.bucket_counts(1000))


KEY_SETS = {
    "random": lambda: distinct_keys(5000, 1),
    "negative": lambda: -np.abs(distinct_keys(3000, 2)) - 1,
    "int_limits": lambda: np.array([[a, b, c] for a in (INT_MIN, INT_MIN + 1, -1, 0, 1, INT_MAX - 1, INT_MAX)
                                    for b in (INT_MIN, 0, INT_MAX) for c in (INT_MIN, -7, INT_MAX)], np.int32),
    "single": lambda: np.array([[3, -4, 5]], np.int32),
}


@pytest.mark.parametrize("name", list(KEY_SETS))
def test_host_hash_is_key3hash(name):
    k = KEY_SETS[name]()
    assert np.array_equal(U.library_hash(k), U.key_hash(k))


# ---- keys that collide modulo the bucket counts ---------------------------------------------------------------------
def colliding_keys(count, buckets, seed):
    """keys whose hashes fall into a few buckets modulo `buckets`"""
    cand = distinct_keys(count * buckets // 2 + 1000, seed, span=1 << 14)
    h = U.key_hash(cand) % np.uint64(buckets)
    pick = cand[h < np.uint64(3)]
    assert len(pick) >= count
    return pick[:count]


# ---- the literal order -----------------------------------------------------------------------------------------------
def test_pyref_matches_the_container():
    for k in (distinct_keys(300, 3), distinct_keys(20_000, 4), colliding_keys(500, 59, 5), KEY_SETS["int_limits"](),
              np.repeat(distinct_keys(2000, 6), 3, axis=0)[np.random.default_rng(6).permutation(6000)]):
        assert np.array_equal(pyref_order(k), U.order_keys(k))


def test_pyref_matches_the_container_on_a_lidar_submap():
    _, sub, _ = scenes.lidar_pair(pair=1)
    pts = sub.astype(np.float32)
    assert np.array_equal(M.order_points(pts, 0.1, U.library_hash, U.library_bucket_counts), U.order_points(pts, 0.1))
    _, keys = CM.voxel_keys(pts, 0.1)
    assert np.array_equal(pyref_order(keys.astype(np.int32)), U.order_points(pts, 0.1))


def test_model_every_count_up_to_300():
    keys = distinct_keys(300, 7)
    for m in range(0, 301):
        assert np.array_equal(model_order(keys[:m]), U.order_keys(keys[:m])), m


def test_model_around_every_threshold_up_to_2_20():
    limit = 1 << 20
    keys = distinct_keys(limit + 2, 8)
    for c in thresholds(limit):
        for m in (c - 1, c, c + 1):
            if 0 <= m <= limit + 1:
                assert np.array_equal(model_order(keys[:m]), U.order_keys(keys[:m])), m


@pytest.mark.parametrize("buckets", [13, 29, 59, 127, 541])
def test_model_on_colliding_keys(buckets):
    k = colliding_keys(400, buckets, buckets)
    assert np.array_equal(model_order(k), U.order_keys(k))


@pytest.mark.parametrize("name", list(KEY_SETS))
def test_model_on_key_sets(name):
    k = KEY_SETS[name]()
    assert np.array_equal(model_order(k), U.order_keys(k))


def test_model_with_repeated_keys():
    k = np.repeat(distinct_keys(4000, 9), 5, axis=0)[np.random.default_rng(9).permutation(20000)]
    assert np.array_equal(model_order(k), U.order_keys(k))


@pytest.mark.parametrize("voxel,count", [(0.1, 100), (0.2, 36), (0.4, 9)])
def test_model_on_the_reference_lattice(voxel, count):
    pts = scenes.reference_voxel_test_cloud()
    got = M.order_points(pts, voxel, U.library_hash, U.library_bucket_counts)
    assert len(got) == count and np.array_equal(got, U.order_points(pts, voxel))


@pytest.mark.parametrize("voxel", [0.1, 0.2, 0.4])
@pytest.mark.parametrize("size", ["60k", "500k"])
def test_model_on_lidar_submaps(voxel, size):
    sub = scenes.lidar_pair(pair=1)[1] if size == "60k" else scenes.full_size_pair(0)[1]
    pts = sub.astype(np.float32)
    assert np.array_equal(M.order_points(pts, voxel, U.library_hash, U.library_bucket_counts),
                          U.order_points(pts, voxel))
    keys = np.unique(CM.voxel_keys(pts, voxel)[1], axis=0).astype(np.int32)
    assert np.array_equal(U.library_hash(keys), U.key_hash(keys))
