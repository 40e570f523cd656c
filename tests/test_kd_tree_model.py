"""The numpy model of the k-d tree build and the radix sort (tests/kd_tree_model.py) against the recursive
restatements of tests/pyref.py, node for node, without a GPU.  tests/test_gpu_kdtree_stages.py then holds the device
stages to this model bit for bit."""
import numpy as np
import pytest

import kd_tree_model as M
import pyref


def cloud(kind, n, seed=0):
    """small clouds built for the tie rule: every kind but 'uniform' has equal coordinates on some axis"""
    rng = np.random.default_rng(seed * 7919 + n)
    if kind == "uniform":
        return rng.uniform(-5, 5, (n, 3))
    if kind == "duplicates":                      # exact duplicate points
        base = rng.uniform(-5, 5, (max(1, n // 3), 3))
        return base[rng.integers(0, base.shape[0], n)]
    if kind == "signed_zeros":                    # -0.0 and +0.0 must be one coordinate
        return rng.choice(np.array([-0.0, 0.0, 0.0, -0.0, 1.0, -1.0, 2.5]), (n, 3))
    if kind == "flat":                            # a zero-spread axis
        p = rng.uniform(-5, 5, (n, 3))
        p[:, 0] = 1.25
        return p
    if kind == "lattice":                         # ties on every axis
        return rng.integers(-2, 3, (n, 3)).astype(np.float64)
    if kind == "identical":
        return np.tile(np.array([[0.5, -0.0, 3.0]]), (n, 1))
    raise ValueError(kind)


KINDS = ("uniform", "duplicates", "signed_zeros", "flat", "lattice", "identical")


def assert_matches_pynabo(pts, bucket):
    t = M.Tree(pts, bucket)
    ref = M.heap_from_pynabo(pyref.PyNabo(pts, bucket_size=bucket).nodes)
    assert sorted(ref) == sorted(np.nonzero(t.exists())[0].tolist())
    for h, (dim, a, _) in ref.items():
        assert t.dim[h] == dim, h
        if dim == M.LEAF:
            got = t.leaf_order[t.first[h]:t.first[h] + t.count[h]]
            assert got.tolist() == list(a), h
        else:
            assert np.float64(t.cut[h]).tobytes() == np.float64(a).tobytes(), h   # the raw coordinate, -0.0 kept
    return t


@pytest.mark.parametrize("bucket", range(2, 9))
def test_every_small_n_matches_pynabo(bucket):
    for n in range(1, 301):
        for kind in (KINDS[n % len(KINDS)], KINDS[(n + 3) % len(KINDS)]):
            assert_matches_pynabo(cloud(kind, n, bucket), bucket)


@pytest.mark.parametrize("kind", KINDS)
def test_tie_heavy_clouds_match_pynabo(kind):
    for bucket in range(2, 9):
        for n in (1, bucket, bucket + 1, 2 * bucket + 1, 97, 256 * bucket, 256 * bucket + 1):
            assert_matches_pynabo(cloud(kind, n, 1), bucket)


@pytest.mark.parametrize("n", [511, 1000, 1537, 2049, 3001, 4097, 5000])
def test_larger_clouds_match_pynabo(n):
    for kind, bucket in (("uniform", 8), ("lattice", 7), ("signed_zeros", 2), ("duplicates", 5)):
        assert_matches_pynabo(cloud(kind, n, 2), bucket)


@pytest.mark.parametrize("n", [1, 7, 8, 300, 2000])
def test_bucket7_leaves_are_calculate_normals_leaves(n):
    # the restatement also solves each leaf's plane, so the clouds keep leaves off planes through the origin
    for kind in ("uniform", "duplicates", "flat", "lattice"):
        pts = cloud(kind, n, 3) + np.array([10.5, -20.25, 30.125])
        _, _, leaves = pyref.calculate_normals(pts, leaf_size=7)
        t = M.Tree(pts, 7)
        assert sorted(tuple(x) for x in leaves) == sorted(tuple(x.tolist()) for x in t.leaf_sets())


@pytest.mark.parametrize("n, leaves", [(5000, 1024), (120_000, 21_696), (500_000, 106_784)])
def test_known_leaf_counts(n, leaves):
    t = M.Tree(np.random.default_rng(n).uniform(-50, 50, (n, 3)), 7)
    assert t.leaves.size == leaves
    assert np.array_equal(np.sort(t.leaf_order), np.arange(n))
    assert t.count[t.leaves].sum() == n and t.count[t.leaves].max() <= 7


def test_blocked_index_restates_common_cuh():
    def ref(h):                                    # the loop of common.cuh
        l = 0
        while ((h + 1) >> (l + 1)) != 0:
            l += 1
        j = h + 1 - (1 << l)
        bl, sl = l // 3, l % 3
        return ((((1 << (3 * bl)) - 1) // 7) + (j >> sl)) * 8 + (1 << sl) - 1 + (j & ((1 << sl) - 1))
    hs = np.concatenate([np.arange(5000), (1 << np.arange(1, 25)) - 2, (1 << np.arange(1, 25)) - 1,
                         (1 << np.arange(1, 25))])
    got = M.blocked_index(hs)
    assert got.tolist() == [ref(int(h)) for h in hs]
    for levels in range(0, 22):                    # every node of the heap fits blocked_node_slots
        last = (1 << (levels + 1)) - 2
        assert M.blocked_index(np.arange(last + 1)).max() < M.blocked_node_slots(levels)
    assert len(set(M.blocked_index(np.arange((1 << 13) - 1)).tolist())) == (1 << 13) - 1


def test_compact_layout_of_a_small_tree():
    """the compact layout by hand for n = 11, bucket 4: levels 2, the right child of the root (5 points) splits,
    the left child (6 points) splits too; every deepest slot owns one leaf"""
    pts = np.array([[float(i), 0.0, 0.0] for i in range(11)])
    t = M.Tree(pts, 4)
    assert t.levels == 2
    c = t.compact()
    assert c["mask"].all() and c["dim"].tolist() == [0, 0, 0]
    assert c["cut"].tolist() == [6.0, 3.0, 9.0]
    pb = c["pb"].reshape(4, 3, 8)
    assert pb[0, 0, :3].tolist() == [0.0, 1.0, 2.0] and np.isinf(pb[0, :, 3:]).all()
    assert c["pid"].reshape(4, 8)[3].tolist() == [9, 10] + [-1] * 6
    # n = 9, bucket 4: the root's left child (5) splits, its right child (4) is a leaf one level up: it owns slot 2,
    # slot 3 stays empty
    t = M.Tree(pts[:9], 4)
    c = t.compact()
    assert c["dim"].tolist() == [0, 0, M.LEAF]
    assert c["node"][2].tolist() == [0, M.LEAF]
    pid = c["pid"].reshape(4, 8)
    assert pid[2].tolist() == [5, 6, 7, 8] + [-1] * 4 and (pid[3] == -1).all()
    assert np.isinf(c["pb"].reshape(4, 3, 8)[3]).all()


def test_keys_order_signed_zeros_equal_and_the_rest_totally():
    v = np.array([-np.inf, -1e308, -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0, 1e308, np.inf])
    k = M.sortable_key(v)
    assert (np.diff(k.astype(object)) > 0).all()                 # -0.0 < +0.0 as bit patterns
    tk = M.tree_keys(np.stack([v, v, v], 1))
    assert tk[0][4] == tk[0][5]                                  # but equal after + 0.0
    f = np.array([-np.inf, -3.5, -1e-45, 0.0, 1e-45, 2.0, np.inf], np.float32).astype(np.float64)
    fk = M.float_key(f)
    assert (np.diff(fk.astype(object)) > 0).all() and fk.max() < (1 << 32)


def test_radix_model_orders_only_the_low_bits():
    rng = np.random.default_rng(5)
    keys = rng.integers(0, 1 << 63, 1000, dtype=np.uint64) | np.uint64(1 << 63)
    keys[::3] = keys[1]                                            # equal keys keep input order
    vals = np.arange(1000, dtype=np.uint32)
    for passes in (2, 4, 8):
        k, v = M.radix_sort(keys, vals, passes)
        low = k & np.uint64((1 << (8 * passes)) - 1 if passes < 8 else 0xFFFFFFFFFFFFFFFF)
        assert (np.diff(low.astype(object)) >= 0).all()
        assert np.array_equal(keys[v], k)                          # high bits carried with their key
        same = np.diff(low.astype(object)) == 0
        assert (np.diff(v.astype(np.int64))[same] > 0).all()       # stable
