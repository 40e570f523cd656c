"""The radix sort and the k-d tree build on the GPU, array by array, against the numpy model of
tests/kd_tree_model.py, bit for bit.

Every matcher builds on these two stages; the k-NN and CalculateNormals tests see them only through their results,
and an exact 1-NN search is right over any valid partition.  Here the sort runs through sm_debug_radix_sort and each
tree owner (KdCompactTree with normals or ids, NormalsPipeline, FloatTree) through sm_debug_kd_tree, which builds
with the owner's own reserve / build / run, and every array the owner fills is compared: blocked nodes, leaf order,
cut / dim / node, padded buckets, normals, ids, bucket points.  The sizes straddle the points where the launch paths
change: the fused and the chunked scan of the sort (128 tiles, 32 chunks per carry pass), the fused and the separate
scan of the tree's partition (256 tiles), the capacity of kd_subtree_kernel, and deeper trees than the k-NN tests
reach.  The consumers then meet the oracle at those sizes."""
import ctypes as C

import numpy as np
import pytest

import kd_tree_model as M
import oracle_lib as O
import staticmapping_b200 as smb
from staticmapping_b200 import _lib, synth

pytestmark = pytest.mark.gpu

U64 = np.uint64
SENTINEL_KEY = U64(0xDEADBEEFCAFEF00D)
SENTINEL_VAL = np.uint32(0xA5A5A5A5)
BIG = 2_100_003                                       # > 2^21 / 2: 19 tree levels at bucket 8, 1026 sort tiles


# ------------------------------------------------------------------------------------------------ hook bindings
def device_sort(keys, vals, passes):
    """keys / vals: (batch, n) -> the sorted (batch, n) pairs; asserts that the padding up to the stride is untouched"""
    keys, vals = np.atleast_2d(keys), np.atleast_2d(vals)
    batch, n = keys.shape
    stride = (n + 63) & ~63
    k = np.full((batch, stride), SENTINEL_KEY, np.uint64)
    v = np.full((batch, stride), SENTINEL_VAL, np.uint32)
    k[:, :n], v[:, :n] = keys, vals
    ko, vo = np.zeros_like(k), np.zeros_like(v)
    rc = _lib.lib().sm_debug_radix_sort(0, k.ctypes.data, v.ctypes.data, n, batch, stride, passes, ko.ctypes.data,
                                        vo.ctypes.data)
    assert rc == 0
    assert (ko[:, n:] == SENTINEL_KEY).all() and (vo[:, n:] == SENTINEL_VAL).all()
    return ko[:, :n], vo[:, :n]


def _aos(a, dtype):
    return np.ascontiguousarray(np.asarray(a, dtype=dtype))


def device_tree(variant, pts, bucket, normals=None, first=None, first_normals=None):
    dt = np.float32 if variant == 3 else np.float64
    p = _aos(pts, dt)
    n = p.shape[0]
    L = M.num_levels(n, bucket)
    nrm = _aos(normals, np.float64) if normals is not None else None
    f = _aos(first, dt) if first is not None else None
    fn = _aos(first_normals, np.float64) if first_normals is not None else None
    entries = 8 << L
    out = {"levels": L,
           "nodes": np.zeros((M.blocked_node_slots(L), 2), np.uint64),
           "order": np.zeros(n, np.uint32),
           "cut": np.zeros(max(1, (1 << L) - 1)), "dim": np.zeros(max(1, (1 << L) - 1), np.uint8),
           "node": np.zeros((1 << L, 2), np.uint64),
           "pb": np.zeros(entries * 3), "pn": np.zeros((entries, 4)), "pid": np.zeros(entries, np.int32),
           "bpts": np.zeros((n, 4), np.uint64)}
    ptr = lambda a: None if a is None else a.ctypes.data     # noqa: E731
    rc = _lib.lib().sm_debug_kd_tree(0, variant, bucket, ptr(f), ptr(fn), 0 if f is None else f.shape[0], p.ctypes.data,
                                     ptr(nrm), n, L, out["nodes"].ctypes.data, out["order"].ctypes.data,
                                     out["cut"].ctypes.data, out["dim"].ctypes.data, out["node"].ctypes.data,
                                     out["pb"].ctypes.data, out["pn"].ctypes.data, out["pid"].ctypes.data,
                                     out["bpts"].ctypes.data)
    assert rc == 0
    return out


# ------------------------------------------------------------------------------------------------ radix sort
def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def check_sort(keys, passes, seed=0):
    keys = np.atleast_2d(keys)
    batch, n = keys.shape
    vals = (np.arange(batch * n, dtype=np.uint64).reshape(batch, n) * U64(2654435761) + U64(seed)).astype(np.uint32)
    gk, gv = device_sort(keys, vals, passes)
    for b in range(batch):
        wk, wv = M.radix_sort(keys[b], vals[b], passes)
        assert np.array_equal(gk[b], wk), (n, batch, passes, b, int(np.argmax(gk[b] != wk)))
        assert np.array_equal(gv[b], wv), (n, batch, passes, b, int(np.argmax(gv[b] != wv)))


SORT_SIZES = [1, 2, 2047, 2048, 2049, 262_144, 262_145, 294_912, 294_913, 1_048_576, 1_048_577, (1 << 21) + 5]


@pytest.mark.parametrize("n", SORT_SIZES)
@pytest.mark.parametrize("batch", [1, 3])
def test_sort_random_keys(n, batch):
    rng = np.random.default_rng(n + batch)
    keys = rng.integers(0, 1 << 64, (batch, n), dtype=np.uint64, endpoint=False)
    for passes in (2, 4, 8):
        check_sort(keys, passes, seed=passes)


@pytest.mark.parametrize("n", [2049, 262_145, 1_048_577, (1 << 21) + 5])
def test_sort_equal_keys(n):
    """one digit holds every key of every tile in every pass"""
    keys = np.full((3, n), U64(0x0123456789ABCDEF))
    for passes in (2, 4, 8):
        check_sort(keys, passes)


@pytest.mark.parametrize("n", [2048, 294_913, 1_048_577])
def test_sort_leaves_the_high_bits_unordered(n):
    """only bits above the sorted ones vary: the order is the input order, the high bits travel with their keys"""
    rng = np.random.default_rng(n)
    high = rng.integers(0, 1 << 32, (3, n), dtype=np.uint64) << U64(32)
    for passes in (2, 4):
        low = U64(0x5A5A)
        keys = high | low
        if passes == 4:
            keys = keys | (rng.integers(0, 4, (3, n), dtype=np.uint64) << U64(16))  # a few low-half digits vary
        check_sort(keys, passes)


def _special_doubles(rng, n):
    v = rng.standard_normal(n) * np.exp(rng.uniform(-700, 700, n))
    pool = np.array([0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324, 2.2250738585072014e-308, -1e-310, 1e-310,
                     np.finfo(np.float64).max, -np.finfo(np.float64).max, 1.0, -1.0])
    pick = rng.random(n) < 0.3
    v[pick] = rng.choice(pool, int(pick.sum()))
    return v


@pytest.mark.parametrize("n", [2049, 262_145, 1_048_577, (1 << 21) + 5])
def test_sort_double_keys(n):
    """sortable_key of doubles incl. +-0, +-inf and denormals (8 passes), and kd_keys_kernel's float keys (4 passes)"""
    rng = np.random.default_rng(n + 11)
    dbl = np.stack([_special_doubles(rng, n) for _ in range(3)])
    check_sort(np.stack([M.sortable_key(d) for d in dbl]), 8)
    with np.errstate(over="ignore"):                                 # beyond the float range: +-inf
        flt = dbl.astype(np.float32).astype(np.float64)
    check_sort(M.tree_keys(flt.T, keys32=True), 4)
    check_sort(M.tree_keys(dbl.T), 8)


# ------------------------------------------------------------------------------------------------ trees
def check_tree(variant, pts, bucket, normals=None, first=None, first_normals=None):
    got = device_tree(variant, pts, bucket, normals, first, first_normals)
    src = np.asarray(pts, np.float32 if variant == 3 else np.float64).astype(np.float64)
    t = M.Tree(src, bucket)
    assert got["levels"] == t.levels
    slots, rec = t.blocked_nodes()
    bad = np.nonzero((got["nodes"][slots] != rec).any(1))[0]
    assert bad.size == 0, ("nodes", int(slots[bad[0]]))
    bad = np.nonzero(got["order"] != t.leaf_order)[0]
    assert bad.size == 0, ("order", int(bad[0]))
    if variant <= 1:
        c = t.compact(normals)
        m = c["mask"]
        top = m.size
        bad = np.nonzero(m & (got["dim"][:top] != c["dim"]))[0]
        assert bad.size == 0, ("dim", int(bad[0]))
        inner = m & (c["dim"] != M.LEAF)
        bad = np.nonzero(inner & (_bits(got["cut"][:top]) != _bits(c["cut"])))[0]
        assert bad.size == 0, ("cut", int(bad[0]))
        bad = np.nonzero(m & (got["node"][1:top + 1] != c["node"]).any(1))[0]
        assert bad.size == 0, ("node", int(bad[0]) + 1)
        bad = np.nonzero(_bits(got["pb"]) != _bits(c["pb"]))[0]
        assert bad.size == 0, ("pb", int(bad[0]))
        if variant == 0:
            bad = np.nonzero((_bits(got["pn"]) != _bits(c["pn"])).any(1))[0]
            assert bad.size == 0, ("pn", int(bad[0]))
        else:
            bad = np.nonzero(got["pid"] != c["pid"])[0]
            assert bad.size == 0, ("pid", int(bad[0]))
    if variant == 3:
        xyz, ids = t.bucket_points()
        bad = np.nonzero((got["bpts"][:, :3] != _bits(xyz)).any(1) | (got["bpts"][:, 3] != ids.astype(np.uint64)))[0]
        assert bad.size == 0, ("bpts", int(bad[0]))
    return t


def tie_cloud(kind, n, seed=0):
    rng = np.random.default_rng(seed * 7919 + n)
    if kind == "uniform":
        return rng.uniform(-50, 50, (n, 3))
    if kind == "duplicates":
        base = rng.uniform(-5, 5, (max(1, n // 3), 3))
        return base[rng.integers(0, base.shape[0], n)]
    if kind == "signed_zeros":
        return rng.choice(np.array([-0.0, 0.0, 0.0, -0.0, 1.0, -1.0, 2.5]), (n, 3))
    if kind == "flat":
        p = rng.uniform(-5, 5, (n, 3))
        p[:, 0] = 1.25
        return p
    if kind == "lattice":
        side = max(2, int(round(n ** (1 / 3))) // 2)
        return rng.integers(-side, side + 1, (n, 3)).astype(np.float64)
    if kind == "identical":
        return np.tile(np.array([[0.5, -0.0, 3.0]]), (n, 1))
    raise ValueError(kind)


KINDS = ("uniform", "duplicates", "signed_zeros", "flat", "lattice", "identical")
_LIDAR = {}


def lidar_cloud(n):
    """a lidar scan of the synthetic scene, tiled with whole-metre offsets up to n float points"""
    if "scan" not in _LIDAR:
        _LIDAR["scan"] = synth.lidar_scan(synth.make_scene(seed=3), seed=3, n_az=1000)
    scan = _LIDAR["scan"].astype(np.float64)
    reps = -(-n // scan.shape[0])
    tiles = [scan + np.array([0.0, 0.0, 40.0 * r]) for r in range(reps)]
    return np.concatenate(tiles)[:n].astype(np.float32)


def _normals_for(pts, seed=1):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(np.asarray(pts).shape)
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def small_sizes(bucket):
    cap = M.sub_capacity(bucket)
    return [1, bucket, bucket + 1, cap, cap + 1, 2 * cap, 2 * cap + 1]


@pytest.mark.parametrize("bucket", range(2, 9))
@pytest.mark.parametrize("variant", [0, 1])
def test_compact_tree_small_sizes_every_bucket(variant, bucket):
    for i, n in enumerate(small_sizes(bucket)):
        for kind in (KINDS[i % len(KINDS)], KINDS[(i + 3) % len(KINDS)]):
            pts = tie_cloud(kind, n, bucket)
            t = check_tree(variant, pts, bucket, _normals_for(pts) if variant == 0 else None)
            if n == 2 * M.sub_capacity(bucket) + 1:
                assert t.global_levels() == 2


@pytest.mark.parametrize("kind", KINDS)
def test_normals_pipeline_and_float_tree_small_sizes(kind):
    for variant, bucket in ((2, 7), (3, 8)):
        for n in small_sizes(bucket) + [5000]:
            check_tree(variant, tie_cloud(kind, n, variant), bucket)


LARGE = [524_288, 524_289, 1_048_577, BIG]


@pytest.mark.parametrize("variant, n", [(v, n) for v in range(4) for n in LARGE] + [(1, 917_505), (2, 917_505)])
def test_trees_past_the_launch_path_changes(variant, n):
    """n > 524 288: the partition's separate block-sum scan; > 1 048 576 sort keys per axis: more than 32 scan chunks;
    917 505 = 1792 * 2^9 + 1 at bucket 7 (NormalsPipeline, a bucket-7 KdCompactTree): one global level more than
    917 504"""
    bucket = {2: 7, 3: 8}.get(variant, 7 if n == 917_505 else 8)
    if variant == 3:
        pts = lidar_cloud(n)
    else:
        pts = tie_cloud("uniform" if n % 2 else "lattice", n, variant)
    t = check_tree(variant, pts, bucket, _normals_for(pts) if variant == 0 else None)
    assert t.levels >= 16 and t.global_levels() >= 8


@pytest.mark.parametrize("variant", [0, 1, 2, 3])
def test_reused_owner_equals_a_fresh_build(variant):
    """an owner that built a 600 k-point cloud, then a 3 k-point one (buffers only grow), and the reverse order"""
    bucket = {2: 7, 3: 8}.get(variant, 8)
    if variant == 3:
        big, small = lidar_cloud(600_000), lidar_cloud(3000) + np.float32(0.5)
    else:
        big, small = tie_cloud("uniform", 600_000, 5), tie_cloud("lattice", 3000, 6)
    nb = _normals_for(big, 2) if variant == 0 else None
    ns = _normals_for(small, 3) if variant == 0 else None
    check_tree(variant, small, bucket, ns, first=big, first_normals=nb)
    check_tree(variant, big, bucket, nb, first=small, first_normals=ns)


# ------------------------------------------------------------------------------------------------ the consumers
def _queries(target, n, seed):
    rng = np.random.default_rng(seed)
    t = np.asarray(target, np.float64)
    q = t[rng.integers(0, t.shape[0], n)] + rng.normal(0, 0.3, (n, 3))
    return np.concatenate([q, t[:64]])                # and some queries exactly on target points


@pytest.mark.parametrize("nt", [524_289, 1_100_003])
def test_knn1_on_deep_targets_against_the_oracle(nt):
    tgt = tie_cloud("uniform", nt, 9)
    assert M.num_levels(nt, 8) in (17, 18)
    q = _queries(tgt, 20_000, nt)
    for eps in (0.0, 3.16):
        ids, d2 = smb.knn1(tgt, q, epsilon=eps)
        oi, od = O.knn1(tgt, q, epsilon=eps)
        assert np.array_equal(ids, oi), eps
        assert _bits(d2).tobytes() == _bits(od).tobytes(), eps


@pytest.mark.parametrize("n", [917_505, 1_100_003])
def test_calculate_normals_at_large_sizes_against_the_oracle(n):
    pts = lidar_cloud(n).astype(np.float64)
    got = smb.CalculateNormals(pts)
    wp, wn = O.calculate_normals(pts)
    assert got.points.shape == wp.shape
    assert _bits(got.points).tobytes() == _bits(wp).tobytes()
    assert _bits(got.normals).tobytes() == _bits(wn).tobytes()


def test_float_tree_knn1_at_large_size_against_the_oracle():
    cloud = lidar_cloud(1_100_003)
    q = _queries(cloud, 20_000, 4)
    ids = np.zeros(q.shape[0], np.int32)
    d2 = np.zeros(q.shape[0])
    rc = _lib.lib().sm_debug_float_tree_knn(0, cloud.ctypes.data, cloud.shape[0], np.ascontiguousarray(q).ctypes.data,
                                            q.shape[0], 1, ids.ctypes.data, d2.ctypes.data)
    assert rc == 0
    oi, od = O.knn1(cloud.astype(np.float64), q, epsilon=0.0)
    assert np.array_equal(ids, oi)
    assert _bits(d2).tobytes() == _bits(od).tobytes()


def test_voxel_grid_filter_past_32_scan_chunks_against_the_oracle():
    rng = np.random.default_rng(21)
    n = 2_200_001
    pts = np.zeros((n, 5), np.float32)
    pts[:, :3] = rng.uniform(-60, 60, (n, 3))
    pts[:, 3] = rng.uniform(0, 255, n)
    m, want = O.voxel_grid_filter(pts, 0.5)
    got = smb.VoxelGridFilter(pts, 0.5)
    assert got.shape == (m, 5)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
