"""VoxelGrid in the reference's std::unordered_map order on an H100 (SM_VOXEL_ORDER_UNORDERED_MAP,
csrc/voxel_filter.cu) against libstdc++'s own container (oracle/unordered_map_oracle.cc and the oracle's VoxelGrid
with order_mode 1): records byte for byte, the epoch hook against the model, the filter chain in both run forms, the
submap target through CalculateNormals in std::nth_element's order and IcpFast, and the C++ adapter."""
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

import chain_all_model as CM
import filter_scenes as FS
import oracle_lib as O
import oracle_mt19937 as OM
import oracle_unordered_map as U
import scenes
import staticmapping_b200 as smb
import test_gpu_filter_chain_all as G
import voxel_order_model as M
from cxx import adapter_exe
from staticmapping_b200 import _lib

pytestmark = pytest.mark.gpu
UMAP = smb.VoxelOrder.UNORDERED_MAP
F32 = np.float32


def as5(xyz, seed=0):
    rng = np.random.default_rng(seed)
    p = np.zeros((len(xyz), 5), F32)
    p[:, :3] = xyz
    p[:, 3] = rng.uniform(0, 255, len(xyz))
    p[:, 4] = rng.uniform(0, 1, len(xyz))
    return p


def ordered(pts, voxel, order=UMAP):
    """sm_voxel_grid_filter_ordered -> (rc, records)"""
    out = np.full((max(len(pts), 1), 5), -7.0, F32)
    m = C.c_int64(-3)
    p = np.ascontiguousarray(pts, F32)
    rc = _lib.lib().sm_voxel_grid_filter_ordered(0, p.ctypes.data, len(p), 20, voxel, int(order), out.ctypes.data,
                                                  C.byref(m))
    return rc, out[:max(m.value, 0)], m.value


def check_against_oracle(pts, voxel, finite=None):
    rc, got, m = ordered(pts, voxel)
    want_m, want = O.voxel_grid_filter(pts if finite is None else finite, voxel, order_mode=1)
    assert rc == 0 and m == want_m
    assert got.tobytes() == want.tobytes()
    assert np.array_equal(smb.VoxelGridFilter(pts, voxel, order=UMAP), want)
    return m


# ---- the clouds ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sub60k():
    return as5(scenes.lidar_pair(pair=1)[1].astype(F32), seed=1)


@pytest.fixture(scope="module")
def sub500k():
    return as5(scenes.full_size_pair(0)[1].astype(F32), seed=2)


def cloud_with_voxels(count, voxel, seed, per_voxel=3):
    """a cloud of exactly `count` occupied voxels, per_voxel points in each, shuffled"""
    rng = np.random.default_rng(seed)
    keys = np.unique(rng.integers(-2000, 2000, (count + count // 2 + 8, 3)), axis=0)
    keys = keys[rng.permutation(len(keys))[:count]]
    xyz = (np.repeat(keys, per_voxel, axis=0) + rng.uniform(-0.3, 0.3, (count * per_voxel, 3))) * voxel
    return as5(xyz.astype(F32)[rng.permutation(count * per_voxel)], seed)


def thresholds(limit):
    return [c for c, _ in M.epochs_of(U.library_bucket_counts(limit))]


def test_reference_lattice():
    pts = scenes.reference_voxel_test_cloud()
    for voxel, count in ((0.1, 100), (0.2, 36), (0.4, 9), (10.0, 1)):
        assert check_against_oracle(pts, voxel) == count


@pytest.mark.parametrize("voxel", [0.1, 0.2, 0.4])
def test_submaps(sub60k, sub500k, voxel):
    for pts in (sub60k, sub500k):
        check_against_oracle(pts, voxel)


def test_voxel_counts_at_every_rehash_threshold():
    for c in thresholds(200_000)[1:]:
        for count in (c - 1, c, c + 1):
            pts = cloud_with_voxels(count, 0.1, count)
            assert check_against_oracle(pts, 0.1) == count


def test_all_distinct_and_dense_voxels():
    rng = np.random.default_rng(4)
    distinct = as5((np.arange(150_000)[:, None] * np.array([0.1, 0.0, 0.0]) + [0.0, 1.0, 2.0]).astype(F32), 4)
    assert check_against_oracle(distinct[rng.permutation(len(distinct))], 0.1) == 150_000
    dense = cloud_with_voxels(200, 0.8, 5, per_voxel=1000)                 # 1000 points per 0.8 m voxel
    assert check_against_oracle(dense, 0.8) == 200


def test_far_from_the_origin():
    rng = np.random.default_rng(3)
    xyz = rng.uniform(-20, 20, (20000, 3)) + np.array([150_000.0, -90_000.0, 30.0])
    check_against_oracle(as5(xyz.astype(F32), 3), 0.1)


def test_non_finite_points_are_dropped_before_insertion(sub60k):
    dirty = sub60k.copy()
    bad = [0, 7, 11, 13, 5000, len(dirty) - 1]
    dirty[0, 0] = np.nan; dirty[7, 0] = np.nan; dirty[11, 2] = np.inf; dirty[13, 1] = -np.inf
    dirty[5000, 1] = np.nan; dirty[-1, 2] = np.inf
    check_against_oracle(dirty, 0.1, finite=np.delete(sub60k, bad, axis=0))


def test_argument_errors_and_default_order(sub60k):
    one = sub60k[:10]
    for order in (2, -1):
        rc, out, m = ordered(one, 0.1, order)
        assert rc == -1 and m == -3 and np.all(out == -7.0)
    with pytest.raises(ValueError):
        smb.VoxelGridFilter(one, 0.1, order=2)
    m, want = O.voxel_grid_filter(sub60k, 0.2)
    rc, got, _ = ordered(sub60k, 0.2, smb.VoxelOrder.ASCENDING)
    assert rc == 0 and got.tobytes() == want.tobytes() == smb.VoxelGridFilter(sub60k, 0.2).tobytes()


# ---- the epoch hook --------------------------------------------------------------------------------------------------
def device_epochs(pts, voxel):
    n = len(pts)
    hashes, ranks = np.zeros(n, np.uint64), np.zeros(n, np.int32)
    cap = n * 40
    pos = np.zeros(cap, np.int32)
    m, ne = C.c_int64(-1), C.c_int32(-1)
    p = np.ascontiguousarray(pts, F32)
    rc = _lib.lib().sm_debug_voxel_unordered_epochs(0, p.ctypes.data, n, 20, voxel, hashes.ctypes.data,
                                                     ranks.ctypes.data, pos.ctypes.data, cap, C.byref(m), C.byref(ne))
    assert rc == 0
    m, ne = m.value, ne.value
    return hashes[:m], ranks[:m], pos[:m * ne].reshape(ne, m)


@pytest.mark.parametrize("name", ["lattice", "threshold", "sub60k"])
def test_epoch_hook_matches_the_model(sub60k, name):
    pts, voxel = {"lattice": (scenes.reference_voxel_test_cloud(), 0.1),
                  "threshold": (cloud_with_voxels(5087, 0.2, 9), 0.2), "sub60k": (sub60k, 0.1)}[name]
    hashes, ranks, pos = device_epochs(pts, voxel)
    _, keys = CM.voxel_keys(pts, voxel)
    first, by_rank = M.ranks_of_keys(keys)
    asc, first_of_asc = np.unique(keys, axis=0, return_index=True)
    want_rank = np.searchsorted(first, first_of_asc)
    assert np.array_equal(ranks, want_rank)
    assert np.array_equal(hashes, U.key_hash(asc.astype(np.int32)))
    steps = M.epoch_positions(U.key_hash(by_rank.astype(np.int32)), M.epochs_of(U.bucket_counts(len(first))))
    assert len(steps) == len(pos)
    for e, want in enumerate(steps):
        assert np.array_equal(pos[e, :len(want)], want), e
        assert np.all(pos[e, len(want):] == -1)


# ---- the filter chain ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scan():
    return FS.scan()            # 120 000 points


def literal_chain(filters, cloud, voxel_literal, samplers=None, seed=1):
    """Factory::Filter composed from the oracles, VoxelGrid stages listed in voxel_literal in the container's order"""
    samplers = samplers or {}
    r = np.ascontiguousarray(np.asarray(cloud, F32)[:, :5])
    index = np.arange(len(r), dtype=np.int32)
    for k, (name, params) in enumerate(filters):
        if len(r) == 0:
            break
        if name == "VoxelGrid" and k in voxel_literal:
            voxel = F32(params["voxel_size"])
            kept, _ = CM.voxel_keys(r, voxel)
            rows = np.flatnonzero(kept)
            finite = np.ascontiguousarray(r[rows])           # the oracle leaves lround(NaN) undefined
            first = U.order_points(finite, voxel)
            _, r = O.voxel_grid_filter(finite, voxel, order_mode=1)
            index = index[rows[first]]
        elif name == "RandomSampler" and samplers.get(k, (0, 0))[0] == OM.MT19937:
            keep = OM.sampler_flags(len(r), F32(params.get("sampling_rate", 1.0)), samplers[k][1])
            r, index = r[keep], index[keep]
        else:
            r, index = CM.oracle_stage(name, params, r, index, seed)
        r, index = np.ascontiguousarray(r, F32), np.asarray(index, np.int32)
    return r, index


class Chain(G.Chain):
    """test_gpu_filter_chain_all.Chain with its VoxelGrid stages in `voxel_literal` set to UNORDERED_MAP and its
    RandomSamplers in `samplers` set to (mode, seed)"""

    def __init__(self, filters, voxel_literal=(), samplers=None):
        super().__init__(filters, all_filters=True)
        for k in voxel_literal:
            assert self.lib.sm_filter_chain_set_voxel_order(self.h, k, int(UMAP)) == 0
        for k, (mode, seed) in (samplers or {}).items():
            assert self.lib.sm_filter_chain_set_random_sampler(self.h, k, mode, seed) == 0


VG = lambda size: ("VoxelGrid", dict(voxel_size=size))                # noqa: E731
RS = lambda rate: ("RandomSampler", dict(sampling_rate=rate))         # noqa: E731


@pytest.mark.parametrize("voxel", [0.1, 0.4])
def test_chain_voxel_grid_then_mt19937_sampler(scan, voxel):
    filters = [VG(voxel), RS(0.5)]
    samplers = {1: (OM.MT19937, 77)}
    want = literal_chain(filters, scan, {0}, samplers)
    c = Chain(filters, {0}, samplers)
    G.same(c.run(scan), want)
    G.same(c.run_device(scan), want)
    import torch
    G.same(c.run_device(scan, 32, torch.cuda.Stream()), want)
    assert 0 < len(want[1]) < len(scan)
    # the order decides the sampler's keep set: the ascending chain keeps other records
    asc = Chain(filters, (), samplers).run(scan)
    assert asc[0].tobytes() != want[0].tobytes()


def test_chain_between_predicates(scan):
    filters = [("Range", dict(min_range=5.0)), VG(0.2), ("AxisRange", dict(min=-1.0))]
    want = literal_chain(filters, scan, {1})
    c = Chain(filters, {1})
    G.same(c.run(scan), want)
    G.same(c.run_device(scan), want)
    G.same(c.run(scan, 32), want)
    # ascending again from the next run on
    assert c.lib.sm_filter_chain_set_voxel_order(c.h, 1, 0) == 0
    G.same(c.run(scan), G.oracle(filters, scan))


def test_chain_with_non_finite_points(scan):
    dirty = scan.copy()
    dirty[[3, 900, 40000], [0, 1, 2]] = [np.nan, np.inf, -np.inf]
    filters = [VG(0.1)]
    G.same(Chain(filters, {0}).run(dirty), literal_chain(filters, dirty, {0}))


def test_setter_errors_leave_the_chain_unchanged(scan):
    filters = [("Range", dict(min_range=5.0)), VG(0.2)]
    c = Chain(filters, {1})
    want = c.run(scan)
    lib = c.lib
    for k, order in ((0, 1), (2, 1), (-1, 1), (1, 2), (1, -1)):
        assert lib.sm_filter_chain_set_voxel_order(c.h, k, order) == -1
    assert lib.sm_filter_chain_set_voxel_order(None, 1, 1) == -1
    G.same(c.run(scan), want)
    G.same(want, literal_chain(filters, scan, {1}))


def test_python_factory(scan):
    f = smb.Factory()
    f.SetAllFilters(True)
    f.InitFromXmlText('<filters><filter name="VoxelGrid"><param type="1" name="voxel_size">0.2</param></filter>'
                      '<filter name="RandomSampler"><param type="1" name="sampling_rate">0.5</param></filter>'
                      '</filters>')
    f.SetVoxelOrder(0, UMAP)
    f.SetRandomSampler(1, smb.RandomSamplerMode.MT19937, 5)
    with pytest.raises(ValueError):
        f.SetVoxelOrder(1, UMAP)
    with pytest.raises(ValueError):
        f.SetVoxelOrder(0, 7)
    f.SetInputCloud(scan)
    out = f.Filter()
    want = literal_chain([VG(0.2), RS(0.5)], scan, {0}, {1: (OM.MT19937, 5)})
    assert out.points.tobytes() == want[0].tobytes()
    assert np.array_equal(f.Inliers(), want[1])


# ---- the submap target end to end ------------------------------------------------------------------------------------
def test_submap_target_and_icp_fast_match_the_reference(sub500k):
    """Submap::InsertFrame (builder/submap.cc:144-161) at its default 0.1 m: VoxelGrid in the container's order, then
    CalculateNormals in std::nth_element's order, against the literal order fed to the oracle (tie_mode 1)"""
    _, voxels = O.voxel_grid_filter(sub500k, 0.1, order_mode=1)
    got = smb.VoxelGridFilter(sub500k, 0.1, order=UMAP)
    assert got.tobytes() == voxels.tobytes()
    tp, tn = O.calculate_normals(voxels[:, :3].astype(np.float64), tie_mode=1)
    g = smb.CalculateNormals(got[:, :3].astype(np.float64), order=smb.NormalsOrder.NTH_ELEMENT)
    assert g.points.tobytes() == tp.tobytes() and g.normals.tobytes() == tn.tobytes()
    # the ascending order gives another target
    a = smb.CalculateNormals(smb.VoxelGridFilter(sub500k, 0.1)[:, :3].astype(np.float64),
                             order=smb.NormalsOrder.NTH_ELEMENT)
    assert a.points.tobytes() != tp.tobytes()
    src = scenes.full_size_pair(0)[0]
    m = smb.IcpFast()
    m.SetInputSource(smb.EigenCloud(src)); m.SetInputTarget(g)
    ok, res = m.Align(np.eye(4))
    o = O.icp_fast_align(src, tp, tn)
    assert ok and o["rc"] == 1
    assert m.GetAlignInfo()["iterations"] == o["iterations"]
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= 1e-4 and dr <= 1e-4, (dt, dr)


# ---- VoxelGridFilterB200 and FilterChainB200 through tests/cpp/voxel_order_adapter_run.cc ----------------------------
@pytest.mark.parametrize("order", [0, 1])
def test_adapter(tmp_path, sub60k, order):
    exe = adapter_exe(tmp_path, "voxel_order_adapter_run")
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    voxel, seed = 0.2, 2 ** 31 - 1
    with open(src, "wb") as f:
        f.write(struct.pack("<ifIq", order, voxel, seed, len(sub60k)))
        f.write(np.ascontiguousarray(sub60k).tobytes())
    r = subprocess.run([exe, src, dst], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = open(dst, "rb").read()
    m = struct.unpack_from("<q", raw)[0]
    got = np.frombuffer(raw, F32, 5 * m, 8).reshape(m, 5)
    _, want = O.voxel_grid_filter(sub60k, voxel, order_mode=order)
    assert got.tobytes() == want.tobytes()
    off = 8 + 20 * m
    k = struct.unpack_from("<q", raw, off)[0]
    recs = np.frombuffer(raw, F32, 5 * k, off + 8).reshape(k, 5)
    idx = np.frombuffer(raw, np.int32, k, off + 8 + 20 * k)
    filters = [VG(voxel), RS(0.5)]
    want = literal_chain(filters, sub60k, {0} if order else set(), {1: (OM.MT19937, seed)})
    assert recs.tobytes() == want[0].tobytes() and np.array_equal(idx, want[1])
