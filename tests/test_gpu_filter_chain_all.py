"""GroundRemoval, StatisticRemoval and VoxelGrid as stages of the filter chain on an H100 (the chain option all_filters):
one-filter chains against the filters' own entry points bit for bit, chains of the predicates and the new stages in
several orders against the composition of the C++ restatements (chain_all_model) bit for bit, chains that also hold
RangeImage or GroundRemoval2 stage by stage, both entries at strides 20 and 32 and sizes around the compaction tile up
to 1.2 M points, two chains on two streams, reuse, every new error with nothing written, the option on with the
existing kinds only, and the Python Factory."""
import ctypes as C

import numpy as np
import pytest

import chain_all_model as M
import filter_scenes as FS
import ground_removal_scenes as GS
import oracle_filters as OF
from staticmapping_b200 import _lib
import staticmapping_b200 as smb

pytestmark = pytest.mark.gpu

F32 = np.float32
INT_PARAMS = {"axis_index", "vertical_line_num", "horizontal_line_num", "bin_num", "segment_num", "thread_num",
              "point_num_meank", "min_point_num_in_voxel"}
ATAN2 = {"RangeImage", "GroundRemoval2"}


def _strided(rec, stride):
    buf = np.full((len(rec), stride // 4), 9.0, F32)
    buf[:, :5] = rec
    return buf


class Chain:
    def __init__(self, filters=(), seed=None, all_filters=True):
        self.lib = _lib.lib()
        self.h = C.c_void_p()
        assert self.lib.sm_filter_chain_create(0, C.byref(self.h)) == 0
        if all_filters:
            assert self.lib.sm_filter_chain_set_option(self.h, b"all_filters", b"1") == 0
        for name, params in filters:
            i = self.lib.sm_filter_chain_add(self.h, name.encode())
            assert i >= 0, name
            for k, v in (params or {}).items():
                t, text = (0, str(int(v))) if k in INT_PARAMS else (1, "%.9g" % v)
                assert self.lib.sm_filter_chain_set_param(self.h, i, k.encode(), t, text.encode()) == 0, k
        if seed is not None:
            assert self.lib.sm_filter_chain_set_option(self.h, b"sample_seed", str(seed).encode()) == 0

    def __del__(self):
        self.lib.sm_filter_chain_destroy(self.h)

    def error(self):
        return self.lib.sm_filter_chain_last_error(self.h).decode()

    def run(self, cloud, stride=20, expect=0):
        n = len(cloud)
        src = _strided(cloud, stride)
        out = np.full((max(n, 1), 5), -7.0, F32)
        idx = np.full(max(n, 1), -7, np.int32)
        m = C.c_int64(-1)
        rc = self.lib.sm_filter_chain_run(self.h, src.ctypes.data, n, stride, out.ctypes.data, C.byref(m),
                                          idx.ctypes.data)
        assert rc == expect, (rc, self.error())
        if rc != 0:
            assert m.value == 0 and np.all(out == -7.0) and np.all(idx == -7)      # nothing written
            return None, None
        return out[:m.value], idx[:m.value]

    def run_device(self, cloud, stride=20, stream=None, expect=0):
        import torch
        n = len(cloud)
        d_in = torch.from_numpy(_strided(cloud, stride)).cuda()
        d_out = torch.full((max(n, 1), 5), -7.0, dtype=torch.float32, device="cuda")
        d_idx = torch.full((max(n, 1),), -7, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        m = C.c_int64(-1)
        rc = self.lib.sm_filter_chain_run_device(self.h, d_in.data_ptr(), n, stride, d_out.data_ptr(), C.byref(m),
                                                 d_idx.data_ptr(), None if stream is None else stream.cuda_stream)
        assert rc == expect, (rc, self.error())
        if rc != 0:
            assert bool((d_out == -7.0).all()) and bool((d_idx == -7).all())        # nothing written
            return None, None
        return d_out[:m.value].cpu().numpy(), d_idx[:m.value].cpu().numpy()


def oracle(filters, cloud, seed=1):
    return M.chain(filters, cloud, seed=seed)


def same(got, want):
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1]), (len(got[1]), len(want[1]))


@pytest.fixture(scope="module")
def scan():
    return FS.scan()            # 120 000 points


# ---- one-filter chains against the own entry points ----------------------------------------------------------------
def own_ground_removal(rec, params):
    lib = _lib.lib()
    h = C.c_void_p()
    assert lib.sm_ground_removal_create(0, C.byref(h)) == 0
    try:
        for k, v in params.items():
            t, text = (0, str(int(v))) if k in INT_PARAMS else (1, "%.9g" % v)
            assert lib.sm_ground_removal_set_param(h, k.encode(), t, text.encode()) == 0
        out, idx, m = np.empty_like(rec), np.empty(len(rec), np.int32), C.c_int64(0)
        assert lib.sm_ground_removal_run(h, rec.ctypes.data, len(rec), 20, out.ctypes.data, C.byref(m),
                                         idx.ctypes.data) == 0
        return out[:m.value], idx[:m.value]
    finally:
        lib.sm_ground_removal_destroy(h)


def own_statistic_removal(rec, params):
    f = smb.StatisticRemoval()
    for k, v in params.items():
        f.SetParam(k, 0 if k in INT_PARAMS else 1, str(int(v)) if k in INT_PARAMS else "%.9g" % v)
    f.SetInputCloud(rec)
    return f.Filter().points, f.Inliers()


def own_voxel_grid(rec, params):
    return smb.VoxelGridFilter(rec, params["voxel_size"]), M.voxel_first_members(rec, params["voxel_size"])


OWN = {"GroundRemoval": own_ground_removal, "StatisticRemoval": own_statistic_removal, "VoxelGrid": own_voxel_grid}
SINGLE = [("GroundRemoval", M.GR_DEFAULT), ("GroundRemoval", dict(min_point_num_in_voxel=3, leaf_size=0.2,
                                                                  height_threshold=0.1)),
          ("StatisticRemoval", M.SR_DEFAULT), ("StatisticRemoval", dict(point_num_meank=8, std_mul=0.5)),
          ("VoxelGrid", M.VG_DEFAULT), ("VoxelGrid", dict(voxel_size=0.4))]


@pytest.mark.parametrize("name,params", SINGLE, ids=[f"{n}{i}" for i, (n, _) in enumerate(SINGLE)])
def test_one_filter_chain_equals_its_own_entry_point(scan, name, params):
    want = OWN[name](scan, params)
    ch = Chain([(name, params)])
    same(ch.run(scan), want)
    same(ch.run_device(scan, stride=32), want)
    assert 0 < len(want[1]) < len(scan)


# ---- mixed chains against the oracle composition ---------------------------------------------------------------------
GR = ("GroundRemoval", M.GR_DEFAULT)
SR = ("StatisticRemoval", dict(point_num_meank=10, std_mul=1.0))
VG = ("VoxelGrid", dict(voxel_size=0.2))
SAMPLER = ("RandomSampler", dict(sampling_rate=0.5))
AXIS = ("AxisRange", dict(min=-1.5))
RANGE = ("Range", dict(min_range=3.0))
MIXED = {
    "voxel_sampler": [VG, SAMPLER],
    "ground_statistic_axis": [GR, SR, AXIS],
    "statistic_first": [SR] + FS.CHAIN_SCAN,
    "statistic_last": FS.CHAIN_SCAN + [SR],
    "voxel_middle": [RANGE, VG, AXIS],
    "ground_last": FS.CHAIN_SCAN + [GR],
    "all_three": [VG, SR, ("GroundRemoval", dict(min_point_num_in_voxel=2, leaf_size=1.0, height_threshold=0.3))],
    "ground_voxel_sampler": [GR, ("VoxelGrid", dict(voxel_size=0.5)), SAMPLER],
}


@pytest.mark.parametrize("name", list(MIXED))
def test_mixed_chains_equal_the_oracle_composition(scan, name):
    filters = MIXED[name]
    want = oracle(filters, scan, seed=5)
    assert len(want[1]) > 0
    ch = Chain(filters, seed=5)
    same(ch.run(scan), want)
    same(ch.run(scan, stride=32), want)
    for stride in (20, 32):
        same(ch.run_device(scan, stride), want)


# ---- chains that also hold RangeImage or GroundRemoval2: stage by stage ----------------------------------------------
STAGED = {
    "matcher_then_voxel": FS.CHAIN_MATCHER + [VG],
    "gr2_statistic_range_image": [("GroundRemoval2", FS.GROUND), SR, ("RangeImage", FS.RANGE_IMAGE)],
    "voxel_range_image_ground": [VG, ("RangeImage", FS.RANGE_IMAGE), GR],
    "range_image_statistic_voxel": [("RangeImage", FS.RANGE_IMAGE), SR, ("VoxelGrid", dict(voxel_size=0.5))],
}


@pytest.mark.parametrize("name", list(STAGED))
def test_chains_with_atan2_stages_stage_by_stage(scan, name):
    """each oracle stage reads the GPU's previous-stage output (the chain cut after that stage); the new stages and the
    predicates must match exactly, RangeImage and GroundRemoval2 within 0.1 % of the scan"""
    filters = STAGED[name]
    prev = (scan, np.arange(len(scan), dtype=np.int32))
    for k, (fname, params) in enumerate(filters):
        got = Chain(filters[:k + 1], seed=5).run(scan)
        want = M.oracle_stage(fname, params, np.ascontiguousarray(prev[0]), prev[1], seed=5)
        if fname in ATAN2:
            differ = np.setxor1d(got[1], want[1])
            assert len(differ) < 0.001 * len(scan), (fname, len(differ))
            row = {int(i): r for r, i in enumerate(prev[1])}
            assert got[0].tobytes() == np.ascontiguousarray(prev[0][[row[int(i)] for i in got[1]]]).tobytes()
        else:
            same(got, want)
        prev = got
    same(Chain(filters, seed=5).run_device(scan, stride=32), prev)


# ---- entry points and sizes --------------------------------------------------------------------------------------------
def tiled(scan, copies):
    """copies of the scan side by side, 200 m apart"""
    parts = []
    for c in range(copies):
        p = scan.copy()
        p[:, 0] += F32(200.0 * c)
        parts.append(p)
    return np.concatenate(parts)


@pytest.mark.parametrize("n", [1, 2, 2047, 2048, 2049, 4095, 4097, 65537])
def test_sizes_around_the_tile(scan, n):
    cloud = np.ascontiguousarray(scan[:n])
    for filters in ([VG, SAMPLER], [AXIS, GR, ("VoxelGrid", dict(voxel_size=0.5))]):
        want = oracle(filters, cloud, seed=5)
        ch = Chain(filters, seed=5)
        same(ch.run(cloud), want)
        same(ch.run_device(cloud, stride=32), want)
    if n > 64:
        want = oracle([GR, SR, AXIS], cloud, seed=5)
        same(Chain([GR, SR, AXIS], seed=5).run(cloud, stride=32), want)


def test_one_point_two_million_points(scan):
    cloud = tiled(scan, 10)
    assert len(cloud) == 1_200_000
    for filters in ([VG, SAMPLER], [GR, SR, AXIS]):
        want = oracle(filters, cloud, seed=5)
        ch = Chain(filters, seed=5)
        same(ch.run(cloud), want)
        same(ch.run_device(cloud, stride=32), want)


# ---- streams and reuse -------------------------------------------------------------------------------------------------
def test_two_streams_and_reuse(scan):
    import torch
    fa, fb = MIXED["ground_statistic_axis"], MIXED["voxel_sampler"]
    a, b = Chain(fa, seed=5), Chain(fb, seed=5)
    want_a, want_b = a.run(scan), b.run(scan)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    for _ in range(2):
        same(a.run_device(scan, stream=sa), want_a)
        same(b.run_device(scan, stride=32, stream=sb), want_b)
    big = tiled(scan, 4)
    small = np.ascontiguousarray(scan[:5000])
    want_big, want_small = oracle(fa, big, seed=5), oracle(fa, small, seed=5)
    same(a.run(big), want_big)                        # large -> small -> large on one chain
    same(a.run(small), want_small)
    same(a.run_device(big, stride=32), want_big)
    same(b.run(small), oracle(fb, small, seed=5))


# ---- errors ---------------------------------------------------------------------------------------------------------------
def _errors(scan):
    far = FS.records(np.array([[0.0, 0.0, 0.0]] * 5 + [[209716.0, 0.0, 0.0]] * 5))   # 2^21 + 8 voxels of 0.1 m
    gr_span = GS.span_limit()[-1][0]
    few = FS.records(np.concatenate([np.stack([np.arange(10.0)] * 3, 1), np.full((500, 3), -50.0)]))   # 10 pass z >= -1
    return [
        ([("StatisticRemoval", dict(point_num_meank=0))], scan, -1, "point_num_meank"),
        ([RANGE, ("StatisticRemoval", dict(point_num_meank=64))], scan, -1, "point_num_meank"),
        ([("StatisticRemoval", dict(point_num_meank=30))], scan[:20], -5, "Check failed"),
        ([("AxisRange", dict(min=-1.0)), ("StatisticRemoval", dict(point_num_meank=30))], few, -5, "Check failed"),
        ([("VoxelGrid", dict(voxel_size=1e-6))], scan, -1, "voxel_size"),
        ([RANGE, ("VoxelGrid", dict(voxel_size=0.0))], scan, -1, "voxel_size"),
        ([("VoxelGrid", dict(voxel_size=0.1))], far, -1, "span"),
        ([AXIS, ("VoxelGrid", dict(voxel_size=0.1)), SAMPLER], far, -1, "span"),
        ([("GroundRemoval", dict(min_point_num_in_voxel=1, leaf_size=1e-3, height_threshold=0.15))], gr_span, -1,
         "span"),
        ([AXIS, ("GroundRemoval", dict(min_point_num_in_voxel=1, leaf_size=1e-3, height_threshold=0.15))], gr_span, -1,
         "span"),
    ]


def test_errors_write_nothing(scan):
    for filters, cloud, rc, message in _errors(scan):
        cloud = np.ascontiguousarray(cloud)
        if rc == -5:
            with pytest.raises(M.CheckFailed):
                oracle(filters, cloud)
        ch = Chain(filters)
        ch.run(cloud, expect=rc)
        assert message in ch.error(), (filters, ch.error())
        ch.run_device(cloud, stride=32, expect=rc)
        assert message in ch.error()


def test_an_empty_intermediate_cloud_ends_the_chain(scan):
    ch = Chain([("Range", dict(min_range=1e9)), ("StatisticRemoval", dict(point_num_meank=0)), VG])
    # the invalid K is refused before any work, even behind a stage that empties the cloud
    ch.run(scan, expect=-1)
    ch = Chain([("Range", dict(min_range=1e9)), SR, VG, GR])
    out, idx = ch.run(scan)
    assert len(out) == 0 and len(idx) == 0


# ---- the option on, existing kinds only ----------------------------------------------------------------------------------
@pytest.mark.parametrize("filters", [[f] for f in FS.SINGLE] + [FS.CHAIN_SCAN, FS.CHAIN_MATCHER],
                         ids=[f"{n}{i}" for i, (n, _) in enumerate(FS.SINGLE)] + ["chain_scan", "chain_matcher"])
def test_the_option_leaves_existing_chains_unchanged(scan, filters):
    on, off = Chain(filters, seed=5, all_filters=True), Chain(filters, seed=5, all_filters=False)
    want = off.run(scan)
    same(on.run(scan), want)
    same(on.run_device(scan, stride=32), off.run_device(scan, stride=32))
    assert np.all(np.diff(want[1]) > 0)


# ---- the Python Factory --------------------------------------------------------------------------------------------------
def test_factory_inliers_and_outliers(scan):
    f = smb.Factory()
    f.SetAllFilters(True)
    f.SetSampleSeed(5)
    f.InitFromXmlText('<filters><filter name="GroundRemoval"/>'
                      '<filter name="VoxelGrid"><param type="1" name="voxel_size">0.5</param></filter>'
                      '<filter name="RandomSampler"><param type="1" name="sampling_rate">0.5</param></filter></filters>')
    f.SetInputCloud(scan)
    out = f.Filter()
    want = oracle(MIXED["ground_voxel_sampler"], scan, seed=5)
    assert out.points.tobytes() == want[0].tobytes() and np.array_equal(f.Inliers(), want[1])
    assert np.array_equal(f.Outliers(), np.setdiff1d(np.arange(len(scan)), want[1]).astype(np.int32))
    g = smb.Factory()
    g.SetAllFilters(True)
    g.InitFromXmlText('<filters><filter name="Range"><param type="1" name="min_range">5</param></filter></filters>')
    g.SetInputCloud(scan)
    g.Filter()
    _, keep = OF.chain([("Range", dict(min_range=5.0))], scan)
    assert np.array_equal(g.Inliers(), keep) and np.array_equal(g.Outliers(), np.setdiff1d(np.arange(len(scan)), keep))
