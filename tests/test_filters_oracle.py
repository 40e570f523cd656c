"""The scan pre-processing filters without a GPU: the reference's own unit-test assertions
(pre_processors/test/test_filter_{range,axis_range,bounding_box,random_sample}.cc) on the C++ restatement, the C++
restatement against the independent numpy one on a lidar scan and on clouds built to sit on the decision borders, the
product's per-point functions compiled for the host against both, and the chain's C ABI."""
import ctypes as C

import numpy as np
import pytest

import filter_scenes as FS
import oracle_filters as OF
import pyref_filters as PF
from staticmapping_b200 import _lib
import staticmapping_b200 as smb

FLT_MAX = FS.FLT_MAX


@pytest.fixture(scope="module")
def cloud1000():
    rng = np.random.default_rng(7)
    return FS.records(rng.uniform(0.0, 100.0, (1000, 3)))


def both(name, params, cloud, **kw):
    a = OF.filter_flags(name, params, cloud, **kw).astype(bool)
    b = PF.filter_flags(name, params, cloud, **kw)
    assert np.array_equal(np.nonzero(a)[0], np.nonzero(b)[0]), name
    return a


# ---- the reference's unit tests ------------------------------------------------------------------------------------------
def test_reference_range_tests(cloud1000):
    c = cloud1000
    assert both("Range", None, c).all()
    keep = both("Range", dict(min_range=20, max_range=80), c)
    r = np.linalg.norm(c[:, :3].astype(np.float64), axis=1)
    assert 0 < keep.sum() < 1000 and (r[keep] >= 20 - 1e-4).all() and (r[keep] <= 80 + 1e-4).all()
    assert ((r[~keep] < 20 + 1e-4) | (r[~keep] > 80 - 1e-4)).all()


def test_reference_axis_range_tests(cloud1000):
    c = cloud1000
    assert both("AxisRange", None, c).all()
    for params, axis, lo, hi in [(dict(min=50), 2, 50, FLT_MAX), (dict(min=50, max=80), 2, 50, 80),
                                 (dict(min=60, max=80, axis_index=1), 1, 60, 80),
                                 (dict(min=10, max=70, axis_index=0), 0, 10, 70)]:
        keep = both("AxisRange", params, c)
        assert np.array_equal(keep, (c[:, axis] >= lo) & (c[:, axis] <= hi)) and 0 < keep.sum() < 1000
    assert not PF.valid("AxisRange", dict(min=90, max=80)) and not PF.valid("AxisRange", dict(axis_index=-1))


def test_reference_bounding_box_tests(cloud1000):
    c = cloud1000
    assert both("BoundingBoxRemoval", None, c).sum() == 0
    box = dict(min_x=0, min_y=0, min_z=0, max_x=100, max_y=100, max_z=100)
    assert both("BoundingBoxRemoval", box, c).sum() == 0
    box = dict(min_x=10, min_y=20, min_z=30, max_x=80, max_y=70, max_z=80)
    keep = both("BoundingBoxRemoval", box, c)
    k = c[keep]
    inside = (k[:, 0] >= 10) & (k[:, 0] <= 80) & (k[:, 1] >= 20) & (k[:, 1] <= 70) & (k[:, 2] >= 30) & (k[:, 2] <= 80)
    assert 0 < keep.sum() < 1000 and not inside.any()
    for bad in (dict(min_x=5, max_x=1), dict(min_y=5, max_y=5), dict(min_z=5, max_z=-5)):
        assert not PF.valid("BoundingBoxRemoval", bad)
        with pytest.raises(OF.CheckFailed):
            OF.filter_flags("BoundingBoxRemoval", bad, c)
        with pytest.raises(PF.CheckFailed):
            PF.filter_flags("BoundingBoxRemoval", bad, c)


def test_reference_random_sampler_tests(cloud1000):
    assert both("RandomSampler", dict(sampling_rate=1.0), cloud1000).all()
    assert not PF.valid("RandomSampler", dict(sampling_rate=1.5)) and not PF.valid("RandomSampler", dict(sampling_rate=-0.1))
    keep = both("RandomSampler", dict(sampling_rate=0.3), cloud1000, seed=9)
    assert abs(keep.sum() - 300) <= 3 * np.sqrt(1000 * 0.3 * 0.7)


# ---- C++ restatement vs numpy restatement --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lidar():
    return FS.scan(n_az=625)


@pytest.mark.parametrize("name,params", FS.SINGLE, ids=[f"{n}{i}" for i, (n, _) in enumerate(FS.SINGLE)])
def test_restatements_agree_on_a_scan(lidar, name, params):
    keep = both(name, params, lidar)
    assert 0 < keep.sum() < len(lidar)


@pytest.mark.parametrize("filters", [FS.CHAIN_SCAN, FS.CHAIN_MATCHER], ids=["scan", "matcher"])
def test_restated_chains_agree(lidar, filters):
    ra, ia = OF.chain(filters, lidar, seed=5)
    rb, ib = PF.chain(filters, lidar, seed=5)
    assert np.array_equal(ia, ib) and ra.tobytes() == rb.tobytes() and 0 < len(ia) < len(lidar)
    assert np.all(np.diff(ia) > 0) and ra.tobytes() == lidar[ia].tobytes()


def test_predicate_edges():
    c = FS.predicate_edges()
    keep = both("Range", dict(min_range=5, max_range=60), c)
    assert keep[0] and keep[4] and keep[5] and not keep[2] and not keep[10] and not keep[13]   # on min / max: in; NaN: out
    keep = both("AxisRange", dict(min=-2, max=2), c)
    assert keep[6] and keep[7] and keep[12] and not keep[1]                                  # a NaN z is kept
    keep = both("AxisRange", dict(min=-10, max=10, axis_index=0), c)
    assert keep[8] and keep[9] and keep[10] and not keep[13]
    keep = both("BoundingBoxRemoval", dict(min_x=-5, max_x=5, min_y=-5, max_y=5, min_z=-3, max_z=3), c)
    assert not keep[15] and keep[16] and not keep[17] and keep[10] and keep[13]              # closed box; NaN stays
    both("BoundingBoxRemoval", None, c)


def test_range_image_edges():
    for c in FS.range_image_edges():
        both("RangeImage", None, c)
    fwd, rev = FS.range_image_edges()
    px = OF.pixels(None, fwd)
    assert tuple(px[0]) != (-1, -1) and tuple(px[1]) == (-1, -1) and tuple(px[2]) == (-1, -1)   # d_xy 0.01 in, below out
    assert px[3][0] == 0 and px[4][0] == -1                  # a row value of -0.5 truncates to row 0, -1.5 is out
    assert px[5][0] == 39 and px[6][0] == -1
    assert px[7][1] == 0 and px[8][1] == 0                   # column W wraps to 0
    keep = OF.filter_flags("RangeImage", None, fwd).astype(bool)
    assert keep[7] and not keep[8] and keep[9] and not keep[10]
    keep_r = OF.filter_flags("RangeImage", None, rev).astype(bool)[::-1]
    assert keep_r[8] and not keep_r[7] and keep_r[10] and not keep_r[9]
    for name in ("vertical_line_num", "horizontal_line_num"):
        with pytest.raises(ValueError):
            OF.filter_flags("RangeImage", {name: 0}, fwd)


def test_ground_removal2_edges():
    scenes = FS.ground_edges()
    stages = {}
    for key, c in scenes.items():
        keep = both("GroundRemoval2", FS.GROUND, c)
        stages[key] = (OF.gr2_stages(FS.GROUND, c), keep)
    st, keep = stages["min_drops"]
    n = len(scenes["min_drops"])
    assert st["member"][n - 4] and st["member"][n - 3] and st["member"][n - 2] and not st["member"][n - 1]
    st, keep = stages["empty_and_last_bin"]
    assert st["n_lines"][10] == 0 and st["n_lines"][11] == 0 and st["n_lines"][9] >= 1 and st["n_lines"][13] >= 1
    st, keep = stages["long_line_break"]
    # segment 20: the far part lies 0.3 above the extrapolation, the long-line rule ends the line at 19.5 m and no second
    # line starts; segment 21: 0.02 above, one line runs through to 39.5 m
    assert st["n_lines"][20] == 1 and st["n_lines"][21] == 1
    assert abs(st["lines"][20, 0, 2] - 19.5) < 1e-3 and abs(st["lines"][21, 0, 2] - 39.5) < 1e-3
    st, keep = stages["on_the_line"]
    m = len(scenes["on_the_line"])
    assert keep[m - 2] and not keep[m - 1]                   # distance exactly 0: kept; 0.05 away: ground
    st, keep = stages["neighbour_only"]
    m = len(scenes["neighbour_only"])
    assert st["n_lines"][41] == 0 and not keep[m - 2] and keep[m - 1]
    st, keep = stages["plus_k_first"]
    c = scenes["plus_k_first"]
    lone = [i for i in range(len(c)) if st["cell"][i] // 200 in (50, 70)]
    assert len(lone) == 2 and not keep[lone[0]] and keep[lone[1]]     # +5 is asked before -5
    st, keep = stages["wrap_and_nan"]
    m = len(scenes["wrap_and_nan"])
    assert not keep[m - 4] and keep[m - 3:].all()


def test_line_fit_restatements_agree():
    rng = np.random.default_rng(3)
    for n in (2, 3, 4, 7, 30, 199):
        d = np.sort(rng.uniform(1, 80, n)).astype(np.float32)
        z = (-1.7 + 0.02 * d + rng.normal(0, 0.02, n)).astype(np.float32)
        a, b = OF.fit_line(d, z), PF.fit_line(np.stack([d, z], 1))
        assert a[0] == b[0] and a[1] == b[1], n


# ---- the product's host builds -------------------------------------------------------------------------------------------
class Chain:
    def __init__(self, filters=(), device=0):
        self.lib = _lib.lib()
        self.h = C.c_void_p()
        assert self.lib.sm_filter_chain_create(device, C.byref(self.h)) == 0
        for name, params in filters:
            i = self.lib.sm_filter_chain_add(self.h, name.encode())
            assert i >= 0, name
            for k, v in (params or {}).items():
                t = 0 if k in PF.INT_PARAMS else 1
                assert self.lib.sm_filter_chain_set_param(self.h, i, k.encode(), t, repr(v).encode()) == 0, k

    def __del__(self):
        self.lib.sm_filter_chain_destroy(self.h)

    def host(self, filter_index, op, cloud):
        r = OF.records(cloud)
        iout = np.zeros((len(r), 2 if op else 1), np.int32)
        fout = np.zeros(len(r), np.float32)
        assert self.lib.sm_debug_filter_host(self.h, filter_index, op, r.ctypes.data, len(r), iout.ctypes.data,
                                             fout.ctypes.data) == 0
        return iout, fout


def test_host_hooks_match_the_restatements(lidar):
    clouds = [lidar, FS.predicate_edges()] + FS.range_image_edges() + list(FS.ground_edges().values())
    ch = Chain(FS.SINGLE)
    for c in clouds:
        for i, (name, params) in enumerate(FS.SINGLE):
            if name in ("Range", "AxisRange", "BoundingBoxRemoval", "RandomSampler"):
                keep, _ = ch.host(i, 0, c)
                assert np.array_equal(keep[:, 0].astype(bool), both(name, params, c)), name
            elif name == "RangeImage":
                px, _ = ch.host(i, 1, c)
                assert np.array_equal(px, OF.pixels(params, c))
                row, col = PF.range_image_pixels(PF._params(name, params), OF.records(c))
                assert np.array_equal(px[:, 0], row) and np.array_equal(px[:, 1], col)
            else:
                sb, rng = ch.host(i, 2, c)
                osb, orng = OF.cells(params, c)
                assert np.array_equal(sb, osb) and rng.tobytes() == orng.tobytes()
                s, b, prng = PF.gr2_cells(PF._params(name, params), OF.records(c))
                assert np.array_equal(sb[:, 0], s) and np.array_equal(sb[:, 1], b) and rng.tobytes() == prng.tobytes()


def test_host_line_fit_and_distance_match_the_restatements():
    lib = _lib.lib()
    rng = np.random.default_rng(4)
    for n in (2, 3, 5, 12, 60, 199):
        for slope in (0.0, 0.05, -0.1):
            d = np.sort(rng.uniform(0.5, 90, n)).astype(np.float32)
            z = (-1.7 + slope * d + rng.normal(0, 0.03, n)).astype(np.float32)
            mb = np.zeros(2, np.float32)
            assert lib.sm_debug_filter_fit_host(d.ctypes.data, z.ctypes.data, n, mb.ctypes.data) == 0
            o, p = OF.fit_line(d, z), PF.fit_line(np.stack([d, z], 1))
            assert mb.tobytes() == o.tobytes() and mb[0] == p[0] and mb[1] == p[1], (n, slope)
    same = np.full(5, 3.0, np.float32)                         # a rank-deficient system: both columns parallel
    mb = np.zeros(2, np.float32)
    assert lib.sm_debug_filter_fit_host(same.ctypes.data, same.ctypes.data, 5, mb.ctypes.data) == 0
    assert mb.tobytes() == OF.fit_line(same, same).tobytes()
    lines = np.array([[2, -1.7, 10, -1.6], [9.95, -1.5, 20, -1.4]], np.float32)
    for d, z in [(5.0, -1.6), (9.99, -1.0), (10.05, -1.45), (1.95, -1.7), (1.8, -1.7), (20.2, 0.0), (np.nan, 0.0)]:
        dist = C.c_float()
        assert lib.sm_debug_filter_distance_host(lines.ctypes.data, 2, d, z, C.byref(dist)) == 0
        o = OF.vertical_distance(lines, d, z)
        p = float(PF.vertical_distance((np.float32(d), np.float32(z)), [tuple(l) for l in lines]))
        assert dist.value == o == p, (d, z)
    bad = np.array([[5, 0, 5, 0]], np.float32)
    assert lib.sm_debug_filter_distance_host(bad.ctypes.data, 1, 5.0, 0.0, C.byref(C.c_float())) == -5


# ---- the chain's C ABI and its Python mirror -----------------------------------------------------------------------------
def test_chain_abi_configuration():
    lib = _lib.lib()
    ch = Chain()
    for name in ("GroundRemoval", "StatisticRemoval", "VoxelGrid"):
        assert lib.sm_filter_chain_add(ch.h, name.encode()) == -11
        assert name.encode() in lib.sm_filter_chain_last_error(ch.h)
    assert lib.sm_filter_chain_add(ch.h, b"AxisRangeXXX") == -10
    assert lib.sm_filter_chain_add(ch.h, b"AxisRange") == 0 and lib.sm_filter_chain_add(ch.h, b"BoundingBoxRemoval") == 1
    assert lib.sm_filter_chain_validate(ch.h, 0) == 1
    assert lib.sm_filter_chain_set_param(ch.h, 0, b"min", 1, b" 90. ") == 0
    assert lib.sm_filter_chain_set_param(ch.h, 0, b"max", 1, b"80") == 0
    assert lib.sm_filter_chain_validate(ch.h, 0) == 0
    assert lib.sm_filter_chain_set_param(ch.h, 0, b"max", 0, b"95.7") == 0 and lib.sm_filter_chain_validate(ch.h, 0) == 1
    assert lib.sm_filter_chain_set_param(ch.h, 0, b"axis_index", 0, b"-1") == 0 and lib.sm_filter_chain_validate(ch.h, 0) == 0
    assert lib.sm_filter_chain_set_param(ch.h, 0, b"min_range", 1, b"1") == -10          # another filter's name
    assert lib.sm_filter_chain_set_param(ch.h, 0, b"min", -1, b"1") == -1                # a <param> without type
    assert lib.sm_filter_chain_set_param(ch.h, 5, b"min", 1, b"1") == -1
    for k, v in (("min_x", "5"), ("max_x", "1")):
        assert lib.sm_filter_chain_set_param(ch.h, 1, k.encode(), 1, v.encode()) == 0
    assert lib.sm_filter_chain_validate(ch.h, 1) == 0
    assert lib.sm_filter_chain_set_option(ch.h, b"sample_seed", b"7") == 0
    assert lib.sm_filter_chain_set_option(ch.h, b"seed", b"7") == -10
    m = C.c_int64(-1)
    buf = np.zeros((4, 5), np.float32)
    assert lib.sm_filter_chain_run(ch.h, buf.ctypes.data, 4, 16, buf.ctypes.data, C.byref(m), None) == -1
    assert lib.sm_filter_chain_run(ch.h, None, 4, 20, buf.ctypes.data, C.byref(m), None) == -1


def test_chain_without_a_device():
    lib = _lib.lib()
    if lib.sm_device_count() > 0:
        pytest.skip("GPU present")
    ch = Chain(FS.CHAIN_SCAN)
    c = FS.predicate_edges()
    out = np.empty_like(c)
    m = C.c_int64(-1)
    assert lib.sm_filter_chain_run(ch.h, c.ctypes.data, len(c), 20, out.ctypes.data, C.byref(m), None) == -20
    assert lib.sm_filter_chain_run(ch.h, c.ctypes.data, 0, 20, out.ctypes.data, C.byref(m), None) == -20
    assert lib.sm_filter_chain_run_device(ch.h, c.ctypes.data, len(c), 20, out.ctypes.data, C.byref(m), None, None) == -20
    f = smb.Factory()
    f.SetInputCloud(c)
    with pytest.raises(RuntimeError):
        f.Filter()


def test_factory_xml():
    f = smb.Factory()
    f.InitFromXmlText('<filters><filter name="Range"><param type="1" name="min_range"> 5. </param></filter>'
                      '<filter name="Nonsense"/><filter name="AxisRange"><param type="1" name="min"> -2. </param></filter>'
                      '<filter name="RandomSampler"><param type="1" name="sampling_rate"> 0.5 </param></filter></filters>')
    assert f.filter_names == ["Range", "AxisRange", "RandomSampler"] and f.messages == ["Nonsense not supported yet."]
    assert all(f.ConfigsValid(i) for i in range(3))
    for bad in ('<filters><filter name="AxisRange"><param type="1" name="AxisRangeXXX">1</param></filter></filters>',
                '<filters><filter name="Range"><param name="min_range">1</param></filter></filters>',
                '<filters><filter name="VoxelGrid"/></filters>'):
        with pytest.raises(smb.CheckFailure):
            smb.Factory().InitFromXmlText(bad)
