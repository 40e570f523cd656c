"""GroundRemoval, StatisticRemoval and VoxelGrid as stages of the filter chain (the chain option all_filters), without a
GPU: the option's C ABI and its Python and XML mirror, and whole chains composed stage by stage from the C++
restatements against the same chains composed from the numpy ones, each new filter first, in the middle and last."""
import ctypes as C

import numpy as np
import pytest

import chain_all_model as M
import filter_scenes as FS
import ground_removal_scenes as GS
import statistic_removal_scenes as SS
from staticmapping_b200 import _lib
import staticmapping_b200 as smb

NEW = [("GroundRemoval", M.GR_DEFAULT), ("StatisticRemoval", M.SR_DEFAULT), ("VoxelGrid", M.VG_DEFAULT)]


class Chain:
    def __init__(self):
        self.lib = _lib.lib()
        self.h = C.c_void_p()
        assert self.lib.sm_filter_chain_create(0, C.byref(self.h)) == 0

    def __del__(self):
        self.lib.sm_filter_chain_destroy(self.h)

    def add(self, name):
        return self.lib.sm_filter_chain_add(self.h, name.encode())

    def option(self, name, text):
        return self.lib.sm_filter_chain_set_option(self.h, name.encode(), text.encode())

    def param(self, i, name, ptype, text):
        return self.lib.sm_filter_chain_set_param(self.h, i, name.encode(), ptype, text.encode())


# ---- the option's C ABI -----------------------------------------------------------------------------------------------
def test_add_follows_the_option():
    ch = Chain()
    for name, _ in NEW:
        assert ch.add(name) == -11 and name.encode() in ch.lib.sm_filter_chain_last_error(ch.h)
    assert ch.add("Range") == 0
    assert ch.option("all_filters", "1") == 0
    assert [ch.add(name) for name, _ in NEW] == [1, 2, 3]
    assert ch.add("Nonsense") == -10 and ch.add("RandomSamplerWithPlaneDetect") == -10
    assert ch.option("all_filters", "0") == 0
    for name, _ in NEW:
        assert ch.add(name) == -11
    assert ch.add("AxisRange") == 4                                 # the filters added before stay
    assert ch.option("all_filters", "1") == 0 and ch.add("VoxelGrid") == 5
    assert ch.option("sample_seed", "3") == 0 and ch.option("all_filter", "1") == -10
    assert ch.lib.sm_filter_chain_set_option(ch.h, b"all_filters", None) == -1


def test_set_param_names_and_errors():
    ch = Chain()
    assert ch.option("all_filters", "1") == 0
    gr, sr, vg = (ch.add(name) for name, _ in NEW)
    for i, name, ptype, text in ((gr, "min_point_num_in_voxel", 0, "4"), (gr, "leaf_size", 1, "0.5"),
                                 (gr, "height_threshold", 1, "0.2"), (sr, "point_num_meank", 0, "8"),
                                 (sr, "std_mul", 1, "2.5"), (vg, "voxel_size", 1, " 0.25 "), (vg, "voxel_size", 0, "1")):
        assert ch.param(i, name, ptype, text) == 0, name
    for i, name in ((gr, "voxel_size"), (sr, "leaf_size"), (vg, "leaf_size"), (vg, "min_range"), (sr, "min_range")):
        assert ch.param(i, name, 1, "1") == -10, (i, name)
        assert b"unknown param" in ch.lib.sm_filter_chain_last_error(ch.h)
    for i, name in ((gr, "leaf_size"), (sr, "std_mul"), (vg, "voxel_size")):
        assert ch.param(i, name, -1, "1") == -1                     # a <param> without a type
        assert ch.param(i, name, 2, "1") == -1


def test_voxel_grid_configs_valid():
    ch = Chain()
    assert ch.option("all_filters", "1") == 0
    vg, gr, sr = ch.add("VoxelGrid"), ch.add("GroundRemoval"), ch.add("StatisticRemoval")
    assert [ch.lib.sm_filter_chain_validate(ch.h, i) for i in (vg, gr, sr)] == [1, 1, 1]
    for text, valid in (("1e-6", 0), ("1.1e-6", 1), ("0", 0), ("-0.5", 0), ("nan", 0), ("0.1", 1), ("inf", 1)):
        assert ch.param(vg, "voxel_size", 1, text) == 0
        assert ch.lib.sm_filter_chain_validate(ch.h, vg) == valid, text
    for text in ("0", "-3", "64"):                                  # refused at run time, not by ConfigsValid
        assert ch.param(sr, "point_num_meank", 0, text) == 0 and ch.lib.sm_filter_chain_validate(ch.h, sr) == 1
    assert ch.param(gr, "leaf_size", 1, "0") == 0 and ch.lib.sm_filter_chain_validate(ch.h, gr) == 1


def test_run_without_a_device():
    lib = _lib.lib()
    if lib.sm_device_count() > 0:
        pytest.skip("GPU present")
    ch = Chain()
    assert ch.option("all_filters", "1") == 0 and ch.add("VoxelGrid") == 0
    c = FS.predicate_edges()
    out = np.empty_like(c)
    m = C.c_int64(-1)
    assert lib.sm_filter_chain_run(ch.h, c.ctypes.data, len(c), 20, out.ctypes.data, C.byref(m), None) == -20


def test_factory_xml_with_the_option():
    xml = ('<filters><filter name="Range"><param type="1" name="min_range"> 5. </param></filter>'
           '<filter name="VoxelGrid"><param type="1" name="voxel_size"> 0.3 </param></filter>'
           '<filter name="GroundRemoval"><param type="0" name="min_point_num_in_voxel">3</param></filter>'
           '<filter name="StatisticRemoval"><param type="1" name="std_mul">2</param></filter>'
           '<filter name="Nonsense"/></filters>')
    with pytest.raises(smb.CheckFailure):
        smb.Factory().InitFromXmlText(xml)                          # the refusal stays the default
    f = smb.Factory()
    f.SetAllFilters(True)
    f.InitFromXmlText(xml)
    assert f.filter_names == ["Range", "VoxelGrid", "GroundRemoval", "StatisticRemoval"]
    assert f.messages == ["Nonsense not supported yet."] and all(f.ConfigsValid(i) for i in range(4))
    f.SetAllFilters(False)
    with pytest.raises(smb.CheckFailure):
        f.InitFromXmlText('<filters><filter name="VoxelGrid"/></filters>')
    for bad in ('<filters><filter name="VoxelGrid"><param type="1" name="leaf_size">1</param></filter></filters>',
                '<filters><filter name="GroundRemoval"><param name="leaf_size">1</param></filter></filters>'):
        g = smb.Factory()
        g.SetAllFilters(True)
        with pytest.raises(smb.CheckFailure):
            g.InitFromXmlText(bad)


# ---- whole chains: the C++ restatements against the numpy ones --------------------------------------------------------
GR = ("GroundRemoval", dict(min_point_num_in_voxel=4, leaf_size=0.8, height_threshold=0.15))
SR = ("StatisticRemoval", dict(point_num_meank=8, std_mul=1.0))
VG = ("VoxelGrid", dict(voxel_size=0.4))
RANGE = ("Range", dict(min_range=2.0))
AXIS = ("AxisRange", dict(min=-1.5))
SAMPLER = ("RandomSampler", dict(sampling_rate=0.5))
BOX = ("BoundingBoxRemoval", dict(min_x=-3, max_x=3, min_y=-3, max_y=3, min_z=-3, max_z=3))
CHAINS = {
    "voxel_first": [VG, SAMPLER],
    "voxel_middle": [RANGE, VG, AXIS],
    "voxel_last": FS.CHAIN_SCAN + [VG],
    "ground_first": [GR, SR, AXIS],
    "ground_middle": [RANGE, GR, SAMPLER],
    "ground_last": FS.CHAIN_SCAN + [GR],
    "statistic_first": [SR, BOX],
    "statistic_middle": [AXIS, SR, SAMPLER],
    "statistic_last": FS.CHAIN_SCAN + [SR],
    "all_three": [SR, VG, ("GroundRemoval", dict(min_point_num_in_voxel=2, leaf_size=1.0, height_threshold=0.3))],
    "voxel_then_ground": [("VoxelGrid", dict(voxel_size=0.1)), GR, SAMPLER],
}


SCENES = ("scan", "spread", "planted", "non_finite")


@pytest.fixture(scope="module")
def scenes():
    return {"scan": FS.scan(n_az=300), "spread": GS.spread(), "planted": SS.planted()[0],
            "non_finite": SS.non_finite()}


@pytest.mark.parametrize("scene", SCENES)
@pytest.mark.parametrize("name", list(CHAINS))
def test_oracle_composition_equals_the_numpy_one(scenes, scene, name):
    cloud = scenes[scene]
    filters = CHAINS[name]
    try:
        o_rec, o_idx = M.chain(filters, cloud, seed=3)
    except M.CheckFailed:
        with pytest.raises(M.CheckFailed):
            M.chain(filters, cloud, seed=3, stage=M.pyref_stage)
        return
    p_rec, p_idx = M.chain(filters, cloud, seed=3, stage=M.pyref_stage)
    assert o_rec.tobytes() == p_rec.tobytes() and np.array_equal(o_idx, p_idx)
    voxel_or_ground = any(f in ("GroundRemoval", "VoxelGrid") for f, _ in filters)
    if not voxel_or_ground:                                         # ascending, whole input records
        assert np.all(np.diff(o_idx) > 0) and o_rec.tobytes() == np.ascontiguousarray(cloud[o_idx]).tobytes()


def test_the_compositions_carry_scan_indices():
    cloud = FS.scan(n_az=300)
    # the sampler behind a VoxelGrid keys on each voxel's first member in the scan
    vox, first = M.chain([VG], cloud)
    sampled, idx = M.chain([VG, SAMPLER], cloud, seed=3)
    keep = M.OF.filter_flags(*SAMPLER, vox, first, seed=3).astype(bool)
    assert np.array_equal(idx, first[keep]) and sampled.tobytes() == vox[keep].tobytes()
    assert np.all(vox[:, 4] == 0) and len(np.unique(first)) == len(first)
    # GroundRemoval behind a predicate: map order, each record the scan's own
    rec, idx = M.chain([RANGE, GR], cloud)
    assert rec.tobytes() == np.ascontiguousarray(cloud[idx]).tobytes() and not np.all(np.diff(idx) > 0)
    # a stage handed an empty cloud ends the chain
    rec, idx = M.chain([("Range", dict(min_range=1e9)), SR, VG], cloud)
    assert len(rec) == 0 and len(idx) == 0
    with pytest.raises(M.CheckFailed):
        M.chain([("Range", dict(min_range=1.0)), ("StatisticRemoval", dict(point_num_meank=63))], cloud[:40])
