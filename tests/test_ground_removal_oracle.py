"""GroundRemoval without a GPU: the C++ restatement (oracle/ground_removal_oracle.cc) against the numpy one
(tests/pyref_ground_removal.py) on the scan and on every scene, the product's host-compiled voxel index and voxel
decision (include/sm_b200_debug.h) against numpy, the C ABI's argument checks and the Python mirror's parsing."""
import ctypes as C

import numpy as np
import pytest

import ground_removal_scenes as S
import oracle_ground_removal as OG
import pyref_ground_removal as PR
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

F32 = np.float32


def _same(a, b):
    return (a.out.tobytes() == b.out.tobytes() and np.array_equal(a.index, b.index)
            and np.array_equal(a.inliers, b.inliers) and np.array_equal(a.outliers, b.outliers))


def _against_numpy(rec, params):
    o = OG.ground_removal(rec, *params)
    p = PR.ground_removal(rec, *params)
    assert _same(o, p), params
    assert np.array_equal(np.sort(o.index), o.inliers) and not np.any(np.isin(o.inliers, o.outliers))
    return o


def test_hand_computed():
    # leaf 1: voxel (0,0,0) flat (ground), (0,0,-1) spread 0.5 (kept), (0,0,1) flat but iz > 0 (kept), (3,0,0) too small
    z = [0.1, 0.1, -1.2, -1.7, 1.5, 1.5, 0.1]
    rec = S.records([[0.5, 0.5, z[0]], [0.2, 0.5, z[1]], [0.5, 0.5, z[2]], [0.5, 0.5, z[3]], [0.5, 0.5, z[4]],
                     [0.5, 0.5, z[5]], [3.5, 0.5, z[6]]])
    o = OG.ground_removal(rec, 2, 1.0, 0.15)
    assert o.index.tolist() == [2, 3, 4, 5] and o.out.tobytes() == rec[[2, 3, 4, 5]].tobytes()
    assert o.inliers.tolist() == [2, 3, 4, 5] and o.outliers.tolist() == [0, 1]
    # map order, not input order: (-1, ...) before (0, ...)
    o = OG.ground_removal(S.records([[0.5, 0, 2], [-1.5, 0, 2]]), 1, 1.0, 0.15)
    assert o.index.tolist() == [1, 0] and o.inliers.tolist() == [0, 1]


@pytest.mark.parametrize("leaf", [0.2, 0.8, 2.0])
def test_scan(leaf):
    o = _against_numpy(S.scan(), (10, leaf, 0.15))
    assert 0 < len(o.inliers) and 0 < len(o.outliers) and len(o.inliers) + len(o.outliers) <= 120_000


@pytest.mark.parametrize("name", sorted(S.scenes()))
def test_scenes(name):
    rec, params = S.scenes()[name]
    for p in params:
        _against_numpy(rec, p)


def test_scene_rules():
    rec, _ = S.scenes()["trunc_not_floor"]
    o = OG.ground_removal(rec, *S.DEFAULT)
    assert o.outliers.tolist() == list(range(20)) + list(range(30, 40))   # +-0.4 share a voxel; z = 0.8 is not tested
    rec, _ = S.scenes()["delta_at_threshold"]
    o = OG.ground_removal(rec, *S.DEFAULT)
    assert len(o.outliers) == len(o.inliers) > 0                      # delta == threshold: ground; one ulp above: kept
    rec, _ = S.scenes()["z_rules"]
    all_nan = np.flatnonzero(np.isnan(rec[:, 2]) & (rec[:, 0] == F32(2.1)))
    for p in S.scenes()["z_rules"][1]:
        assert np.all(np.isin(all_nan, OG.ground_removal(rec, *p).inliers))   # delta = -2e9: never ground
    assert len(OG.ground_removal(S.scan()[:0], *S.DEFAULT).index) == 0


def test_span_cases_still_run_in_the_oracle():
    for rec, leaf, _ in S.span_limit():
        _against_numpy(rec, (1, leaf, 0.15))


def _index_host(rec, leaf, stride=20):
    rec = np.ascontiguousarray(rec, F32)
    out = np.zeros((len(rec), 3), np.int32)
    assert _lib.lib().sm_debug_ground_removal_index_host(rec.ctypes.data, len(rec), stride, leaf, out.ctypes.data) == 0
    return out


def test_index_host_against_numpy():
    rng = np.random.default_rng(5)
    clouds = [S.scan()[::7], S.rounding(), S.non_finite(), S.z_rules(),
              S.records(rng.uniform(-3e9, 3e9, (2000, 3))), S.records(rng.normal(size=(2000, 3)) * 1e-3)]
    for rec in clouds:
        for leaf in (0.8, 0.1, 0.3, 2.0, 0.0, -0.8, -0.0, 1e-30, float("inf"), float("nan")):
            assert np.array_equal(_index_host(rec, leaf), PR.voxel_index(rec[:, :3], leaf)), leaf
    r = S.records([[0.4, -0.4, np.nextafter(F32(0.8), F32(0))], [0.8, -0.8, 2147483520.0], [np.nan, np.inf, 3e9]])
    assert _index_host(r, 0.8).tolist() == [[0, 0, 0], [1, -1, -2147483648], [-2147483648] * 3]
    assert _index_host(r, 1.0)[1].tolist() == [0, 0, 2147483520]


def _voxel_host(z, iz, min_points, thr):
    z = np.ascontiguousarray(z, F32)
    st = C.c_int32(-1)
    mm = np.zeros(2, F32)
    assert _lib.lib().sm_debug_ground_removal_voxel_host(z.ctypes.data, len(z), iz, min_points, thr, C.byref(st),
                                                         mm.ctypes.data) == 0
    return st.value, mm


def test_voxel_host_against_numpy():
    rng = np.random.default_rng(6)
    nan = np.nan
    cases = [[0.0, 0.15], [-0.0, 0.0], [0.0, -0.0], [nan, 0.1, nan], [nan] * 4, [-2e9, -3e9], [1e12, nan, -5e9],
             [0.1] * 9, list(rng.normal(size=50) * 0.04), [np.inf, 0.0], [-np.inf, 0.0]]
    for z in cases:
        for iz in (-2, 0, 1, -2147483648):
            for mp in (-1, 0, 1, len(z), len(z) + 1):
                for thr in (0.15, 0.0, -0.0, -0.1, nan, 1e13):
                    st, mm = _voxel_host(z, iz, mp, thr)
                    assert st == PR.voxel_status(z, iz, mp, thr), (z, iz, mp, thr)
                    if len(z) >= mp and iz <= 0:
                        zz = np.asarray(z, F32)
                        zz = zz[~np.isnan(zz)]
                        assert mm[0] == (max(F32(-1e9), zz.max()) if len(zz) else F32(-1e9))
                        assert mm[1] == (min(F32(1e9), zz.min()) if len(zz) else F32(1e9))
    assert _voxel_host([], 0, 0, 0.15)[0] == 2 and _voxel_host([], 0, 1, 0.15)[0] == 0


def test_abi_arguments_and_no_device():
    lib = _lib.lib()
    h = C.c_void_p()
    assert lib.sm_ground_removal_create(-1, C.byref(h)) == -1
    assert lib.sm_ground_removal_create(0, None) == -1
    assert lib.sm_ground_removal_create(0, C.byref(h)) == 0
    try:
        assert lib.sm_ground_removal_set_param(h, b"std_mul", 1, b"1") == -10           # StatisticRemoval's
        assert b"unknown param std_mul" in lib.sm_ground_removal_last_error(h)
        assert lib.sm_ground_removal_set_param(h, b"min", 1, b"1") == -10               # AxisRange's, same storage
        assert lib.sm_ground_removal_set_param(h, b"leaf_size", 2, b"1") == -1
        assert lib.sm_ground_removal_set_param(h, b"leaf_size", 1, b"0") == 0           # every value is accepted
        assert lib.sm_ground_removal_set_param(h, b"height_threshold", 1, b"-3") == 0
        assert lib.sm_ground_removal_set_param(h, b"min_point_num_in_voxel", 1, b"3.9") == 0
        assert lib.sm_ground_removal_set_param(None, b"leaf_size", 1, b"1") == -1
        pts = np.zeros((100, 5), F32)
        out = np.zeros((100, 5), F32)
        m = C.c_int64(-7)
        run = lambda n, stride, p=pts.ctypes.data, o=out.ctypes.data: lib.sm_ground_removal_run(  # noqa: E731
            h, p, n, stride, o, C.byref(m), None)
        assert run(100, 16) == -1 and run(100, 22) == -1 and run(-1, 20) == -1 and run((1 << 30) + 1, 20) == -1
        assert run(100, 20, p=None) == -1 and run(100, 20, o=None) == -1
        assert lib.sm_ground_removal_run(h, pts.ctypes.data, 100, 20, out.ctypes.data, None, None) == -1
        assert m.value == -7
        ni, no = C.c_int64(-7), C.c_int64(-7)
        assert lib.sm_ground_removal_indices(h, None, C.byref(ni), None, C.byref(no)) == 0
        assert ni.value == 0 and no.value == 0                                        # before any run
        assert lib.sm_ground_removal_indices(h, None, None, None, C.byref(no)) == -1
        assert lib.sm_ground_removal_indices(None, None, C.byref(ni), None, C.byref(no)) == -1
        if lib.sm_device_count() == 0:
            assert run(100, 20) == -20 and b"no CUDA device" in lib.sm_ground_removal_last_error(h)
            assert run(0, 20) == -20
            assert lib.sm_ground_removal_run_device(h, pts.ctypes.data, 100, 20, out.ctypes.data, C.byref(m), None,
                                                    None) == -20
            assert m.value == -7
    finally:
        assert lib.sm_ground_removal_destroy(h) == 0
    assert lib.sm_ground_removal_destroy(None) == -1


def test_python_mirror_parses_like_the_factory():
    f = smb.GroundRemoval()
    f.InitFromXmlText('<filter name="GroundRemoval"><param type="0" name="min_point_num_in_voxel">12</param>'
                      '<param type="1" name="leaf_size"> 0.5 </param>'
                      '<param type="1" name="height_threshold">0.2</param></filter>')
    with pytest.raises(smb.CheckFailure):
        f.InitFromXmlText('<filter name="GroundRemoval"><param type="1" name="leaf">0.5</param></filter>')
    with pytest.raises(smb.CheckFailure):
        f.InitFromXmlText('<filter name="GroundRemoval"><param name="leaf_size">1</param></filter>')
    with pytest.raises(ValueError):
        f.InitFromXmlText('<filter name="GroundRemoval2"/>')
    with pytest.raises(ValueError):
        f.InitFromXmlText('<filters><filter name="GroundRemoval"/></filters>')
    assert f.Filter() is None
    f.SetInputCloud(np.zeros((3, 5), F32))
    with pytest.raises(ValueError):
        f.SetInputCloud(np.zeros((3, 4), F32))
    if _lib.lib().sm_device_count() == 0:
        with pytest.raises(RuntimeError):
            f.Filter()
