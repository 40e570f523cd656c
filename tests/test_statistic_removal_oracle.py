"""StatisticRemoval without a GPU: the CPU oracle (oracle/statistic_removal_oracle.cc) against a hand-computed answer and
against the numpy restatement (tests/pyref_statistic_removal.py), product mode against PCL's literal mode, the product's
host-compiled exact sum and per-point distance (include/sm_b200_debug.h) against math.fsum and numpy, and the C ABI's
argument checks."""
import ctypes as C
import math

import numpy as np
import pytest

import oracle_statistic_removal as OS
import pyref_statistic_removal as PR
import statistic_removal_scenes as S
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

F32 = np.float32


def _bits(a, b):
    """equal as IEEE doubles, NaN equal to NaN"""
    return all((x == y) or (math.isnan(x) and math.isnan(y)) for x, y in zip(a, b))


def _kept(res, n):
    k = np.zeros(n, bool)
    k[res.inliers] = True
    return k


def _against_numpy(rec, K, std_mul):
    o = OS.statistic_removal(rec, K, std_mul, OS.PRODUCT)
    p = PR.statistic_removal(rec, K, std_mul, rank="double")
    assert np.array_equal(o.distances.view(np.int32), p.distances.view(np.int32)), (K, std_mul)
    assert _bits(o.stats, p.stats), (o.stats, p.stats)
    assert np.array_equal(_kept(o, len(rec)), p.kept)
    assert o.out.tobytes() == np.ascontiguousarray(rec[p.kept, :5]).tobytes()
    ol = OS.statistic_removal(rec, K, std_mul, OS.LITERAL)
    pf = PR.statistic_removal(rec, K, std_mul, rank="float")
    assert np.array_equal(ol.distances.view(np.int32), pf.distances.view(np.int32)), (K, std_mul)
    return o


def test_hand_computed_line():
    # x = 0, 1, 2, 3, 10 with K = 2: mean distances 1.5, 1, 1, 1.5, 7.5
    rec = S.records([[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 0, 0], [10, 0, 0]])
    mean = 12.5 / 5
    variance = (62.75 - 12.5 * 12.5 / 5) / 4
    want = (mean, math.sqrt(variance), mean + math.sqrt(variance), 5.0)
    assert want[2] == pytest.approx(5.3062430, abs=1e-6)
    for mode in (OS.PRODUCT, OS.LITERAL):
        r = OS.statistic_removal(rec, 2, 1.0, mode)
        assert r.distances.tolist() == [1.5, 1.0, 1.0, 1.5, 7.5]
        assert r.stats == want
        assert r.inliers.tolist() == [0, 1, 2, 3] and r.out.tobytes() == rec[:4].tobytes()
    assert PR.statistic_removal(rec, 2, 1.0).stats == want
    assert OS.statistic_removal(rec, 2, -0.5).inliers.tolist() == [1, 2]        # threshold 2.5 - 1.403 = 1.097
    assert OS.statistic_removal(rec, 2, -3.0).inliers.tolist() == []


def test_scan():
    o = _against_numpy(S.scan(), 30, 1.0)
    assert 0 < len(o.inliers) < 120_000


def test_planted_outliers_are_removed():
    rec, at = S.planted()
    for K in (7, 30):
        o = _against_numpy(rec, K, 1.0)
        assert not np.any(np.isin(at, o.inliers)), K


@pytest.mark.parametrize("name", ["duplicates", "grid", "line"])
@pytest.mark.parametrize("K", [1, 7, 8, 30, 63])
def test_ties(name, K):
    _against_numpy(S.ties()[name], K, 1.0)


@pytest.mark.parametrize("std_mul", [0.0, 1.0, -3.0, float("nan")])
def test_non_finite_points_and_std_mul(std_mul):
    rec = S.non_finite()
    o = _against_numpy(rec, 8, std_mul)
    bad = ~np.all(np.isfinite(rec[:, :3]), axis=1)
    assert o.stats[3] == float(np.count_nonzero(~bad)) and np.all(o.distances[bad] == 0)
    if math.isnan(std_mul):
        assert len(o.inliers) == len(rec)         # NaN threshold: nothing is > it
    if std_mul == -3.0:
        assert np.all(np.isin(np.flatnonzero(bad), o.inliers)) == (o.stats[2] >= 0)


@pytest.mark.parametrize("K", [1, 7, 8, 30, 63])
def test_n_equals_K_plus_one(K):
    rec = S.records(np.random.default_rng(K).normal(size=(K + 1, 3)))
    _against_numpy(rec, K, 1.0)
    with pytest.raises(RuntimeError):
        OS.statistic_removal(rec[:K], K, 1.0)


def test_no_finite_point_keeps_everything():
    rec = S.records(np.full((40, 3), np.nan))
    o = _against_numpy(rec, 5, 1.0)
    assert len(o.inliers) == 40 and math.isnan(o.stats[2]) and o.stats[3] == 0.0


@pytest.mark.parametrize("name", sorted(S.adversarial()))
def test_adversarial_clouds(name):
    _against_numpy(S.adversarial()[name], 30, 1.0)


def test_product_against_literal():
    """the correctly rounded sums and libnabo's double ranking against PCL's serial sums and float ranking: distances
    within 1e-6, kept sets equal but for points in the band around the threshold the two modes' differences bound;
    on these scenes the band is empty"""
    scenes = [("scan", S.scan(), 30), ("planted", S.planted()[0], 30), ("non-finite", S.non_finite(), 8)]
    scenes += [(k, v, 30) for k, v in S.ties().items()] + [(k, v, 30) for k, v in S.adversarial().items()]
    band_total = 0
    for name, rec, K in scenes:
        p = OS.statistic_removal(rec, K, 1.0, OS.PRODUCT)
        lit = OS.statistic_removal(rec, K, 1.0, OS.LITERAL)
        dp, dl = p.distances.astype(np.float64), lit.distances.astype(np.float64)
        assert np.all(np.abs(dp - dl) <= 1e-6 * np.maximum(np.abs(dl), 1e-30)), name
        tp, tl = p.stats[2], lit.stats[2]
        # a point can be decided differently only within |tp - tl| + |dp - dl| of tp, and not at all when both are 0
        width = abs(tp - tl) + np.abs(dp - dl)
        band = (np.abs(dp - tp) <= width) & (width > 0)
        differ = _kept(p, len(rec)) != _kept(lit, len(rec))
        assert not np.any(differ & ~band), name
        band_total += int(np.count_nonzero(band))
        print(f"{name}: threshold {tp!r} vs {tl!r}, {np.count_nonzero(band)} points in the band, "
              f"{np.count_nonzero(differ)} kept differently")
    assert band_total == 0


def _exact_sum(terms):
    t = np.ascontiguousarray(np.asarray(terms, F32))
    out = C.c_double()
    rc = _lib.lib().sm_debug_statistic_removal_exact_sum_host(t.ctypes.data, len(t), C.byref(out))
    assert rc == 0
    return out.value


def test_exact_sum_against_fsum():
    rng = np.random.default_rng(3)
    tiny = np.float32(1.4e-45)
    cases = {
        "empty": np.zeros(0, F32),
        "zeros": np.zeros(1000, F32),
        "subnormals": rng.integers(1, 1 << 23, 5000).astype(np.uint32).view(F32),
        "smallest": np.full(3, tiny, F32),
        "full range": rng.integers(0, 0x7f7fffff, 20_000).astype(np.uint32).view(F32),
        "max": np.full(1000, np.finfo(F32).max, F32),
        "equal terms": np.full(1 << 20, F32(0.1)),
        "mixed scales": np.concatenate([np.full(7, F32(1e30)), np.full(1 << 16, F32(3e-8)), [F32(1.0)]]),
        "ties to even": np.array([2.0 ** 53, 1.0, 2.0 ** -30], F32),
        "one distance cloud": OS.statistic_removal(S.scan(), 30, 1.0).distances,
    }
    for name, t in cases.items():
        want = math.fsum(t.astype(np.float64).tolist())
        got = _exact_sum(t)
        assert got == want, (name, got, want)
    assert _exact_sum(np.array([1.0, np.inf, 2.0], F32)) == math.inf
    for bad in ([-1.0], [np.nan], [1.0, -0.5]):
        out = C.c_double()
        assert _lib.lib().sm_debug_statistic_removal_exact_sum_host(np.asarray(bad, F32).ctypes.data, len(bad),
                                                                    C.byref(out)) == -1


def test_distance_host_against_numpy():
    rng = np.random.default_rng(4)
    for K in (1, 2, 30, 63):
        for _ in range(50):
            q = (rng.normal(size=3) * rng.choice([1e-3, 1.0, 1e4])).astype(F32)
            nb = (q + rng.normal(size=(K, 3)) * rng.choice([1e-4, 1.0, 100.0])).astype(F32)
            got = C.c_float()
            assert _lib.lib().sm_debug_statistic_removal_distance_host(q.ctypes.data, np.ascontiguousarray(nb).ctypes.data,
                                                                       K, C.byref(got)) == 0
            d2 = PR._float_d2(q[None, :], nb[None])[0]
            s = 0.0
            for v in d2:
                s = s + math.sqrt(float(v))
            assert np.float32(got.value) == np.float32(s / K)


def test_abi_arguments_and_no_device():
    lib = _lib.lib()
    h = C.c_void_p()
    assert lib.sm_statistic_removal_create(-1, C.byref(h)) == -1
    assert lib.sm_statistic_removal_create(0, None) == -1
    assert lib.sm_statistic_removal_create(0, C.byref(h)) == 0
    try:
        assert lib.sm_statistic_removal_set_param(h, b"min_range", 1, b"1") == -10       # Range's, not this filter's
        assert b"unknown param min_range" in lib.sm_statistic_removal_last_error(h)
        assert lib.sm_statistic_removal_set_param(h, b"std_mul", 2, b"1") == -1
        assert lib.sm_statistic_removal_set_param(h, b"std_mul", 1, b"2.5") == 0
        pts = np.zeros((100, 5), F32)
        out = np.zeros((100, 5), F32)
        m = C.c_int64(-7)
        run = lambda n, stride, p=pts.ctypes.data, o=out.ctypes.data: lib.sm_statistic_removal_run(  # noqa: E731
            h, p, n, stride, o, C.byref(m), None)
        for K in (b"0", b"64", b"-3"):
            assert lib.sm_statistic_removal_set_param(h, b"point_num_meank", 0, K) == 0
            assert run(100, 20) == -1 and b"point_num_meank" in lib.sm_statistic_removal_last_error(h)
        assert lib.sm_statistic_removal_set_param(h, b"point_num_meank", 1, b"63.9") == 0    # as_float, then (int)
        assert run(100, 16) == -1 and run(100, 22) == -1 and run(-1, 20) == -1 and run((1 << 30) + 1, 20) == -1
        assert run(100, 20, p=None) == -1 and run(100, 20, o=None) == -1
        assert lib.sm_statistic_removal_run(h, pts.ctypes.data, 100, 20, out.ctypes.data, None, None) == -1
        assert m.value == -7
        if lib.sm_device_count() == 0:
            assert run(100, 20) == -20 and b"no CUDA device" in lib.sm_statistic_removal_last_error(h)
            assert run(0, 20) == -20
            assert lib.sm_statistic_removal_run_device(h, pts.ctypes.data, 100, 20, out.ctypes.data, C.byref(m), None,
                                                       None) == -20
        stats = (C.c_double * 4)()
        assert lib.sm_statistic_removal_stats(h, stats) == 0 and stats[3] == 0.0 and math.isnan(stats[0])
        assert lib.sm_statistic_removal_stats(h, None) == -1
    finally:
        assert lib.sm_statistic_removal_destroy(h) == 0
    assert lib.sm_statistic_removal_destroy(None) == -1


def test_python_mirror_parses_like_the_factory():
    f = smb.StatisticRemoval()
    f.InitFromXmlText('<filter name="StatisticRemoval"><param type="0" name="point_num_meank">12</param>'
                      '<param type="1" name="std_mul"> 0.5 </param></filter>')
    with pytest.raises(smb.CheckFailure):
        f.InitFromXmlText('<filter name="StatisticRemoval"><param type="0" name="mean_k">12</param></filter>')
    with pytest.raises(smb.CheckFailure):
        f.InitFromXmlText('<filter name="StatisticRemoval"><param name="std_mul">1</param></filter>')
    with pytest.raises(ValueError):
        f.InitFromXmlText('<filter name="VoxelGrid"/>')
    assert f.Filter() is None
    f.SetInputCloud(np.zeros((3, 5), F32))
    if _lib.lib().sm_device_count() == 0:
        with pytest.raises(RuntimeError):
            f.Filter()
