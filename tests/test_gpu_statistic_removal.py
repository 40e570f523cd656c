"""StatisticRemoval on an H100 (sm_statistic_removal_*) bit for bit against the CPU oracle's product mode
(oracle/statistic_removal_oracle.cc): kept records, inlier indices, per-point distances and the four statistics.  Also
the host and device entry points, strides, every k-list path of the search, the compaction and tree-build launch
paths, the CHECK case, two handles on two streams, reuse of one handle, repeatability and the device hand-off to Ndt."""
import ctypes as C
import math
import threading

import numpy as np
import pytest

import kd_tree_model as M
import oracle_statistic_removal as OS
import statistic_removal_scenes as S
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

pytestmark = pytest.mark.gpu

F32 = np.float32


class Filter:
    """one sm_statistic_removal handle"""

    def __init__(self, K=30, std_mul=1.0):
        self.lib = _lib.lib()
        self.h = C.c_void_p()
        assert self.lib.sm_statistic_removal_create(0, C.byref(self.h)) == 0
        assert self.lib.sm_statistic_removal_set_param(self.h, b"point_num_meank", 0, str(int(K)).encode()) == 0
        assert self.lib.sm_statistic_removal_set_param(self.h, b"std_mul", 1, ("%.9g" % std_mul).encode()) == 0

    def __del__(self):
        self.lib.sm_statistic_removal_destroy(self.h)

    def stats(self):
        s = (C.c_double * 4)()
        assert self.lib.sm_statistic_removal_stats(self.h, s) == 0
        return tuple(s)

    def distances(self, n):
        out = np.zeros(max(n, 1), F32)
        got = C.c_int64(0)
        assert self.lib.sm_debug_statistic_removal_distances(self.h, out.ctypes.data, n, C.byref(got)) == 0
        assert got.value == n
        return out[:n]

    def run(self, rec, stride=20):
        """host entry: rec (n, 5) float32 -> (out, inliers, rc)"""
        n = len(rec)
        buf = _strided(rec, stride)
        out = np.full((max(n, 1), 5), -7.0, F32)
        idx = np.full(max(n, 1), -7, np.int32)
        m = C.c_int64(-7)
        rc = self.lib.sm_statistic_removal_run(self.h, buf.ctypes.data, n, stride, out.ctypes.data, C.byref(m),
                                               idx.ctypes.data)
        if rc != 0:
            assert m.value == -7 and np.all(out == -7.0) and np.all(idx == -7)      # outputs untouched
            return None, None, rc
        return out[:m.value].copy(), idx[:m.value].copy(), rc

    def run_device(self, rec, stride=20, stream=None):
        import torch
        n = len(rec)
        d_in = torch.from_numpy(_strided(rec, stride).reshape(-1)).cuda()
        d_out = torch.empty((max(n, 1), 5), dtype=torch.float32, device="cuda")
        d_idx = torch.empty(max(n, 1), dtype=torch.int32, device="cuda")
        m = C.c_int64(0)
        s = stream or torch.cuda.current_stream()
        torch.cuda.synchronize()
        rc = self.lib.sm_statistic_removal_run_device(self.h, d_in.data_ptr(), n, stride, d_out.data_ptr(), C.byref(m),
                                                      d_idx.data_ptr(), C.c_void_p(s.cuda_stream))
        assert rc == 0
        k = m.value
        return d_out[:k].cpu().numpy(), d_idx[:k].cpu().numpy(), d_out


def _strided(rec, stride):
    rec = np.ascontiguousarray(np.asarray(rec, F32)[:, :5])
    if stride == 20:
        return rec
    buf = np.full((len(rec), stride // 4), 9.0, F32)
    buf[:, :5] = rec
    return buf


def _same_stats(a, b):
    return all(x == y or (math.isnan(x) and math.isnan(y)) for x, y in zip(a, b))


def _check(rec, K=30, std_mul=1.0, f=None, stride=20, device=False):
    f = f or Filter(K, std_mul)
    o = OS.statistic_removal(rec, K, std_mul, OS.PRODUCT)
    if device:
        out, idx, _ = f.run_device(rec, stride)
    else:
        out, idx, rc = f.run(rec, stride)
        assert rc == 0
    ctx = dict(n=len(rec), K=K, std_mul=std_mul, stride=stride, device=device)
    assert np.array_equal(idx, o.inliers), ctx
    assert out.tobytes() == o.out.tobytes(), ctx
    got = f.distances(len(rec))
    bad = np.flatnonzero(got.view(np.int32) != o.distances.view(np.int32))
    assert bad.size == 0, (ctx, bad[:5], got[bad[:5]], o.distances[bad[:5]])
    assert _same_stats(f.stats(), o.stats), (ctx, f.stats(), o.stats)
    return o


@pytest.fixture(scope="module")
def scan():
    return S.scan()


@pytest.mark.parametrize("stride", [20, 32])
@pytest.mark.parametrize("device", [False, True])
def test_scan_host_and_device_entries(scan, stride, device):
    o = _check(scan, 30, 1.0, stride=stride, device=device)
    assert 0 < len(o.inliers) < len(scan)


@pytest.mark.parametrize("K", [1, 3, 7, 8, 30, 63])
def test_every_list_path(K):
    # k = K + 1 crosses the 4- and 8-entry register lists and the shared-memory list at k = 4, 8 and 9
    rec, at = S.planted(20_000, 40, seed=K)
    for std_mul in (1.0, 0.0, -3.0):
        o = _check(rec, K, std_mul)
    assert not np.any(np.isin(at, _check(rec, K, 1.0).inliers))


def test_launch_path_sizes():
    # around the compaction tile (2048) and the tree builder's launch-path changes, up to 1.2 M points
    cap = M.sub_capacity(8)
    rng = np.random.default_rng(11)
    f = Filter(30, 1.0)
    for n in (31, 2047, 2048, 2049, 4097, cap + 1, 2 * cap + 1, 262_145, 1_200_000):
        xyz = rng.normal(size=(n, 3)) * [20.0, 20.0, 2.0]
        _check(S.records(xyz), 30, 1.0, f=f)


@pytest.mark.parametrize("name", sorted(S.adversarial()) + ["duplicates", "grid", "line"])
def test_adversarial_and_tie_clouds(name):
    rec = {**S.adversarial(), **S.ties()}[name]
    for K in (1, 8, 30, 63):
        _check(rec, K, 1.0)


def test_non_finite_points_and_the_check_case():
    rec = S.non_finite()
    for std_mul in (1.0, -3.0, float("nan")):
        _check(rec, 8, std_mul)
    f = Filter(30, 1.0)
    few = S.records(np.concatenate([np.random.default_rng(1).normal(size=(30, 3)), np.full((50, 3), np.nan)]))
    assert f.run(few)[2] == -5                                          # 30 finite points, K = 30
    assert b"Check failed" in f.lib.sm_statistic_removal_last_error(f.h)
    o = _check(few[:25].copy() * np.nan, 30, 1.0, f=f)                  # no finite point: all kept
    assert len(o.inliers) == 25 and math.isnan(f.stats()[2])
    out, idx, rc = f.run(np.zeros((0, 5), F32))
    assert rc == 0 and len(idx) == 0 and f.stats()[3] == 0.0


def test_two_handles_on_two_streams(scan):
    import torch
    jobs = [(scan, 30, 1.0), (S.planted(50_000, 30)[0], 7, 0.5)]
    want = [OS.statistic_removal(r, K, s) for r, K, s in jobs]
    filters = [Filter(K, s) for _, K, s in jobs]
    out = [None, None]
    errors = []

    def run(i):
        try:
            for _ in range(3):
                out[i] = filters[i].run_device(jobs[i][0], stream=torch.cuda.Stream())
                assert np.array_equal(out[i][1], want[i].inliers) and out[i][0].tobytes() == want[i].out.tobytes()
        except Exception as e:      # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors


def test_reuse_large_small_large_and_repeatability(scan):
    f = Filter(30, 1.0)
    first = _check(scan, f=f)
    bytes_first = f.run(scan)[0].tobytes()
    _check(scan[:3000].copy(), f=f)
    _check(scan, f=f)
    assert f.run(scan)[0].tobytes() == bytes_first == first.out.tobytes()


def test_python_mirror(scan):
    f = smb.StatisticRemoval()
    f.InitFromXmlText('<filter name="StatisticRemoval"><param type="0" name="point_num_meank">30</param>'
                      '<param type="1" name="std_mul">1.0</param></filter>')
    f.SetInputCloud(smb.InnerCloud(scan))
    cloud = f.Filter()
    o = OS.statistic_removal(scan, 30, 1.0)
    assert np.array_equal(f.Inliers(), o.inliers) and cloud.points.tobytes() == o.out.tobytes()
    assert len(f.Inliers()) + len(f.Outliers()) == len(scan) and _same_stats(f.Stats(), o.stats)
    f.SetInputCloud(scan[:20])
    with pytest.raises(smb.CheckFailure):
        f.Filter()


def test_device_output_feeds_the_matcher(scan):
    """device StatisticRemoval -> sm_set_input_source_f32_device -> Ndt.Align, against the host path"""
    lib = _lib.lib()
    src, tgt = scan[::4].copy(), S.scan(seed=3)[::6].copy()
    f = Filter(30, 1.0)
    host_out, _, rc = f.run(src)
    assert rc == 0
    _, idx, d_out = f.run_device(src)
    m = len(idx)
    assert m == len(host_out)
    tgt3 = np.ascontiguousarray(tgt[:, :3])
    results = []
    for device_path in (True, False):
        h = C.c_void_p()
        assert lib.sm_create(5, 0, C.byref(h)) == 0                 # SM_TYPE_NDT
        assert lib.sm_set_input_target_f32(h, tgt3.ctypes.data, len(tgt3), 12) == 0
        if device_path:
            assert lib.sm_set_input_source_f32_device(h, d_out.data_ptr(), m, 20) == 0
        else:
            assert lib.sm_set_input_source_f32(h, host_out.ctypes.data, m, 20) == 0
        guess, res = np.asfortranarray(np.eye(4)), np.zeros(16)
        assert lib.sm_align(h, guess.ctypes.data_as(_lib._DP), res.ctypes.data_as(_lib._DP)) >= 0
        lib.sm_destroy(h)
        results.append(res)
    assert np.array_equal(results[0], results[1]) and not np.array_equal(results[0], np.eye(4).ravel())
