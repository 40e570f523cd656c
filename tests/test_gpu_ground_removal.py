"""GroundRemoval on an H100 (sm_ground_removal_*) bit for bit against the C++ restatement
(oracle/ground_removal_oracle.cc): emitted records, their order, their input indices, inliers and outliers.  On the scan
at three leaf sizes, on every scene, at sizes around the compaction tile and the radix sort's launch-path change up to
1.2 M points, at strides 20 and 32, through the host and device entries, on two handles on two streams, on one handle
reused with other parameters and sizes, past the key's span limit, and through the device hand-off to Ndt."""
import ctypes as C
import threading

import numpy as np
import pytest

import ground_removal_scenes as S
import oracle_ground_removal as OG
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

pytestmark = pytest.mark.gpu

F32 = np.float32


class Filter:
    """one sm_ground_removal handle"""

    def __init__(self, params=S.DEFAULT):
        self.lib = _lib.lib()
        self.h = C.c_void_p()
        assert self.lib.sm_ground_removal_create(0, C.byref(self.h)) == 0
        self.set(params)

    def set(self, params):
        min_points, leaf, thr = params
        for name, ptype, text in ((b"min_point_num_in_voxel", 0, str(int(min_points))),
                                  (b"leaf_size", 1, "%.9g" % leaf), (b"height_threshold", 1, "%.9g" % thr)):
            assert self.lib.sm_ground_removal_set_param(self.h, name, ptype, text.encode()) == 0

    def __del__(self):
        self.lib.sm_ground_removal_destroy(self.h)

    def indices(self):
        ni, no = C.c_int64(0), C.c_int64(0)
        assert self.lib.sm_ground_removal_indices(self.h, None, C.byref(ni), None, C.byref(no)) == 0
        inl, outl = np.full(max(ni.value, 1), -7, np.int32), np.full(max(no.value, 1), -7, np.int32)
        assert self.lib.sm_ground_removal_indices(self.h, inl.ctypes.data, C.byref(ni), outl.ctypes.data,
                                                  C.byref(no)) == 0
        return inl[:ni.value], outl[:no.value]

    def run(self, rec, stride=20):
        """host entry: rec (n, 5) float32 -> (out, index, rc)"""
        n = len(rec)
        buf = _strided(rec, stride)
        out = np.full((max(n, 1), 5), -7.0, F32)
        idx = np.full(max(n, 1), -7, np.int32)
        m = C.c_int64(-7)
        rc = self.lib.sm_ground_removal_run(self.h, buf.ctypes.data, n, stride, out.ctypes.data, C.byref(m),
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
        rc = self.lib.sm_ground_removal_run_device(self.h, d_in.data_ptr(), n, stride, d_out.data_ptr(), C.byref(m),
                                                   d_idx.data_ptr(), C.c_void_p(s.cuda_stream))
        assert rc == 0, self.lib.sm_ground_removal_last_error(self.h)
        k = m.value
        return d_out[:k].cpu().numpy(), d_idx[:k].cpu().numpy(), d_out


def _strided(rec, stride):
    rec = np.ascontiguousarray(np.asarray(rec, F32)[:, :5])
    if stride == 20:
        return rec
    buf = np.full((len(rec), stride // 4), 9.0, F32)
    buf[:, :5] = rec
    return buf


def _check(rec, params=S.DEFAULT, f=None, stride=20, device=False):
    if f is None:
        f = Filter(params)
    else:
        f.set(params)
    o = OG.ground_removal(rec, *params)
    if device:
        out, idx, _ = f.run_device(rec, stride)
    else:
        out, idx, rc = f.run(rec, stride)
        assert rc == 0, f.lib.sm_ground_removal_last_error(f.h)
    ctx = dict(n=len(rec), params=params, stride=stride, device=device)
    assert np.array_equal(idx, o.index), ctx
    assert out.tobytes() == o.out.tobytes(), ctx
    inl, outl = f.indices()
    assert np.array_equal(inl, o.inliers) and np.array_equal(outl, o.outliers), ctx
    return o


@pytest.fixture(scope="module")
def scan():
    return S.scan()


@pytest.mark.parametrize("leaf", [0.2, 0.8, 2.0])
@pytest.mark.parametrize("stride", [20, 32])
@pytest.mark.parametrize("device", [False, True])
def test_scan_host_and_device_entries(scan, leaf, stride, device):
    o = _check(scan, (10, leaf, 0.15), stride=stride, device=device)
    assert len(o.inliers) > 0 and len(o.outliers) > 0


@pytest.mark.parametrize("name", sorted(S.scenes()))
def test_scenes(name):
    rec, params = S.scenes()[name]
    f = Filter()
    for p in params:
        _check(rec, p, f=f)
        _check(rec, p, f=f, stride=32, device=True)


def test_sizes_around_the_launch_paths():
    # around the compaction tile (2048) and the radix sort's switch to the multi-block scan (262 144 keys), to 1.2 M
    rng = np.random.default_rng(11)
    f = Filter()
    for n in (1, 2, 31, 2047, 2048, 2049, 4097, 262_144, 262_145, 1_200_000):
        xyz = rng.uniform([-40, -40, -2.0], [40, 40, 3.0], (n, 3))
        xyz[: n // 2, 2] = -1.73 + rng.normal(size=n // 2) * 0.03
        _check(S.records(xyz), (3, 0.8, 0.15), f=f)


def test_one_voxel_holds_every_point():
    rng = np.random.default_rng(12)
    rec = S.records(rng.uniform([-30, -30, -2.0], [30, 30, 0.5], (1_200_000, 3)))
    for thr in (5.0, 0.15):
        _check(rec, (10, 1000.0, thr))
    _check(rec, (10, 0.0, 0.15))                         # leaf 0: every point in (INT_MIN, INT_MIN, INT_MIN)


def test_empty_input():
    f = Filter()
    _check(S.scan()[:5000], f=f)
    out, idx, rc = f.run(np.zeros((0, 5), F32))
    assert rc == 0 and len(idx) == 0 and all(len(a) == 0 for a in f.indices())


def test_span_limit():
    f = Filter()
    for rec, leaf, fits in S.span_limit():
        if fits:
            _check(rec, (1, leaf, 0.15), f=f)
            continue
        before = f.indices()
        f.set((1, leaf, 0.15))
        assert f.run(rec)[2] == -1
        assert b"2^21 - 1" in f.lib.sm_ground_removal_last_error(f.h)
        after = f.indices()                              # still the last successful run's
        assert all(np.array_equal(a, b) for a, b in zip(before, after))


def test_two_handles_on_two_streams(scan):
    import torch
    jobs = [(scan, (10, 0.8, 0.15)), (S.spread(200_000, seed=4), (4, 0.3, 0.05))]
    want = [OG.ground_removal(r, *p) for r, p in jobs]
    filters = [Filter(p) for _, p in jobs]
    errors = []

    def run(i):
        try:
            for _ in range(3):
                out, idx, _ = filters[i].run_device(jobs[i][0], stream=torch.cuda.Stream())
                assert np.array_equal(idx, want[i].index) and out.tobytes() == want[i].out.tobytes()
                inl, outl = filters[i].indices()
                assert np.array_equal(inl, want[i].inliers) and np.array_equal(outl, want[i].outliers)
        except Exception as e:      # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors


def test_reuse_with_other_parameters_and_sizes(scan):
    f = Filter()
    first = _check(scan, f=f)
    _check(scan[:3000].copy(), (3, 0.2, 0.05), f=f)
    _check(S.spread(300_000), (10, 2.0, 0.3), f=f, device=True)
    _check(scan, f=f)
    assert f.run(scan)[0].tobytes() == first.out.tobytes()


def test_python_mirror(scan):
    f = smb.GroundRemoval()
    f.InitFromXmlText('<filter name="GroundRemoval"><param type="0" name="min_point_num_in_voxel">10</param>'
                      '<param type="1" name="leaf_size">0.8</param>'
                      '<param type="1" name="height_threshold">0.15</param></filter>')
    f.SetInputCloud(smb.InnerCloud(scan))
    cloud = f.Filter()
    o = OG.ground_removal(scan, 10, 0.8, 0.15)
    assert cloud.points.tobytes() == o.out.tobytes()
    assert np.array_equal(f.Inliers(), o.inliers) and np.array_equal(f.Outliers(), o.outliers)
    f.SetInputCloud(scan[:0])
    assert len(f.Filter().points) == 0 and len(f.Inliers()) == 0 and len(f.Outliers()) == 0
    f.SetParam("leaf_size", 1, "1e-3")
    f.SetInputCloud(S.span_limit()[-1][0])
    with pytest.raises(ValueError):
        f.Filter()


def test_device_output_feeds_the_matcher(scan):
    """device GroundRemoval -> sm_set_input_source_f32_device -> Ndt.Align, against the host path"""
    lib = _lib.lib()
    src, tgt = scan[::4].copy(), S.scan(seed=3)[::6].copy()
    f = Filter((3, 0.8, 0.15))
    host_out, _, rc = f.run(src)
    assert rc == 0
    _, idx, d_out = f.run_device(src)
    m = len(idx)
    assert m == len(host_out) and 0 < m < len(src)
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
