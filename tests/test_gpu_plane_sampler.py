"""RandomSamplerWithPlaneDetect on an H100 (sm_plane_sampler_*) bit for bit against the C++ restatement
(oracle/plane_sampler_oracle.cc): kept records, inliers, outliers, plane indices and the per-voxel RANSAC traces
(status, iterations, best count, refined coefficients, final count).  On every scene, the scan and the 500 k submap at
three leaf sizes and two rates, voxels on both launch shapes (one warp, one CTA past 512 points), strides 20 and 32,
the host and device entries, two handles on two streams, one handle reused with other parameters and sizes, 2^24
records, the span limit, and the device hand-off to a matcher's target."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_plane_sampler as OP
import plane_sampler_scenes as S
import staticmapping_b200 as smb
from staticmapping_b200 import _lib, synth

pytestmark = pytest.mark.gpu

F32 = np.float32


class Sampler:
    """one sm_plane_sampler handle with the trace on"""

    def __init__(self, params=S.DEFAULT):
        self.lib = _lib.lib()
        self.h = C.c_void_p()
        assert self.lib.sm_plane_sampler_create(0, C.byref(self.h)) == 0
        assert self.lib.sm_debug_plane_sampler_trace(self.h, 1) == 0
        self.set(params)

    def set(self, params):
        rate, leaf, min_points = params
        assert self.lib.sm_plane_sampler_set_sampling_rate(self.h, rate) == 0
        assert self.lib.sm_plane_sampler_set_leaf_size(self.h, leaf) == 0
        assert self.lib.sm_plane_sampler_set_min_point_num_in_voxel(self.h, min_points) == 0

    def __del__(self):
        self.lib.sm_plane_sampler_destroy(self.h)

    def lists(self):
        ni, no, npl = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        assert self.lib.sm_plane_sampler_indices(self.h, None, C.byref(ni), None, C.byref(no)) == 0
        assert self.lib.sm_plane_sampler_plane_indices(self.h, None, C.byref(npl)) == 0
        inl, outl, pl = (np.full(max(k.value, 1), -7, np.int32) for k in (ni, no, npl))
        assert self.lib.sm_plane_sampler_indices(self.h, inl.ctypes.data, C.byref(ni), outl.ctypes.data,
                                                 C.byref(no)) == 0
        assert self.lib.sm_plane_sampler_plane_indices(self.h, pl.ctypes.data, C.byref(npl)) == 0
        return inl[:ni.value], outl[:no.value], pl[:npl.value]

    def traces(self):
        nv = C.c_int64(0)
        assert self.lib.sm_debug_plane_sampler_voxels(self.h, None, 0, C.byref(nv)) in (0, -1)
        out = np.zeros(max(nv.value, 1), OP.TRACE)
        assert self.lib.sm_debug_plane_sampler_voxels(self.h, out.ctypes.data, len(out), C.byref(nv)) == 0
        return out[:nv.value]

    def run(self, rec, stride=20):
        """host entry: rec (n, 5) float32 -> (out, index, rc)"""
        n = len(rec)
        buf = _strided(rec, stride)
        out = np.full((max(n, 1), 5), -7.0, F32)
        idx = np.full(max(n, 1), -7, np.int32)
        m = C.c_int64(-7)
        rc = self.lib.sm_plane_sampler_run(self.h, buf.ctypes.data, n, stride, out.ctypes.data, C.byref(m),
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
        rc = self.lib.sm_plane_sampler_run_device(self.h, d_in.data_ptr(), n, stride, d_out.data_ptr(), C.byref(m),
                                                  d_idx.data_ptr(), C.c_void_p(s.cuda_stream))
        assert rc == 0, self.lib.sm_plane_sampler_last_error(self.h)
        k = m.value
        return d_out[:k].cpu().numpy(), d_idx[:k].cpu().numpy(), d_out


def _strided(rec, stride):
    rec = np.ascontiguousarray(np.asarray(rec, F32)[:, :5])
    if stride == 20:
        return rec
    buf = np.full((len(rec), stride // 4), 9.0, F32)
    buf[:, :5] = rec
    return buf


def _same(f, o, rec, out, idx, ctx):
    assert np.array_equal(idx, o.inliers), ctx
    assert out.tobytes() == np.ascontiguousarray(rec[o.keep, :5], F32).tobytes(), ctx
    inl, outl, pl = f.lists()
    assert np.array_equal(inl, o.inliers) and np.array_equal(outl, o.outliers), ctx
    assert np.array_equal(pl, o.plane), ctx
    t = f.traces()
    assert len(t) == len(o.traces), ctx
    # equal statuses, iteration counts, best counts and final counts, and equal refined coefficient bits voxel by voxel;
    # a NaN coefficient is NaN on both sides (its bit pattern is the device's or the host's default NaN)
    for name in ("status", "iterations", "best", "final_count"):
        bad = np.flatnonzero(t[name] != o.traces[name])
        assert len(bad) == 0, (ctx, name, t[bad][:5], o.traces[bad][:5])
    a, b = t["coef"], o.traces["coef"]
    same = (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    bad = np.flatnonzero(~same.all(axis=1))
    assert len(bad) == 0, (ctx, "coef", t[bad][:5], o.traces[bad][:5])


def _check(rec, params=S.DEFAULT, f=None, stride=20, device=False):
    rec = np.asarray(rec, F32)
    if f is None:
        f = Sampler(params)
    else:
        f.set(params)
    o = OP.plane_sampler(rec, *params)
    if device:
        out, idx, _ = f.run_device(rec, stride)
    else:
        out, idx, rc = f.run(rec, stride)
        assert rc == 0, f.lib.sm_plane_sampler_last_error(f.h)
    _same(f, o, rec, out, idx, dict(n=len(rec), params=params, stride=stride, device=device))
    return o


@pytest.fixture(scope="module")
def scan():
    return S.scan()


@pytest.fixture(scope="module")
def submap():
    xyz = synth.submap(synth.make_scene(0), seed=0)
    return S.records(xyz)


@pytest.mark.parametrize("leaf", [0.5, 0.8, 2.0])
@pytest.mark.parametrize("stride", [20, 32])
@pytest.mark.parametrize("device", [False, True])
def test_scan_host_and_device_entries(scan, leaf, stride, device):
    o = _check(scan, (0.5, leaf, 10), stride=stride, device=device)
    assert len(o.plane) > 0 and 0 < o.keep.sum() < len(scan)


@pytest.mark.parametrize("leaf", [0.5, 0.8, 2.0])
@pytest.mark.parametrize("rate", [0.5, 0.1])
def test_submap(submap, leaf, rate):
    o = _check(submap, (rate, leaf, 10))
    assert len(o.plane) > 0 and (leaf == 2.0 or np.any(o.traces["status"] >= 4))   # RANSAC ran below leaf 2


@pytest.mark.parametrize("name", sorted(S.scenes()))
def test_scenes(name):
    rec, params = S.scenes()[name]
    f = Sampler()
    for p in params:
        _check(rec, p, f=f)
        _check(rec, p, f=f, stride=32, device=True)


def test_both_launch_shapes():
    f = Sampler()
    for count in (511, 512, 513, 3000, 20000):
        o = _check(S.big_voxel(count), f=f)
        assert o.traces["status"][0] in (4, 5) and o.traces["iterations"][0] >= 1


def test_sizes_up_to_2_24():
    rng = np.random.default_rng(11)
    f = Sampler()
    for n in (1, 2, 31, 2047, 2048, 2049, 262_145, 1 << 24):
        xyz = rng.uniform([-60, -60, -2.0], [60, 60, 3.0], (n, 3))
        xyz[: n // 2, 2] = -0.5 + rng.normal(size=n // 2) * 0.03
        _check(S.records(xyz), (0.1, 0.8, 10), f=f)


def test_empty_input_and_limits():
    f = Sampler()
    _check(S.walls(), f=f)
    out, idx, rc = f.run(np.zeros((0, 5), F32))
    assert rc == 0 and len(idx) == 0 and all(len(a) == 0 for a in f.lists()) and len(f.traces()) == 0
    _check(S.walls(), f=f)
    before = f.lists()
    far = S.records(np.array([[0.5, 0.5, 0.5], [2e6, 0.5, 0.5]]))     # 2.5 M voxels apart at 0.8
    assert f.run(far)[2] == -1 and b"2^21 - 1" in f.lib.sm_plane_sampler_last_error(f.h)
    assert all(np.array_equal(a, b) for a, b in zip(before, f.lists()))   # still the last successful run's
    f.set((1.0, 0.8, 10))                                               # the copy path needs no voxels
    _check(far, (1.0, 0.8, 10), f=f)
    _check(far, (0.5, 0.2, 10), f=f)                                    # nor does leaf <= 0.2


def test_two_handles_on_two_streams(scan, submap):
    import torch
    jobs = [(scan, (0.5, 0.8, 10)), (submap[:200_000], (0.1, 0.5, 5))]
    want = [OP.plane_sampler(r, *p) for r, p in jobs]
    samplers = [Sampler(p) for _, p in jobs]
    errors = []

    def run(i):
        try:
            for _ in range(3):
                out, idx, _ = samplers[i].run_device(jobs[i][0], stream=torch.cuda.Stream())
                assert np.array_equal(idx, want[i].inliers)
                assert out.tobytes() == np.ascontiguousarray(jobs[i][0][want[i].keep, :5]).tobytes()
                inl, outl, pl = samplers[i].lists()
                assert np.array_equal(outl, want[i].outliers) and np.array_equal(pl, want[i].plane)
        except Exception as e:      # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors


def test_reuse_with_other_parameters_and_sizes(scan, submap):
    f = Sampler()
    first = _check(scan, f=f)
    _check(scan[:3000].copy(), (0.25, 0.3, 5), f=f)
    _check(submap, (0.1, 2.0, 20), f=f, device=True)
    _check(S.degenerate(), (0.5, 0.8, 10), f=f)
    out, idx, _ = f.run(scan)
    assert np.array_equal(idx, first.inliers)


def test_python_mirror(scan):
    s = smb.RandomSamplerWithPlaneDetect()
    s.SetSamplingRate(0.5)
    s.SetInputCloud(smb.InnerCloud(scan))
    cloud = s.Filter()
    o = OP.plane_sampler(scan, 0.5, 0.8, 10)
    assert cloud.points.tobytes() == np.ascontiguousarray(scan[o.keep, :5]).tobytes()
    assert np.array_equal(s.Inliers(), o.inliers) and np.array_equal(s.Outliers(), o.outliers)
    assert np.array_equal(s.PlaneIndices(), o.plane)
    s.SetSamplingRate(7.0)                                  # clamped to 1: the copy path
    assert s.Filter().points.tobytes() == np.ascontiguousarray(scan[:, :5]).tobytes()
    assert len(s.PlaneIndices()) == 0 and "large than 1" in s.messages[-1]
    s.SetInputCloud(scan[:0])
    assert len(s.Filter().points) == 0 and len(s.Inliers()) == 0 and len(s.Outliers()) == 0


def test_device_output_feeds_the_matcher_target(scan):
    """device sampler -> sm_set_input_target_f32_device -> Ndt.Align, against the host path; and the kept points
    through sm_calculate_normals"""
    lib = _lib.lib()
    tgt, src = scan[::2].copy(), S.scan(seed=3)[::6].copy()
    f = Sampler((0.3, 0.8, 10))
    host_out, _, rc = f.run(tgt)
    assert rc == 0
    _, idx, d_out = f.run_device(tgt)
    m = len(idx)
    assert m == len(host_out) and 0 < m < len(tgt)
    src3 = np.ascontiguousarray(src[:, :3])
    results = []
    for device_path in (True, False):
        h = C.c_void_p()
        assert lib.sm_create(5, 0, C.byref(h)) == 0                 # SM_TYPE_NDT
        assert lib.sm_set_input_source_f32(h, src3.ctypes.data, len(src3), 12) == 0
        if device_path:
            assert lib.sm_set_input_target_f32_device(h, d_out.data_ptr(), m, 20) == 0
        else:
            assert lib.sm_set_input_target_f32(h, host_out.ctypes.data, m, 20) == 0
        guess, res = np.asfortranarray(np.eye(4)), np.zeros(16)
        assert lib.sm_align(h, guess.ctypes.data_as(_lib._DP), res.ctypes.data_as(_lib._DP)) >= 0
        lib.sm_destroy(h)
        results.append(res)
    assert np.array_equal(results[0], results[1]) and not np.array_equal(results[0], np.eye(4).ravel())
    pts = np.asfortranarray(host_out[:, :3].astype(np.float64).T)
    out_p, out_n, k = np.zeros_like(pts), np.zeros_like(pts), C.c_int64(0)
    assert lib.sm_calculate_normals(0, pts.ctypes.data, m, out_p.ctypes.data,
                                    out_n.ctypes.data, C.byref(k)) == 0
    assert 0 < k.value <= m
