"""RandomSamplerWithPlaneDetect without a GPU: the raw stream, the closed-form ratio rule against the sampler's loop
for every k up to 2^24, the C++ restatement (oracle/plane_sampler_oracle.cc) against the numpy one
(tests/pyref_plane_sampler.py) on clouds built against each rule, the host builds of the single-hypothesis pieces
against the oracle's, and the ABI's argument checks."""
import ctypes as C

import numpy as np
import pytest

import oracle_plane_sampler as OP
import plane_sampler_scenes as S
import pyref_plane_sampler as PR
from staticmapping_b200 import _lib

F32 = np.float32
K_MAX = 1 << 24
NAN = float("nan")


def test_raw_stream_is_numpys_mt19937():
    words = OP.raw_stream()
    ref = np.random.RandomState(12345)._bit_generator.random_raw(OP.RAW_WORDS).astype(np.uint32)
    assert np.array_equal(words, ref)
    assert words[0] == 3992670690                      # std::mt19937(12345)'s first output
    assert np.array_equal(PR.RND, (words >> 1).astype(np.int64))
    # boost::uniform_int<int>(0, INT_MAX) over a 32-bit engine: brange = 2^32 - 1, bucket_size = 2, so engine() / 2
    assert int(PR.RND.max()) <= (1 << 31) - 1


def _rates():
    rng = np.random.default_rng(5)
    fixed = [0.5, 0.1, float(F32(1 / 3)), 1e-6, 0.999999, float(np.nextafter(F32(0.5), F32(0))),
             float(np.nextafter(F32(0.25), F32(1)))]
    return fixed + [float(F32(r)) for r in rng.uniform(1e-6, 0.999999, 12)]


@pytest.mark.parametrize("rate", _rates())
def test_closed_form_equals_the_loop_up_to_2_24(rate):
    loop = OP.keep_loop(rate, K_MAX)
    closed = np.empty(K_MAX, np.uint8)
    assert _lib.lib().sm_debug_plane_sampler_keep_host(float(rate), 1, K_MAX + 1, closed.ctypes.data) == 0
    assert np.array_equal(loop, closed.astype(bool))


def test_closed_form_on_a_nan_rate_keeps_nothing():
    out = np.ones(1000, np.uint8)
    assert _lib.lib().sm_debug_plane_sampler_keep_host(float("nan"), 1, 1001, out.ctypes.data) == 0
    assert not out.any() and not OP.keep_loop(float("nan"), 1000).any()


def _same(a, b):
    assert np.array_equal(a.keep, b.keep)
    assert np.array_equal(a.plane, b.plane)
    assert a.traces.tobytes() == b.traces.tobytes()


@pytest.mark.parametrize("name", sorted(S.scenes()))
def test_oracle_against_numpy(name):
    rec, params = S.scenes()[name]
    for p in params:
        _same(OP.plane_sampler(rec, *p), PR.plane_sampler(rec, *p))


def test_scene_rules():
    o = OP.plane_sampler(S.flat_ground(), *S.DEFAULT)
    st = o.traces["status"]
    assert list(st).count(1) == 7 and list(st).count(2) >= 1 and list(st).count(0) >= 1     # voxels split at borders
    o = OP.plane_sampler(S.walls(), *S.DEFAULT)
    assert np.all(o.traces["status"] == 4) and len(o.plane) == len(S.walls())
    o = OP.plane_sampler(S.noisy_planes(), *S.DEFAULT)
    assert list(o.traces["status"]) == [4, 4, 5, 5, 4]
    assert list(o.traces["final_count"][:4]) == [90, 85, 84, 80]
    o = OP.plane_sampler(S.degenerate(), *S.DEFAULT)
    t = o.traces                             # map order: (10, 0), (10, 2), (12, 0), (12, 2), (13, 0)
    assert list(t["status"]) == [4, 5, 4, 3, 5]
    assert t["best"][0] == 25 and t["iterations"][0] == 1 and t["final_count"][0] == 25      # identical points
    assert t["best"][4] == 25 and t["iterations"][4] == 1 and np.all(np.isnan(t["coef"][4]))  # ... zero covariance
    assert t["best"][1] == -(2 ** 31 - 1) and t["iterations"][1] == 0                          # collinear
    assert OP.plane_sampler(S.degenerate(), 0.5, 0.8, 11).traces["status"][2] == 3           # 20 < 2 * 11
    o = OP.plane_sampler(S.nan_x(), *S.DEFAULT)
    assert o.traces["status"][0] == 5 and o.traces["iterations"][0] == 51 and o.traces["best"][0] == 0
    for leaf in (0.2, 0.1):
        o = OP.plane_sampler(S.walls(), 0.5, leaf, 10)
        assert len(o.plane) == 0 and len(o.traces) == 0
    assert OP.plane_sampler(S.walls(), 1.0, 0.8, 10).keep.all()
    o = OP.plane_sampler(S.walls()[:0], *S.DEFAULT)
    assert len(o.keep) == 0 and len(o.plane) == 0


def test_scan_oracle_against_numpy():
    rec = S.scan(n_az=300)
    for p in (S.DEFAULT, (0.1, 0.8, 10), (0.5, 0.5, 5)):
        _same(OP.plane_sampler(rec, *p), PR.plane_sampler(rec, *p))


def _host(op, values):
    out = np.zeros(4, F32)
    v = np.ascontiguousarray(values, F32)
    assert _lib.lib().sm_debug_plane_sampler_piece_host(op, v.ctypes.data, out.ctypes.data) == 0
    return out


def test_host_pieces_against_the_oracle():
    rng = np.random.default_rng(11)
    pts = [rng.normal(0, 3, 9), np.zeros(9), np.tile([1.0, 2.0, 3.0], 3),
           np.array([0, 0, 0, 1 / 4, 1 / 2, 1, 1 / 2, 1, 2]), np.array([0, 0, 0, 1, 0, 0, 2, 0, 0]),
           np.array([NAN, 0, 0, 1, 1, 0, 2, 0, 1])]
    pts += [rng.normal(0, 1, 9) * 10.0 ** rng.integers(-3, 4) for _ in range(200)]
    for p in pts:
        for op in (0, 1):
            a, b = _host(op, p), OP.piece(op, p)
            assert a.tobytes() == b.tobytes(), (op, p)
        c = OP.piece(1, p)
        for q in rng.normal(0, 3, (5, 3)):
            v = np.r_[c, q]
            assert _host(2, v)[:2].tobytes() == OP.piece(2, v)[:2].tobytes()
    for _ in range(300):
        a = rng.normal(0, 1, (3, 3)) * 10.0 ** rng.integers(-4, 3)
        cov = (a @ a.T).astype(F32)
        if rng.integers(0, 4) == 0:
            cov[2, :] = cov[:, 2] = 0
        assert _host(3, cov.ravel())[:3].tobytes() == OP.piece(3, cov.ravel())[:3].tobytes()
        assert np.array_equal(np.array(PR.eigen33(cov), F32), OP.piece(3, cov.ravel())[:3])
    for cov in (np.zeros(9), np.eye(3).ravel(), np.diag([1.0, 1.0, 0.0]).ravel()):
        assert _host(3, cov)[:3].tobytes() == OP.piece(3, cov)[:3].tobytes()


def _nan_eq(a, b):
    return np.array_equal(np.asarray(a, F32), np.asarray(b, F32), equal_nan=True)


def test_numpy_pieces_against_the_oracle():
    rng = np.random.default_rng(12)
    for _ in range(200):
        p = (rng.normal(0, 2, 9)).astype(F32)
        trip = [tuple(p[3 * k:3 * k + 3]) for k in range(3)]
        assert PR.sample_good(*trip) == bool(OP.piece(0, p)[0])
        assert _nan_eq(PR.model(*trip), OP.piece(1, p))


def test_abi_arguments_and_no_device():
    lib = _lib.lib()
    h = C.c_void_p()
    assert lib.sm_plane_sampler_create(-1, C.byref(h)) == -1
    assert lib.sm_plane_sampler_create(0, None) == -1
    assert lib.sm_plane_sampler_create(0, C.byref(h)) == 0
    try:
        assert lib.sm_plane_sampler_set_sampling_rate(h, 2.0) == 0
        assert b"large than 1" in lib.sm_plane_sampler_last_error(h)
        assert lib.sm_plane_sampler_set_sampling_rate(h, 1e-7) == 0
        assert b"less than 1.e-6" in lib.sm_plane_sampler_last_error(h)
        assert lib.sm_plane_sampler_set_sampling_rate(h, 0.5) == 0 and lib.sm_plane_sampler_last_error(h) == b""
        assert lib.sm_plane_sampler_set_min_point_num_in_voxel(h, 4) == 0
        assert b"reset to default minimum : 5" in lib.sm_plane_sampler_last_error(h)
        assert lib.sm_plane_sampler_set_leaf_size(h, 0.1) == 0 and lib.sm_plane_sampler_last_error(h) == b""
        for fn in ("set_sampling_rate", "set_leaf_size"):
            assert getattr(lib, "sm_plane_sampler_" + fn)(None, 0.5) == -1
        assert lib.sm_plane_sampler_set_min_point_num_in_voxel(None, 10) == -1
        pts = np.zeros((100, 5), F32)
        out = np.zeros((100, 5), F32)
        m = C.c_int64(-7)
        run = lambda n, stride, p=pts.ctypes.data, o=out.ctypes.data: lib.sm_plane_sampler_run(  # noqa: E731
            h, p, n, stride, o, C.byref(m), None)
        assert run(100, 16) == -1 and run(100, 22) == -1 and run(-1, 20) == -1
        assert run(100, 20, p=None) == -1 and run(100, 20, o=None) == -1
        assert run(K_MAX + 1, 20) == -1 and b"2^24" in lib.sm_plane_sampler_last_error(h)
        assert lib.sm_plane_sampler_run_device(h, pts.ctypes.data, K_MAX + 1, 20, out.ctypes.data, C.byref(m), None,
                                               None) == -1
        assert lib.sm_plane_sampler_run(h, pts.ctypes.data, 100, 20, out.ctypes.data, None, None) == -1
        assert m.value == -7
        ni, no, npl = C.c_int64(-7), C.c_int64(-7), C.c_int64(-7)
        assert lib.sm_plane_sampler_indices(h, None, C.byref(ni), None, C.byref(no)) == 0
        assert lib.sm_plane_sampler_plane_indices(h, None, C.byref(npl)) == 0
        assert ni.value == 0 and no.value == 0 and npl.value == 0                     # before any run
        assert lib.sm_plane_sampler_indices(h, None, None, None, C.byref(no)) == -1
        assert lib.sm_plane_sampler_plane_indices(h, None, None) == -1
        assert lib.sm_plane_sampler_plane_indices(None, None, C.byref(npl)) == -1
        if lib.sm_device_count() == 0:
            assert run(100, 20) == -20 and b"no CUDA device" in lib.sm_plane_sampler_last_error(h)
            assert m.value == -7
    finally:
        assert lib.sm_plane_sampler_destroy(h) == 0
    assert lib.sm_plane_sampler_destroy(None) == -1
    assert lib.sm_debug_plane_sampler_keep_host(0.5, 0, 3, out.ctypes.data) == -1          # k starts at 1
    assert lib.sm_debug_plane_sampler_keep_host(0.5, 1, K_MAX + 2, out.ctypes.data) == -1
    assert lib.sm_debug_plane_sampler_piece_host(4, out.ctypes.data, out.ctypes.data) == -1


def test_python_mirror_clamps_like_the_setters():
    import staticmapping_b200 as smb
    s = smb.RandomSamplerWithPlaneDetect()
    s.SetSamplingRate(3.0)
    s.SetSamplingRate(0.0)
    s.SetMinPointNumInVoxel(2)
    s.SetLeafSize(0.8)
    assert len(s.messages) == 3
    assert OP.clamp_rate(3.0) == 1.0 and OP.clamp_rate(0.0) == F32(1e-6)
    assert s.Filter() is None
