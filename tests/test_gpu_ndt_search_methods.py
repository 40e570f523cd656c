"""pclomp's neighbour searches of Ndt on the GPU (sm_set_ndt_search_method / Ndt.SetNeighborhoodSearchMethod): the
derivative stage of each method against the oracle at the oracle's own Newton iterates (test hook
sm_debug_ndt_derivatives_search), full Align at the benchmark's Ndt size and on edge clouds, the setter's switching,
batching and errors."""
import ctypes as C

import numpy as np
import pytest

import bench
import oracle_ndt_search as OS
import pyref
import pyref_ndt_search as PS
import scenes
import staticmapping_b200 as smb
from staticmapping_b200 import _lib
from test_gpu_ndt_gicp_stages import EXPF_ULPS, _LIBM, grid_degenerate, grid_invalid_leaf

pytestmark = pytest.mark.gpu

F32 = np.float32
M = smb.NeighborSearchMethod


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=F32))


def device_sums(source, target, poses, method):
    s, t = _f32(source), _f32(target)
    P = np.ascontiguousarray(np.atleast_2d(np.asarray(poses, dtype=np.float64)))
    out = np.zeros((P.shape[0], 44))
    rc = _lib.lib().sm_debug_ndt_derivatives_search(0, t.ctypes.data, t.shape[0], s.ctypes.data, s.shape[0], 1.0, 0.55,
                                                    int(method), P.ctypes.data, P.shape[0], out.ctypes.data)
    assert rc == 0
    return out


def oracle_sums(source, target, p, method):
    score, g, H, nb = OS.ndt_derivatives(source, target, p, int(method))
    return np.concatenate([[score], g, H.ravel(), [round(nb * len(source))]])


def _transformed(source, p):
    T = np.zeros(16)
    assert _lib.lib().sm_debug_ndt_host(1, np.ascontiguousarray(p, np.float64).ctypes.data, T.ctypes.data) == 0
    return pyref._transform_cloud_f32(T.reshape(4, 4).T.astype(F32), _f32(source))


def abs_scale(source, target, p, method):
    """The sums of the absolute (point, voxel) terms, from the numpy restatement over the device's transform."""
    grid = PS.SearchGrid(target, 1.0, int(method))
    score, g, H, _ = pyref.ndt_derivatives(grid, _f32(source), _transformed(source, p), p, absolute=True)
    return np.concatenate([[abs(score)], g, H.ravel()])


def expf_affected_terms(source, target, p, method):
    """(count, sum of |term|) of the (point, voxel) terms whose exponential differs between glibc's expf (the oracle)
    and float(exp(double)) (the device), as tests/test_gpu_ndt_gicp_stages.py locates them, for the method's pairs."""
    src = _f32(source)
    xt = _transformed(source, p)
    grid = PS.SearchGrid(target, 1.0, int(method))
    pi, li = grid.radius_search(xt)
    v = (xt[pi].astype(np.float64) - grid.mean[li]).astype(F32)
    ci = grid.icov[li].astype(F32)
    xc = [(v[:, 0] * ci[:, 0, c] + v[:, 1] * ci[:, 1, c]) + v[:, 2] * ci[:, 2, c] for c in range(3)]
    q = (v[:, 0] * xc[0] + v[:, 1] * xc[1]) + v[:, 2] * xc[2]
    arg = ((-F32(pyref.ndt_gauss_constants()[1])) * q) * F32(0.5)
    dev_e = np.exp(arg.astype(np.float64)).astype(F32)
    hit = [j for j in range(arg.size) if F32(_LIBM.expf(float(arg[j]))) != dev_e[j]]
    total = np.zeros(43)
    pp = np.ascontiguousarray(p, np.float64)
    for j in hit:
        out = np.zeros(43)
        assert _lib.lib().sm_debug_ndt_term(pp.ctypes.data, 0.55, 1.0, 0, src[pi[j]].ctypes.data,
                                            np.ascontiguousarray(xt[pi[j]]).ctypes.data,
                                            np.ascontiguousarray(grid.mean[li[j]]).ctypes.data,
                                            np.ascontiguousarray(grid.icov[li[j]]).ctypes.data, out.ctypes.data) == 0
        total += np.abs(out)
    return len(hit), total


def oracle_newton_iterates(source, target, method):
    """The pose vectors at which the oracle's Newton loop evaluates, with its sums (the product's host loop driven by
    the oracle's evaluation, sm_debug_ndt_newton)."""
    calls = []

    @C.CFUNCTYPE(C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_void_p)
    def evaluate(_T, p_ptr, sums_ptr, _user):
        p = np.array([p_ptr[i] for i in range(6)])
        s = oracle_sums(source, target, p, method)
        for i in range(44):
            sums_ptr[i] = s[i]
        calls.append(p)
        return 0

    final = np.zeros(16); it = C.c_int32(); ev = C.c_int32(); sc = C.c_double()
    guess = np.asfortranarray(np.eye(4))
    rc = _lib.lib().sm_debug_ndt_newton(evaluate, None, guess.ctypes.data, source.shape[0], 1.0, 0.1, 0.55, 0.1, 35,
                                        final.ctypes.data, C.byref(it), C.byref(ev), C.byref(sc))
    assert rc == 0 and ev.value == len(calls) >= 2
    return calls


def _lidar(pair):
    s, t, P = scenes.lidar_pair(pair=pair)
    return _f32(s), _f32(t), P


def _degenerate():
    t = grid_degenerate()
    return _f32(t[::3] + F32(0.3)), t


@pytest.mark.parametrize("method", list(M), ids=[m.name for m in M])
@pytest.mark.parametrize("scene", ["lidar-1", "degenerate"])
def test_stage_sums_at_the_oracles_newton_iterates(scene, method):
    source, target = (_lidar(1)[:2] if scene == "lidar-1" else _degenerate())
    poses = oracle_newton_iterates(source, target, method)
    dev = device_sums(source, target, np.stack(poses), method)
    for p, d in zip(poses, dev):
        ref = oracle_sums(source, target, p, method)
        assert d[43] == ref[43]
        scale = abs_scale(source, target, p, method)
        _, hit = expf_affected_terms(source, target, p, method)
        err = np.abs(d[:43] - ref[:43])
        assert np.all(err <= 1e-10 * scale + EXPF_ULPS * hit), np.max(err / np.maximum(scale, 1e-300))


def test_stage_invalid_leaf_is_a_kdtree_neighbour_only():
    target = grid_invalid_leaf()
    c = PS.SearchGrid(target).centroid[0].astype(np.float64)
    q = _f32([c + (0.5, 0.0, 0.0)])
    for method in M:
        d = device_sums(q, target, np.zeros(6), method)[0]
        assert np.array_equal(d, oracle_sums(q, target, np.zeros(6), method))
        assert d[43] == (1 if method == M.KDTREE else 0)


def _align(src, tgt, method=None, guess=None, handle=None):
    m = handle or smb.Ndt()
    if handle is None:
        m.SetInputSource(smb.InnerCloud(src))
        m.SetInputTarget(smb.InnerCloud(tgt))
    if method is not None:
        m.SetNeighborhoodSearchMethod(method)
    ok, res = m.Align(np.eye(4) if guess is None else guess)
    return ok, res, m.GetFitnessScore(), m.GetAlignInfo()


def assert_matches_oracle(src, tgt, method, ok, res, fit, info, pose_tol=1e-5, fit_tol=1e-6):
    o = OS.ndt_align(src, tgt, int(method))
    assert ok and o["rc"] == 1
    assert info["iterations"] == o["iterations"] and info["evaluations"] == o["evaluations"]
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= pose_tol and dr <= pose_tol, (dt, dr)
    assert abs(fit - o["fitness"]) <= fit_tol * max(1.0, o["fitness"])
    assert abs(info["mean_neighbors"] - o["mean_neighbors"]) <= fit_tol * max(1.0, o["mean_neighbors"])
    return o


@pytest.fixture(scope="module")
def config3():
    src, sub, P = bench.make_workload(0)
    return _f32(src), _f32(sub), P


@pytest.mark.parametrize("method", list(M), ids=[m.name for m in M])
def test_align_at_benchmark_size(config3, method):
    src, sub, P = config3
    ok, res, fit, info = _align(src, sub, method)
    assert_matches_oracle(src, sub, method, ok, res, fit, info)


@pytest.mark.parametrize("method", list(M), ids=[m.name for m in M])
@pytest.mark.parametrize("scene", ["lidar-0", "lidar-2", "degenerate"])
def test_align_on_edge_clouds(scene, method):
    src, tgt = _degenerate() if scene == "degenerate" else _lidar(int(scene[-1]))[:2]
    ok, res, fit, info = _align(src, tgt, method)
    # the degenerate cloud is mostly singular voxels (collinear, planar, repeated points): its Hessian is nearly
    # singular and the solve amplifies the one-ulp expf terms (see the stage test) into the pose.  Measured on an
    # H100: 6.6e-5 m with KDTREE, whose kernel is instruction for instruction the one before the direct searches,
    # and 1.3e-3 m with DIRECT1; iteration and evaluation counts are equal
    loose = scene == "degenerate"
    assert_matches_oracle(src, tgt, method, ok, res, fit, info, pose_tol=5e-3 if loose else 1e-5,
                          fit_tol=1e-2 if loose else 1e-6)


def test_explicit_kdtree_is_the_default_byte_for_byte():
    src, tgt, _ = _lidar(2)
    a = _align(src, tgt)
    b = _align(src, tgt, M.KDTREE)
    assert a[0] == b[0] and a[1].tobytes() == b[1].tobytes() and a[2] == b[2]
    for k in ("iterations", "evaluations", "trans_probability", "mean_neighbors"):
        assert a[3][k] == b[3][k], k


def test_switching_methods_on_one_handle_reproduces_each_result():
    src, tgt, _ = _lidar(0)
    fresh = {m: _align(src, tgt, m) for m in M}
    h = smb.Ndt()
    h.SetInputSource(smb.InnerCloud(src))
    h.SetInputTarget(smb.InnerCloud(tgt))
    for m in (M.DIRECT7, M.KDTREE, M.DIRECT1, M.DIRECT26, M.DIRECT7, M.KDTREE):
        r = _align(src, tgt, m, handle=h)
        assert r[1].tobytes() == fresh[m][1].tobytes() and r[2] == fresh[m][2]
        assert r[3]["evaluations"] == fresh[m][3]["evaluations"]


def test_align_batch_with_mixed_methods_equals_single_calls():
    src, tgt, _ = _lidar(1)
    methods = [M.KDTREE, M.DIRECT26, M.DIRECT7, M.DIRECT1, M.DIRECT7]
    handles = []
    for m in methods:
        h = smb.Ndt()
        h.SetInputSource(smb.InnerCloud(src))
        h.SetInputTarget(smb.InnerCloud(tgt))
        h.SetNeighborhoodSearchMethod(m)
        handles.append(h)
    oks, results = smb.AlignBatch(handles, [np.eye(4)] * len(handles))
    for m, ok, res in zip(methods, oks, results):
        single = _align(src, tgt, m)
        assert ok == single[0] and res.tobytes() == single[1].tobytes()


def test_errors():
    h = smb.Ndt()
    lib = _lib.lib()
    assert lib.sm_set_ndt_search_method(h._h, 4) == -1 and lib.sm_set_ndt_search_method(h._h, -1) == -1
    with pytest.raises(smb.CheckFailure):
        h.SetNeighborhoodSearchMethod(7)
    src, tgt, _ = _lidar(2)
    h.SetInputSource(smb.InnerCloud(src))
    h.SetInputTarget(smb.InnerCloud(tgt))
    assert h.Align(np.eye(4))[1].tobytes() == _align(src, tgt)[1].tobytes()   # the rejected values left KDTREE
    for cls in (smb.IcpUsingPointMatcher, smb.NdtWithGicp, smb.IcpFast):
        m = cls()
        assert lib.sm_set_ndt_search_method(m._h, 2) == -11
    with pytest.raises(smb.CheckFailure):
        smb.NdtWithGicp().SetNeighborhoodSearchMethod(M.DIRECT7)
    assert "search" not in smb.Ndt().PrintOptions()
