"""The IcpUsingPointMatcher stand-in (type 1) with libpointmatcher's eigenvector surface normals on the GPU
(sm_set_pm_surface_normals): the reference filter stage bit for bit against the oracle
(oracle/pm_surface_normals_oracle.cc), Align against the oracle's chain, mode switching, the C++ adapter, and how far
each mode lies from the literal restatement of libpointmatcher's filter (tests/pyref.py) once both sample the reading
cloud with the same hash."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import oracle_pm_surface_normals as PN
import oracle_point_to_point as OP
import pyref
import scenes
import staticmapping_b200 as smb
from cxx import adapter_exe
from staticmapping_b200 import _lib, synth

pytestmark = pytest.mark.gpu

F32 = np.float32
LS, EV = smb.SurfaceNormals.LEAST_SQUARES, smb.SurfaceNormals.EIGENVECTOR


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def device_filter(cloud, mode, first=None):
    """sm_debug_pm_surface_normals -> (points (m,3), normals (m,3), smallest member index (m,))."""
    c = np.ascontiguousarray(cloud, F32)
    f = None if first is None else np.ascontiguousarray(first, F32)
    n = c.shape[0]
    pts = np.zeros((n, 3)); nrm = np.zeros((n, 3)); idx = np.zeros(n, np.int64); m = C.c_int64(-1)
    rc = _lib.lib().sm_debug_pm_surface_normals(0, int(mode), None if f is None else f.ctypes.data,
                                                0 if f is None else f.shape[0], c.ctypes.data, n, pts.ctypes.data,
                                                nrm.ctypes.data, idx.ctypes.data, C.byref(m))
    assert rc == 0
    return pts[:m.value], nrm[:m.value], idx[:m.value]


def check_stage(cloud, first=None):
    gp, gn, gi = device_filter(cloud, EV, first)
    om, on, oi = PN.pm_surface_normals(cloud)
    assert gp.shape == om.shape and np.array_equal(gi, oi)
    assert _bits(gp).tobytes() == _bits(om.astype(np.float64)).tobytes()
    assert _bits(gn).tobytes() == _bits(on.astype(np.float64)).tobytes()
    return gp.shape[0]


def lidar_cloud(n, seed=3):
    scan = synth.lidar_scan(synth.make_scene(seed=seed), seed=seed, n_az=1000).astype(np.float64)
    reps = -(-n // scan.shape[0])
    return np.concatenate([scan + np.array([0.0, 0.0, 40.0 * r]) for r in range(reps)])[:n].astype(F32)


# ------------------------------------------------------------------------------------------------ the stage
# the compaction tile (2048 keep flags), the k-d builder's bucket-7 capacities and its launch-path changes
# (separate block-sum scan past 524 288 points, more than 32 scan chunks past 1 048 576 sort keys), up to 2.1 M points
STAGE_SIZES = [1, 2, 3, 7, 8, 2047, 2048, 2049, 4097, 524_288, 524_289, 917_505, 1_048_577, 2_100_003]


@pytest.mark.parametrize("n", STAGE_SIZES)
def test_stage_against_the_oracle(n):
    rng = np.random.default_rng(n)
    cloud = lidar_cloud(n) if n > 10_000 else rng.uniform(-5, 5, size=(n, 3)).astype(F32)
    m = check_stage(cloud)
    assert (m == 0) if n <= 2 else (m > 0)


def test_stage_on_the_benchmark_submap():
    _, sub, _ = scenes.full_size_pair(0)
    assert check_stage(sub.astype(F32)) > 50_000


def test_stage_with_degenerate_boxes():
    """duplicates, lines and far-from-origin boxes: dropped and kept boxes as the oracle decides"""
    rng = np.random.default_rng(5)
    base = rng.uniform(-1, 1, size=(3000, 3)).astype(F32)
    dup = np.repeat(base[:500], 7, axis=0)                           # coincident members
    line = np.zeros((2000, 3), F32); line[:, 0] = np.arange(2000, dtype=F32) * F32(0.01)   # exactly collinear
    far = (base + F32(2e4)).astype(F32)
    for cloud in (dup, line, far, np.concatenate([dup, line, far])):
        check_stage(cloud)


def test_second_cloud_into_the_same_owner():
    big, small = lidar_cloud(600_000), lidar_cloud(3000, seed=4) + F32(0.5)
    check_stage(small, first=big)
    check_stage(big, first=small)


def test_least_squares_mode_is_calculate_normals():
    for cloud in (lidar_cloud(20_000), scenes.full_size_pair(1)[1].astype(F32)):
        gp, gn, _ = device_filter(cloud, LS)
        want = smb.CalculateNormals(cloud.astype(np.float64))
        assert _bits(gp).tobytes() == _bits(want.points).tobytes()
        assert _bits(gn).tobytes() == _bits(want.normals).tobytes()


# ------------------------------------------------------------------------------------------------ Align
def _matcher(src, tgt, mode=None, p2p=False):
    m = smb.IcpUsingPointMatcher(0)
    if mode is not None:
        m.SetSurfaceNormals(mode)
    if p2p:
        m.SetErrorMinimizer(smb.ErrorMinimizer.POINT_TO_POINT)
    m.SetInputSource(smb.InnerCloud(src))
    m.SetInputTarget(smb.InnerCloud(tgt))
    return m


def _pairs():
    src, tgt, _ = scenes.corner_pair()
    yield src.astype(F32), tgt.astype(F32)
    for pair in (0, 1):
        src, sub, _ = scenes.lidar_pair(pair=pair)
        yield src.astype(F32), sub.astype(F32)


def _check_against(m, ok, res, o):
    info = m.GetAlignInfo()
    assert o["rc"] == 1 and ok == o["ok"]
    assert int(info["aux"][2]) == o["n_source"] and int(info["aux"][3]) == o["n_target"]
    assert info["iterations"] == o["iterations"]
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= 1e-9 and dr <= 1e-9, (dt, dr)
    assert abs(m.GetFitnessScore() - o["score"]) < 1e-12


def test_align_eigenvector_mode_against_the_oracle_chain():
    for src, tgt in _pairs():
        m = _matcher(src, tgt, EV)
        ok, res = m.Align(np.eye(4))
        _check_against(m, ok, res, PN.icp_pm_equivalent(src, tgt, normals="eigenvector"))


def test_align_eigenvector_mode_point_to_point():
    for src, tgt in list(_pairs())[:2]:
        m = _matcher(src, tgt, EV, p2p=True)
        ok, res = m.Align(np.eye(4))
        tp, _, _ = PN.pm_surface_normals(tgt)
        keep = O.pm_keep_mask(src.shape[0])
        o = OP.icp_fast_align(src[keep].astype(np.float64), tp.astype(np.float64), None, max_iteration=150)
        _, d2 = O.knn1(tgt.astype(np.float64), O.pm_moved(src, o["result"]), epsilon=3.16)
        v, _, kept = O.pm_score_trim(d2)
        score = float(np.exp(-(np.sqrt(v[:kept]).sum() / kept)))
        assert m.GetAlignInfo()["iterations"] == o["iterations"] and m.GetAlignInfo()["solve_path"] in (3, 4)
        assert int(m.GetAlignInfo()["aux"][3]) == tp.shape[0]
        dt, dr = scenes.se3_error(o["result"], res)
        assert dt <= 1e-9 and dr <= 1e-9, (dt, dr)
        assert abs(m.GetFitnessScore() - score) < 1e-12 and ok == (score >= float(F32(0.6)))


def test_align_batch_with_both_modes():
    src, tgt = list(_pairs())[1]
    singles = []
    for mode in (EV, LS, EV, LS):
        m = _matcher(src, tgt, mode)
        singles.append((m.Align(np.eye(4)), m.GetFitnessScore()))
    ms = [_matcher(src, tgt, mode) for mode in (EV, LS, EV, LS)]
    oks, rb = smb.AlignBatch(ms, [np.eye(4)] * 4)
    for k in range(4):
        (ok, r), score = singles[k]
        assert oks[k] == ok and rb[k].tobytes() == r.tobytes() and ms[k].GetFitnessScore() == score
    assert not np.array_equal(rb[0], rb[1])
    o = PN.icp_pm_equivalent(src, tgt, normals="eigenvector")
    dt, dr = scenes.se3_error(o["result"], rb[0])
    assert dt <= 1e-9 and dr <= 1e-9


# ------------------------------------------------------------------------------------------------ mode switching
def test_switching_modes_gives_what_fresh_handles_give():
    src, tgt = list(_pairs())[0]
    fresh = {}
    for mode in (LS, EV):
        f = _matcher(src, tgt, mode)
        fresh[mode] = (f.Align(np.eye(4)), f.GetFitnessScore(), f.GetAlignInfo()["aux"][3])
    m = _matcher(src, tgt)
    for mode in (EV, LS, EV):
        m.SetSurfaceNormals(mode)
        (ok, r), score, nt = fresh[mode]
        ok2, r2 = m.Align(np.eye(4))
        assert ok2 == ok and r2.tobytes() == r.tobytes() and m.GetFitnessScore() == score
        assert m.GetAlignInfo()["aux"][3] == nt


def test_same_mode_twice_does_not_rebuild_the_target():
    src, tgt = list(_pairs())[0]
    m = _matcher(src, tgt, EV)
    ok, r = m.Align(np.eye(4))
    assert m.GetAlignInfo()["ms_upload"] > 0.0             # the filtered clouds went into the ICP chain
    m.SetSurfaceNormals(EV)
    ok2, r2 = m.Align(np.eye(4))
    assert m.GetAlignInfo()["ms_upload"] == 0.0            # nothing was filtered or uploaded again
    assert ok2 == ok and r2.tobytes() == r.tobytes()
    m.SetSurfaceNormals(LS)
    m.Align(np.eye(4))
    assert m.GetAlignInfo()["ms_upload"] > 0.0             # a change of mode filters the reference anew


def test_default_mode_is_byte_identical_to_a_handle_that_never_set_it():
    src, tgt = list(_pairs())[1]
    a = _matcher(src, tgt)
    b = _matcher(src, tgt, LS)
    ra, rb = a.Align(np.eye(4)), b.Align(np.eye(4))
    assert ra[0] == rb[0] and ra[1].tobytes() == rb[1].tobytes() and a.GetFitnessScore() == b.GetFitnessScore()
    o = O.icp_pm_equivalent(src, tgt)
    dt, dr = scenes.se3_error(o["result"], ra[1])
    assert dt <= 1e-9 and dr <= 1e-9


def test_other_types_and_bad_modes_are_rejected():
    lib = _lib.lib()
    src, tgt, _ = scenes.corner_pair()
    tp, tn = O.calculate_normals(tgt)
    f = smb.IcpFast(0)
    f.SetInputSource(smb.EigenCloud(src))
    f.SetInputTarget(smb.EigenCloud(tp, tn))
    _, r0 = f.Align(np.eye(4))
    assert lib.sm_set_pm_surface_normals(f._h, 1) == -11
    _, r1 = f.Align(np.eye(4))
    assert r1.tobytes() == r0.tobytes()
    for t in (3, 5):
        h = C.c_void_p()
        assert lib.sm_create(t, 0, C.byref(h)) == 0
        assert lib.sm_set_pm_surface_normals(h, 1) == -11
        lib.sm_destroy(h)
    m = _matcher(src.astype(F32), tgt.astype(F32), EV)
    _, e0 = m.Align(np.eye(4))
    for bad in (-1, 2, 7):
        assert lib.sm_set_pm_surface_normals(m._h, bad) == -1
    _, e1 = m.Align(np.eye(4))
    assert e1.tobytes() == e0.tobytes() and m.GetAlignInfo()["ms_upload"] == 0.0   # still eigenvector, not rebuilt
    with pytest.raises(smb.CheckFailure):
        m.SetSurfaceNormals(5)


# ------------------------------------------------------------------------------------------------ the adapter
def test_cpp_adapter(tmp_path):
    exe = adapter_exe(tmp_path, "pm_surface_normals_adapter_run")
    src, tgt = list(_pairs())[1]
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([src.shape[0], tgt.shape[0]], np.int64).tobytes())
        f.write(np.ascontiguousarray(src, F32).tobytes())
        f.write(np.ascontiguousarray(tgt, F32).tobytes())
    r = subprocess.run([exe, str(inp)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    out = {}
    for line in r.stdout.splitlines():
        k, *v = line.split()
        out[k] = np.array([float(x) for x in v])
    assert int(out["bad_value_rc"][0]) == -1
    for key, mode in (("least_squares", "least_squares"), ("eigenvector", "eigenvector"),
                      ("batch_eigenvector", "eigenvector"), ("batch_least_squares", "least_squares")):
        o = PN.icp_pm_equivalent(src, tgt, normals=mode)
        ok, score, T = out[key][0], out[key][1], out[key][2:].reshape(4, 4).T
        dt, dr = scenes.se3_error(o["result"], T)
        assert dt <= 1e-9 and dr <= 1e-9, (key, dt, dr)
        assert bool(ok) == o["ok"] and abs(score - o["score"]) < 1e-12
    assert out["batch_eigenvector"].tobytes() == out["eigenvector"].tobytes()


# ------------------------------------------------------------------------------------------------ the gain
def icp_pm_literal_hash(source_f32, target_f32, prob=0.9, seed=1):
    """pyref.icp_pm_literal with the engine's hash reading mask in place of rand(): libpointmatcher's literal
    reference filter (float sums, LAPACK eigh) and the chain in double, so that only the reference filter's leaf
    differs from the stand-in."""
    src = np.ascontiguousarray(source_f32, F32)
    tgt = np.ascontiguousarray(target_f32, F32)
    keep = O.pm_keep_mask(src.shape[0], prob, seed)
    tp, tn = pyref.pm_sampling_surface_normal(tgt, 7)
    kn = lambda t, q: O.knn1(t, q, epsilon=3.16)      # noqa: E731  (pinned bit-exact to pyref's search elsewhere)
    return pyref.icp_fast_align(src[keep].astype(np.float64), tp.astype(np.float64), tn.astype(np.float64),
                                max_iteration=150, knn=kn)


def test_eigenvector_mode_removes_the_reference_filter_difference():
    """Measured with the oracle's chain, which the stand-in matches to 1e-9: least-squares mode 0.15 - 0.90 mm and
    0.009 - 0.26 mrad from the literal chain; eigenvector mode 2.5e-9 - 9.6e-9 m and 1.8e-10 - 6.7e-10 rad, what is
    left of float LAPACK eigh against the double Jacobi."""
    for src, tgt in _pairs():
        lit = icp_pm_literal_hash(src, tgt)
        res = {}
        for mode in (LS, EV):
            m = _matcher(src, tgt, mode)
            _, res[mode] = m.Align(np.eye(4))
        dt_ls, _ = scenes.se3_error(lit["result"], res[LS])
        dt_ev, dr_ev = scenes.se3_error(lit["result"], res[EV])
        assert 5e-5 < dt_ls < 2e-3
        assert dt_ev < 1e-7 and dr_ev < 1e-8, (dt_ev, dr_ev)
        assert dt_ev < 1e-3 * dt_ls
