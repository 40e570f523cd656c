"""IcpFast and the IcpUsingPointMatcher stand-in with the point-to-point minimizer on the GPU
(sm_set_icp_error_minimizer) against the CPU oracle (oracle/icp_point_to_point_oracle.cc), through every entry
point, and the switch back to point-to-plane."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from cxx import adapter_exe
import inner_compensation_scenes as ICS
import oracle_lib as O
import oracle_point_to_point as OP
import point_to_point_scenes as S
import scenes
import staticmapping_b200 as smb

pytestmark = pytest.mark.gpu
P2P = smb.ErrorMinimizer.POINT_TO_POINT


def _matcher(src, tp, tn, p2p=True, comp=False, **opts):
    m = smb.IcpFast(0)
    for k, v in opts.items():
        m._check(m._lib.sm_set_option(m._h, k.encode(), str(v).encode()), k)
    if p2p:
        m.SetErrorMinimizer(P2P)
    if comp:
        m.EnableInnerCompensation()
    m.SetInputSource(smb.EigenCloud(src))
    m.SetInputTarget(smb.EigenCloud(tp, tn))
    return m


def _check_vs_oracle(m, src, tp, guess, comp=False, **kw):
    ok, res = m.Align(guess)
    o = OP.icp_fast_align(src, tp, guess, inner_compensation=comp, **kw)
    info = m.GetAlignInfo()
    assert ok and o["rc"] == 1
    assert info["iterations"] == o["iterations"]
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= 1e-9 and dr <= 1e-9, (dt, dr)
    assert abs(m.GetFitnessScore() - o["score"]) <= 1e-12
    assert info["solve_path"] in (3, 4)
    return res, o


@pytest.mark.parametrize("qpc", [0, 1024])
@pytest.mark.parametrize("graphs", [1, 0])
@pytest.mark.parametrize("name", list(S.UNIQUE))
def test_scene_matches_oracle(name, graphs, qpc):
    src, tp, tn, guess, mi = S.SCENES[name]()
    m = _matcher(src, tp, tn, knn_queries_per_cta=qpc, use_graphs=graphs, max_iteration=mi)
    _check_vs_oracle(m, src, tp, guess, max_iteration=mi)


def test_corner_every_iteration():
    src, tp, tn, guess, _ = S.corner()
    o = OP.icp_fast_align(src, tp, guess, trace=True)
    m = _matcher(src, tp, tn, disable_convergence_check=1)
    for k in range(1, o["iterations"] + 1):
        m._check(m._lib.sm_set_option(m._h, b"max_iteration", str(k).encode()), "opt")
        ok, res = m.Align(guess)
        info = m.GetAlignInfo()
        t = o["trace"][k - 1]
        assert info["kept"] == t["kept"] and info["solve_path"] == t["path"]
        assert abs(info["limit"] - t["limit"]) <= 1e-12 * t["limit"]   # T_iter differs by the centring's rounding


def test_reflection_fix_on_the_device():
    src, tp, tn, guess, _ = S.reflection()
    m = _matcher(src, tp, tn, max_iteration=1)
    _check_vs_oracle(m, src, tp, guess, max_iteration=1)
    assert m.GetAlignInfo()["solve_path"] == 4


def test_one_match_and_collinear():
    src, tp, tn, guess, _ = S.one_match()
    m = _matcher(src, tp, tn, max_iteration=1)
    ok, res = m.Align(guess)
    assert ok and m.GetAlignInfo()["kept"] == 1
    assert np.array_equal(res[:3, :3], np.eye(3))           # M = 0 exactly: R = I
    src, tp, tn, guess, _ = S.collinear()
    ok, res = _matcher(src, tp, tn).Align(guess)
    R = res[:3, :3]
    assert ok and np.abs(R.T @ R - np.eye(3)).max() <= 1e-12 and abs(np.linalg.det(R) - 1.0) <= 1e-12
    moved = src @ R.T + res[:3, 3]
    d = tp[-1] / np.linalg.norm(tp[-1])
    assert np.linalg.norm(moved - np.outer(moved @ d, d), axis=1).max() <= 1e-3


def test_full_size_pair_30_iterations():
    src, sub, _ = scenes.full_size_pair()
    tp, tn = O.calculate_normals(sub)
    m = _matcher(src, tp, tn, max_iteration=30)
    _check_vs_oracle(m, src, tp, np.eye(4), max_iteration=30)


def test_inner_compensation():
    src, tp, tn, guess, _ = ICS.model_exact()
    m = _matcher(src, tp, tn, comp=True)
    _check_vs_oracle(m, src, tp, guess, comp=True)


def test_entry_points_bit_identical():
    src, tp, tn, _, _ = S.corner()
    guess = ICS.se3(0.5, (0, 0, 1), (0.02, 0.01, 0.0))
    ref = _matcher(src, tp, tn)
    _, r0 = ref.Align(guess)
    s0 = ref.GetFitnessScore()
    a = _matcher(src, tp, tn)
    a.AlignAsync(guess)
    _, r1 = a.AlignWait()
    assert np.array_equal(r0, r1)
    for graphs in (1, 0):
        for qpc in (0, 1024):
            _, rg = _matcher(src, tp, tn, use_graphs=graphs, knn_queries_per_cta=qpc).Align(guess)
            assert np.array_equal(rg, r0)
            ms = [_matcher(src, tp, tn, p2p=(k % 2 == 0), knn_queries_per_cta=qpc, use_graphs=graphs) for k in range(4)]
            oks, rb = smb.AlignBatch(ms, [guess] * 4)
            assert all(oks) and np.array_equal(rb[0], r0) and np.array_equal(rb[2], r0)
            _, rp = _matcher(src, tp, tn, p2p=False).Align(guess)
            assert np.array_equal(rb[1], rp) and np.array_equal(rb[3], rp) and not np.array_equal(rp, r0)
            pairs = [dict(source=src, target=tp, normals=tn, guess=guess)] * 3
            hs = [_matcher(src, tp, tn, knn_queries_per_cta=qpc, use_graphs=graphs) for _ in range(2)]
            rcs, rr, sc = smb.AlignPairs(hs, pairs)
            assert (rcs == 1).all()
            for k in range(3):
                assert np.array_equal(rr[k], r0) and sc[k] == s0


def test_switching_back_to_point_to_plane():
    src, tp, tn, _, _ = S.corner()
    fresh = _matcher(src, tp, tn, p2p=False)
    _, plane = fresh.Align(np.eye(4))
    info_plane = fresh.GetAlignInfo()
    m = _matcher(src, tp, tn)
    _, p2p = m.Align(np.eye(4))
    assert m.GetAlignInfo()["solve_path"] in (3, 4) and not np.array_equal(p2p, plane)
    m.SetErrorMinimizer(smb.ErrorMinimizer.POINT_TO_PLANE)
    _, back = m.Align(np.eye(4))
    assert back.tobytes() == plane.tobytes() and m.GetFitnessScore() == fresh.GetFitnessScore()
    assert m.GetAlignInfo()["solve_path"] == info_plane["solve_path"] <= 2
    m.SetErrorMinimizer(P2P)
    _, again = m.Align(np.eye(4))
    assert again.tobytes() == p2p.tobytes()


def test_icp_pm_stand_in():
    src, sub, _ = scenes.lidar_pair()
    m = smb.IcpUsingPointMatcher(0)
    m.SetErrorMinimizer(P2P)
    m.SetInputSource(smb.InnerCloud(src))
    m.SetInputTarget(smb.InnerCloud(sub))
    ok, res = m.Align(np.eye(4))
    o = OP.icp_pm_equivalent(src, sub)
    assert o["rc"] == 1 and ok == o["ok"]
    assert m.GetAlignInfo()["iterations"] == o["iterations"] and m.GetAlignInfo()["solve_path"] in (3, 4)
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= 1e-9 and dr <= 1e-9, (dt, dr)
    assert abs(m.GetFitnessScore() - o["score"]) < 1e-9


def test_rejections():
    lib = smb.IcpFast(0)._lib
    for t in (3, 5):
        h = C.c_void_p()
        assert lib.sm_create(t, 0, C.byref(h)) == 0
        assert lib.sm_set_icp_error_minimizer(h, 1) == -11
        lib.sm_destroy(h)
    src, tp, tn, guess, _ = S.corner()
    m = _matcher(src, tp, tn)
    _, r0 = m.Align(guess)
    for bad in (-1, 2, 7):
        assert m._lib.sm_set_icp_error_minimizer(m._h, bad) == -1
    _, r1 = m.Align(guess)
    assert np.array_equal(r0, r1) and m.GetAlignInfo()["solve_path"] in (3, 4)   # still point-to-point
    with pytest.raises(Exception):
        m.SetErrorMinimizer(5)


def test_cpp_adapter(tmp_path):
    exe = adapter_exe(tmp_path, "adapter_point_to_point_run", overlay="stubs_inner_compensation")
    src, tp, tn, _, _ = S.corner()
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([src.shape[0], tp.shape[0]], np.int64).tobytes())
        for a in (src, tp, tn):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    r = subprocess.run([exe, str(inp)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    rows = {ln.split()[0]: np.array([float(v) for v in ln.split()[1:]]) for ln in r.stdout.splitlines()}
    plane = O.icp_fast_align(src, tp, tn)
    p2p = OP.icp_fast_align(src, tp)
    for key, o in (("plane", plane), ("p2p", p2p), ("plane_again", plane), ("batch_p2p", p2p)):
        dt, dr = scenes.se3_error(o["result"], rows[key].reshape(4, 4, order="F"))
        assert dt <= 1e-9 and dr <= 1e-9, key
    assert rows["bad_value_rc"][0] == -1
