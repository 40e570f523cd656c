"""Edge cases through the C ABI: tiny and ragged clouds, root-is-a-leaf trees, clouds smaller
than GICP's k, no searchable NDT voxel, far-away queries (deep stacks)."""
import numpy as np
import pytest

import oracle_lib as O
import scenes
import staticmapping_b200 as smb

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("nt", [1, 2, 7, 8, 9, 15, 16, 17, 33])
def test_knn_tiny_targets(nt):
    rng = np.random.default_rng(nt)
    T = rng.normal(size=(nt, 3))
    Q = np.concatenate([rng.normal(size=(50, 3)), rng.normal(size=(5, 3)) * 1e3], axis=0)
    for eps in (0.0, 3.16):
        io, do = O.knn1(T, Q, epsilon=eps)
        ig, dg = smb.knn1(T, Q, epsilon=eps)
        assert np.array_equal(ig, io) and np.array_equal(dg, do)


def test_knn_far_queries_exact():
    rng = np.random.default_rng(3)
    T = rng.uniform(-1, 1, size=(50000, 3))
    Q = rng.uniform(-1, 1, size=(200, 3)) * 1e4          # far outside: weak pruning, deep stacks
    io, do = O.knn1(T, Q, epsilon=0.0)
    ig, dg = smb.knn1(T, Q, epsilon=0.0)
    assert np.array_equal(ig, io) and np.array_equal(dg, do)


@pytest.mark.parametrize("ns,nt_raw", [(1, 200), (5, 64), (33, 500), (1000, 57)])
def test_icp_ragged_sizes(ns, nt_raw):
    src_all, tgt_all, _ = scenes.corner_pair()
    tp, tn = O.calculate_normals(tgt_all[:nt_raw])
    if tp.shape[0] == 0:
        pytest.skip("no valid leaf")
    src = src_all[:ns]
    m = smb.IcpFast()
    m.InitWithXml({"max_iteration": 12})
    m.SetInputSource(smb.EigenCloud(src))
    m.SetInputTarget(smb.EigenCloud(tp, tn))
    ok, res = m.Align(np.eye(4))
    o = O.icp_fast_align(src, tp, tn, max_iteration=12)
    assert o["rc"] == 1 and ok
    assert m.GetAlignInfo()["iterations"] == o["iterations"]
    fin = np.isfinite(o["result"])
    assert np.array_equal(fin, np.isfinite(res))
    assert np.allclose(res[fin], o["result"][fin], atol=1e-6)


def test_icp_reuse_handle_with_changing_sizes():
    src_all, tgt_all, _ = scenes.corner_pair()
    m = smb.IcpFast()
    for ns, nt_raw in [(4000, 5000), (100, 600), (5000, 3000), (17, 5000)]:
        tp, tn = O.calculate_normals(tgt_all[:nt_raw])
        m.SetInputSource(smb.EigenCloud(src_all[:ns]))
        m.SetInputTarget(smb.EigenCloud(tp, tn))
        ok, res = m.Align(np.eye(4))
        o = O.icp_fast_align(src_all[:ns], tp, tn)
        dt, dr = scenes.se3_error(o["result"], res)
        assert dt <= 1e-4 and dr <= 1e-4 and m.GetAlignInfo()["iterations"] == o["iterations"]


def _pm_align(m, src, tgt):
    m.SetInputSource(smb.InnerCloud(src))
    m.SetInputTarget(smb.InnerCloud(tgt))
    ok, res = m.Align(np.eye(4))
    info = m.GetAlignInfo()
    return ok, res, m.GetFitnessScore(), info["iterations"], list(info["aux"][:4])


def test_icp_pm_reuse_handle_with_changing_sizes():
    # one type-1 handle keeps its normals pipeline, sampling and score buffers across targets and sources that
    # grow and then shrink: every step must give exactly what a fresh handle gives
    src_all, sub_all, _ = scenes.lidar_pair(pair=1)
    rng = np.random.default_rng(5)
    m = smb.IcpUsingPointMatcher()
    for ns, nt in [(1500, 6000), (4000, 25000), (src_all.shape[0], sub_all.shape[0]), (3000, 15000), (800, 3000)]:
        src = src_all[np.sort(rng.choice(src_all.shape[0], ns, replace=False))].astype(np.float32)
        tgt = sub_all[np.sort(rng.choice(sub_all.shape[0], nt, replace=False))].astype(np.float32)
        reused = _pm_align(m, src, tgt)
        fresh = _pm_align(smb.IcpUsingPointMatcher(), src, tgt)
        assert reused[0] == fresh[0] and np.array_equal(reused[1], fresh[1]), (ns, nt)
        assert reused[2:] == fresh[2:], (ns, nt, reused[2:], fresh[2:])


def test_normals_tiny_inputs():
    rng = np.random.default_rng(0)
    for n in (1, 2, 3, 6, 7, 8, 13):
        pts = rng.uniform(1, 5, size=(n, 3))
        op, on = O.calculate_normals(pts)
        g = smb.CalculateNormals(pts)
        assert g.points.shape == op.shape and np.array_equal(g.points, op) and np.array_equal(g.normals, on)


def test_ndt_no_searchable_voxel():
    # fewer than 6 points per voxel everywhere: no neighbours, zero Hessian, Newton step is 0/NaN
    rng = np.random.default_rng(1)
    tgt = (rng.uniform(0, 40, size=(60, 3))).astype(np.float32)
    src = (rng.uniform(0, 40, size=(30, 3))).astype(np.float32)
    m = smb.Ndt()
    m.SetInputSource(smb.InnerCloud(src)); m.SetInputTarget(smb.InnerCloud(tgt))
    ok, res = m.Align(np.eye(4))
    o = O.ndt_align(src, tgt)
    assert ok and o["rc"] == 1 and m.GetAlignInfo()["iterations"] == o["iterations"]
    assert np.allclose(res, o["result"], atol=1e-7)
    assert abs(m.GetFitnessScore() - o["fitness"]) <= 1e-9 * max(1.0, o["fitness"])


def test_ndt_gicp_cloud_smaller_than_k():
    # k_correspondences (20) > cloud size: covariances stay unset (gicp_omp_impl.hpp:61-65)
    src, sub, _ = scenes.lidar_pair(pair=0)
    s = src[:15].astype(np.float32); t = sub[:4000].astype(np.float32)
    xml = '<r><param name="using_voxel_filter">0</param></r>'
    m = smb.CreateMatcher(smb.MatcherOptions(type=smb.Type.kNdtWithGicp, registrator_options_node=xml))
    m.SetInputSource(smb.InnerCloud(s)); m.SetInputTarget(smb.InnerCloud(t))
    o = O.ndt_gicp_align(s, t, using_voxel_filter=False)
    try:
        ok, res = m.Align(np.eye(4))
    except smb.CheckFailure:
        pytest.fail("engine failed where the oracle returned")
    assert bool(o["rc"]) == ok
    fin = np.isfinite(o["result"])
    assert np.array_equal(fin, np.isfinite(res)) and np.allclose(res[fin], o["result"][fin], atol=1e-4)
