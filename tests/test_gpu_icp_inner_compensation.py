"""IcpFast with inner compensation on the GPU (sm_set_inner_compensation) against the CPU restatement
(tests/cpp/icp_compensation_oracle.cc), through every entry point."""
import os
import subprocess

import numpy as np
import pytest

import inner_compensation_scenes as ICS
import oracle_compensation as OC
import oracle_lib as O
import scenes
import staticmapping_b200 as smb

pytestmark = pytest.mark.gpu


def _matcher(src, tp, tn, comp=True, **opts):
    m = smb.IcpFast(0)
    for k, v in opts.items():
        m._check(m._lib.sm_set_option(m._h, k.encode(), str(v).encode()), k)
    if comp:
        m.EnableInnerCompensation()
    m.SetInputSource(smb.EigenCloud(src))
    m.SetInputTarget(smb.EigenCloud(tp, tn))
    return m


def _corner():
    src, _, _ = scenes.corner_pair()
    tp, tn = ICS.corner_target()
    return src, tp, tn


def _check_vs_oracle(m, src, tp, tn, guess, max_iteration=100, disable=False):
    ok, res = m.Align(guess)
    o = OC.icp_fast_align(src, tp, tn, guess, max_iteration=max_iteration, disable_convergence_check=disable)
    info = m.GetAlignInfo()
    assert ok and o["rc"] == 1
    assert info["iterations"] == o["iterations"]
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= 1e-9 and dr <= 1e-9, (dt, dr)
    assert abs(m.GetFitnessScore() - o["score"]) <= 1e-12 * abs(o["score"])
    return res, o


@pytest.mark.parametrize("qpc", [0, 1024])
@pytest.mark.parametrize("graphs", [1, 0])
def test_corner_scene_matches_oracle_every_iteration(qpc, graphs):
    src, tp, tn = _corner()
    m = _matcher(src, tp, tn, knn_queries_per_cta=qpc, use_graphs=graphs)
    _, o = _check_vs_oracle(m, src, tp, tn, np.eye(4))
    # the trace: the first k iterations alone, convergence test off, end in the oracle's k-th T_iter and kept count
    full = OC.icp_fast_align(src, tp, tn, np.eye(4), max_iteration=o["iterations"], disable_convergence_check=True,
                             trace=True)
    m._check(m._lib.sm_set_option(m._h, b"disable_convergence_check", b"1"), "opt")
    for k in range(1, o["iterations"] + 1):
        m._check(m._lib.sm_set_option(m._h, b"max_iteration", str(k).encode()), "opt")
        ok, _ = m.Align(np.eye(4))
        info = m.GetAlignInfo()
        assert ok and info["iterations"] == k
        assert info["kept"] == full["trace"][k - 1]["kept"]
        assert info["limit"] == pytest.approx(full["trace"][k - 1]["limit"], rel=1e-12, abs=0)


@pytest.mark.parametrize("disable", [False, True])
def test_full_size_matches_oracle(disable):
    src, tp, tn = scenes._lidar_with_normals(full_size=True)
    kw = dict(max_iteration=30, disable_convergence_check=1) if disable else {}
    m = _matcher(src, tp, tn, **kw)
    res, o = _check_vs_oracle(m, src, tp, tn, np.eye(4), max_iteration=30 if disable else 100, disable=disable)
    assert m.GetAlignInfo()["kept"] == OC.icp_fast_align(src, tp, tn, np.eye(4), max_iteration=o["iterations"],
                                                         disable_convergence_check=True, trace=True)["trace"][-1]["kept"]


def test_model_exact_scene_recovers_the_motion():
    src, tp, tn, G, expected = ICS.model_exact()
    m = _matcher(src, tp, tn)
    res, _ = _check_vs_oracle(m, src, tp, tn, G)
    dt, dr = scenes.se3_error(res, expected)
    assert dt <= 0.02 and dr <= np.radians(0.2)


def test_entry_points_agree_bit_for_bit():
    src, tp, tn = _corner()
    guess = ICS.se3(0.5, (0, 0, 1), (0.02, 0.01, 0.0))
    ref = _matcher(src, tp, tn)
    _, r0 = ref.Align(guess)
    s0 = ref.GetFitnessScore()
    a = _matcher(src, tp, tn)
    a.AlignAsync(guess)
    _, r1 = a.AlignWait()
    assert np.array_equal(r0, r1)
    for qpc in (0, 1024):
        ms = [_matcher(src, tp, tn, comp=(k % 2 == 0), knn_queries_per_cta=qpc) for k in range(4)]
        oks, rb = smb.AlignBatch(ms, [guess] * 4)
        assert all(oks)
        assert np.array_equal(rb[0], r0) and np.array_equal(rb[2], r0)      # compensated, either schedule
        plain = _matcher(src, tp, tn, comp=False)
        _, rp = plain.Align(guess)
        assert np.array_equal(rb[1], rp) and np.array_equal(rb[3], rp) and not np.array_equal(rp, r0)
        pairs = [dict(source=src, target=tp, normals=tn, guess=guess)] * 3
        rcs, rr, sc = smb.AlignPairs([_matcher(src, tp, tn, knn_queries_per_cta=qpc) for _ in range(2)], pairs)
        assert (rcs == 1).all()
        for k in range(3):
            assert np.array_equal(rr[k], r0) and sc[k] == s0


def test_toggling_recaptures_the_graphs():
    src, tp, tn = _corner()
    m = _matcher(src, tp, tn, comp=False)
    _, off1 = m.Align(np.eye(4))
    m.EnableInnerCompensation()
    _, on = m.Align(np.eye(4))
    m.DisableInnerCompensation()
    _, off2 = m.Align(np.eye(4))
    assert np.array_equal(off1, off2) and not np.array_equal(on, off1)
    _, fresh = _matcher(src, tp, tn).Align(np.eye(4))
    assert np.array_equal(on, fresh)


def test_one_point_source():
    _, tp, tn = _corner()
    src = tp[:1] + 0.01
    m = _matcher(src, tp, tn)
    ok, res = m.Align(np.eye(4))
    o = OC.icp_fast_align(src, tp, tn)
    assert ok and m.GetAlignInfo()["iterations"] == o["iterations"]
    assert np.array_equal(res, o["result"])


def test_identical_source_and_target():
    _, tp, tn = _corner()
    m = _matcher(tp, tp, tn)
    ok, res = m.Align(np.eye(4))
    o = OC.icp_fast_align(tp, tp, tn)
    assert ok and m.GetAlignInfo()["iterations"] == o["iterations"]
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= 1e-9 and dr <= 1e-9


def test_ndt_ignores_the_flag():
    src, sub, P = scenes.lidar_pair(pair=0)
    out = []
    for comp in (False, True):
        m = smb.Ndt()
        if comp:
            m.EnableInnerCompensation()
        m.SetInputSource(smb.InnerCloud(src))
        m.SetInputTarget(smb.InnerCloud(sub))
        out.append((m.Align(np.eye(4)), m.GetFitnessScore()))
    (ok0, r0), s0 = out[0]
    (ok1, r1), s1 = out[1]
    assert ok0 == ok1 and np.array_equal(r0, r1) and s0 == s1


def test_cpp_adapter_enable_inner_compensation(tmp_path):
    import test_adapter_cpp as A
    exe = str(tmp_path / "adapter_compensation_run")
    root = A.ROOT
    cmd = ["/usr/bin/g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(root, "tests", "stubs_inner_compensation"),
           "-I", os.path.join(root, "tests", "stubs"),
           "-I", os.path.join(root, "include"), "-I", os.path.join(root, "adapter"),
           os.path.join(root, "tests", "cpp", "adapter_compensation_run.cc"), "-o", exe,
           "-L", A.LIBDIR, "-l:libsm_b200.so", "-Wl,-rpath," + A.LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    src, tp, tn = _corner()
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([src.shape[0], tp.shape[0]], np.int64).tobytes())
        for a in (src, tp, tn):
            f.write(np.ascontiguousarray(a, np.float64).tobytes())
    r = subprocess.run([exe, str(inp)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    rows = {ln.split()[0]: np.array([float(v) for v in ln.split()[1:]]) for ln in r.stdout.splitlines()}
    plain = O.icp_fast_align(src, tp, tn)
    comp = OC.icp_fast_align(src, tp, tn)
    for key, o in (("plain", plain), ("comp", comp), ("plain_again", plain), ("batch_comp", comp)):
        dt, dr = scenes.se3_error(o["result"], rows[key].reshape(4, 4, order="F"))
        assert dt <= 1e-9 and dr <= 1e-9, key
    assert not np.array_equal(rows["plain"], rows["comp"])
