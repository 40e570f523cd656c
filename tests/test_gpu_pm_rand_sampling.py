"""The IcpUsingPointMatcher stand-in's rand reading sampler on the GPU (sm_set_pm_reading_sampler GLIBC_RAND): the
device filter bit for bit against glibc's own stream (oracle/pm_rand_oracle.cc), Align against the oracle's chain at
the same seed and position, against the literal chain of tests/pyref.py, the stream position across Aligns and
handles, and the C++ adapter."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import oracle_pm_rand as R
import oracle_pm_surface_normals as PN
import oracle_point_to_point as OP
import pyref
import scenes
import staticmapping_b200 as smb
from cxx import adapter_exe
from staticmapping_b200 import _lib

pytestmark = pytest.mark.gpu

F32 = np.float32
HASH, RAND = smb.ReadingSampler.HASH, smb.ReadingSampler.GLIBC_RAND
LS, EV = smb.SurfaceNormals.LEAST_SQUARES, smb.SurfaceNormals.EIGENVECTOR
SLICE = 992            # draws per generator thread (31 words of 32 flags)
BLOCK = 128 * SLICE    # draws per generator block


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def device_sample(pts, prob, seed, position):
    """sm_debug_pm_rand_sample -> (keep mask, kept points (m,3) double)"""
    p = np.ascontiguousarray(pts, F32)
    n = p.shape[0]
    kept = C.c_int64(-1)
    out = np.zeros((n, 3))
    keep = np.zeros(n, np.uint8)
    rc = _lib.lib().sm_debug_pm_rand_sample(0, p.ctypes.data, n, prob, seed, position, C.byref(kept), out.ctypes.data,
                                            keep.ctypes.data)
    assert rc == 0
    return keep.astype(bool), out[:kept.value]


def host_mask(n, prob, seed, position):
    """the filter's float expression on draws from the host build of the jump-ahead, for positions glibc's own
    random_r cannot reach in a test (the host build equals random_r wherever it can: test_pm_rand_sampling.py)"""
    d = np.zeros(n, np.int32)
    assert _lib.lib().sm_debug_pm_rand_draws_host(seed, position, n, d.ctypes.data) == 0
    return (d.astype(F32) / F32(2147483647)) < F32(prob)


def check_sample(pts, prob=0.9, seed=1, position=0, want=None):
    keep, got = device_sample(pts, prob, seed, position)
    if want is None:
        want = R.pm_rand_mask(pts.shape[0], prob, seed, position)
    assert np.array_equal(keep, want)
    assert _bits(got).tobytes() == _bits(pts[want].astype(np.float64)).tobytes()
    return int(want.sum())


def cloud(n, seed=0):
    return np.random.default_rng(seed).uniform(-50, 50, size=(n, 3)).astype(F32)


# ------------------------------------------------------------------------------------------------ the filter
# the generator's slice (992 draws) and block (126 976), the compaction tile (2048), up to 2^24 points
SIZES = [1, 2, 31, 32, 33, 991, 992, 993, 2047, 2048, 2049, 4096, BLOCK - 1, BLOCK, BLOCK + 1, 1_000_003]


@pytest.mark.parametrize("n", SIZES)
def test_filter_against_glibc(n):
    assert check_sample(cloud(n, n)) > (0 if n < 100 else 0.85 * n)


def test_filter_at_2_24_points():
    n = 1 << 24
    pts = np.random.default_rng(24).standard_normal((n, 3), dtype=F32)
    check_sample(pts, seed=3, position=12345)


@pytest.mark.parametrize("position", [1, SLICE - 1, SLICE, SLICE + 1, 3 * SLICE + 17, BLOCK - 1, BLOCK, 2**20])
def test_positions_straddling_slice_starts(position):
    check_sample(cloud(3 * SLICE + 5, 1), seed=12345, position=position)
    check_sample(cloud(BLOCK + 7, 2), seed=2**32 - 1, position=position)


@pytest.mark.parametrize("position", [2**40, 2**40 + SLICE - 1, 2**62 + 3])
def test_far_positions(position):
    pts = cloud(300_001, 5)
    check_sample(pts, seed=7, position=position, want=host_mask(pts.shape[0], 0.9, 7, position))


def test_prob_0_1_and_exact_thresholds():
    pts = cloud(50_000, 9)
    assert check_sample(pts, prob=0.0, position=77) == 0
    k1 = check_sample(pts, prob=1.0, position=77)
    assert 49_900 < k1 <= 50_000          # (float)rand() / (float)RAND_MAX is 1.0 for draws within 64 of 2^31
    d = R.glibc_rand(1, 77, 50_000)
    for k in (3, 4999, 31_337):           # a prob that some draw's float equals: that draw is not kept
        prob = float(F32(d[k]) / F32(2**31))
        want = R.pm_rand_mask(50_000, prob, 1, 77)
        assert not want[k] and np.array_equal(want, (d.astype(F32) / F32(2**31)) < F32(prob))
        check_sample(pts, prob=prob, position=77, want=want)
    # prob 1 drops draw 13 068 230 of seed 1, the first whose float is 2^31
    assert F32(R.glibc_rand(1, 13_068_230, 1)[0]) == F32(2**31)
    keep, _ = device_sample(pts, 1.0, 1, 13_068_230 - 1000)
    assert keep[:1000].all() and not keep[1000]
    check_sample(pts, prob=1.0, position=13_068_230 - 1000)


def test_non_finite_points_take_draws():
    pts = cloud(20_000, 4)
    pts[::7, 0] = np.nan
    pts[5::11, 2] = np.inf
    pts[100:3000] = np.nan
    m = check_sample(pts, position=31)
    assert m > 0.85 * 20_000


# ------------------------------------------------------------------------------------------------ Align
def _matcher(src, tgt, sampler=RAND, normals=None, p2p=False, seed=None, position=None):
    m = smb.IcpUsingPointMatcher(0)
    if normals is not None:
        m.SetSurfaceNormals(normals)
    if p2p:
        m.SetErrorMinimizer(smb.ErrorMinimizer.POINT_TO_POINT)
    if seed is not None:
        assert m._lib.sm_set_option(m._h, b"sample_seed", str(seed).encode()) == 0
    m.SetReadingSampler(sampler)
    if position is not None:
        m.SetRandPosition(position)
    m.SetInputSource(smb.InnerCloud(src))
    m.SetInputTarget(smb.InnerCloud(tgt))
    return m


def _pairs():
    src, tgt, _ = scenes.corner_pair()
    yield src.astype(F32), tgt.astype(F32)
    for pair in (0, 1):
        src, sub, _ = scenes.lidar_pair(pair=pair)
        yield src.astype(F32), sub.astype(F32)


def rand_chain(src, tgt, normals=LS, p2p=False, seed=1, position=0):
    """the stand-in's chain composed from the oracle's pieces, reading filter = glibc's rand() at (seed, position)"""
    if normals == LS and not p2p:
        return R.icp_pm_equivalent(src, tgt, seed=seed, position=position)
    keep = R.pm_rand_mask(src.shape[0], 0.9, seed, position)
    tp, tn = PN.pm_reference_filter(tgt, "least_squares" if normals == LS else "eigenvector")
    s = src[keep].astype(np.float64)
    o = OP.icp_fast_align(s, tp, None, max_iteration=150) if p2p else O.icp_fast_align(s, tp, tn, None, max_iteration=150)
    o["n_source"], o["n_target"] = int(keep.sum()), int(tp.shape[0])
    _, d2 = O.knn1(tgt.astype(np.float64), O.pm_moved(src, o["result"]), epsilon=3.16)
    v, _, kept = O.pm_score_trim(d2)
    o["score"] = float(np.exp(-(np.sqrt(v[:kept]).sum() / kept)))
    o["ok"] = o["score"] >= float(F32(0.6))
    return o


def _check(m, ok, res, o):
    info = m.GetAlignInfo()
    assert ok == o["ok"]
    assert int(info["aux"][2]) == o["n_source"] and int(info["aux"][3]) == o["n_target"]
    assert info["iterations"] == o["iterations"]
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= 1e-9 and dr <= 1e-9, (dt, dr)
    assert abs(m.GetFitnessScore() - o["score"]) < 1e-12


@pytest.mark.parametrize("normals", [LS, EV])
@pytest.mark.parametrize("p2p", [False, True])
def test_align_against_the_oracle_chain(normals, p2p):
    for k, (src, tgt) in enumerate(_pairs()):
        seed, position = (1, 0) if k == 0 else (12345 + k, 1000 * k + 3)
        m = _matcher(src, tgt, normals=normals, p2p=p2p, seed=seed, position=position)
        ok, res = m.Align(np.eye(4))
        _check(m, ok, res, rand_chain(src, tgt, normals, p2p, seed, position))
        assert m.GetRandPosition() == position + src.shape[0]


def test_eigenvector_mode_is_the_literal_chain():
    """seed 1, position 0: the first type-1 Align of a process that never called srand.  With libpointmatcher's
    reference filter and its reading filter both restated, only double against float LAPACK arithmetic is left"""
    src, tgt = next(_pairs())
    kn = lambda t, q: O.knn1(t, q, epsilon=3.16)      # noqa: E731
    rng = pyref.GlibcRand(1)
    m = _matcher(src, tgt, normals=EV)
    for _ in range(2):                                # two consecutive Aligns share one stream, as two calls do
        lit = pyref.icp_pm_literal(src, tgt, rng=rng, knn_full=kn)
        ok, res = m.Align(np.eye(4))
        assert int(m.GetAlignInfo()["aux"][2]) == lit["n_source"]
        dt, dr = scenes.se3_error(lit["result"], res)
        assert dt <= 1e-8 and dr <= 1e-8, (dt, dr)
    assert m.GetRandPosition() == 2 * src.shape[0]


# ------------------------------------------------------------------------------------------------ the position
def test_consecutive_aligns_draw_on():
    src, tgt = list(_pairs())[1]
    m = _matcher(src, tgt)
    n = src.shape[0]
    for k in range(3):
        assert m.GetRandPosition() == k * n
        ok, res = m.Align(np.eye(4))
        _check(m, ok, res, rand_chain(src, tgt, position=k * n))


def test_setting_a_position_back_reproduces_an_align():
    src, tgt = list(_pairs())[1]
    m = _matcher(src, tgt, position=5)
    first = m.Align(np.eye(4)), m.GetFitnessScore(), m.GetAlignInfo()["aux"][2]
    second = m.Align(np.eye(4))
    assert second[1].tobytes() != first[0][1].tobytes()
    m.SetRandPosition(5)
    again = m.Align(np.eye(4)), m.GetFitnessScore(), m.GetAlignInfo()["aux"][2]
    assert again[0][0] == first[0][0] and again[0][1].tobytes() == first[0][1].tobytes()
    assert again[1] == first[1] and again[2] == first[2]


def test_sample_seed_resets_the_position():
    src, tgt = next(_pairs())
    m = _matcher(src, tgt)
    m.Align(np.eye(4))
    assert m.GetRandPosition() == src.shape[0]
    assert m._lib.sm_set_option(m._h, b"sample_seed", b"9") == 0
    assert m.GetRandPosition() == 0
    ok, res = m.Align(np.eye(4))
    _check(m, ok, res, rand_chain(src, tgt, seed=9, position=0))


def test_hash_mode_leaves_the_position_and_is_unchanged():
    src, tgt = list(_pairs())[1]
    a = _matcher(src, tgt, sampler=HASH, position=17)
    b = smb.IcpUsingPointMatcher(0)
    b.SetInputSource(smb.InnerCloud(src))
    b.SetInputTarget(smb.InnerCloud(tgt))
    for _ in range(2):
        ra, rb = a.Align(np.eye(4)), b.Align(np.eye(4))
        assert ra[0] == rb[0] and ra[1].tobytes() == rb[1].tobytes() and a.GetFitnessScore() == b.GetFitnessScore()
    assert a.GetRandPosition() == 17 and b.GetRandPosition() == 0
    dt, dr = scenes.se3_error(O.icp_pm_equivalent(src, tgt)["result"], ra[1])
    assert dt <= 1e-9 and dr <= 1e-9


def test_switching_samplers_gives_what_fresh_handles_give():
    src, tgt = list(_pairs())[1]
    h = _matcher(src, tgt, sampler=HASH)
    want_hash = h.Align(np.eye(4))
    m = _matcher(src, tgt)
    r1 = m.Align(np.eye(4))
    m.SetReadingSampler(HASH)
    r2 = m.Align(np.eye(4))
    assert r2[1].tobytes() == want_hash[1].tobytes() and m.GetRandPosition() == src.shape[0]
    m.SetReadingSampler(RAND)
    m.SetRandPosition(0)
    r3 = m.Align(np.eye(4))
    assert r3[1].tobytes() == r1[1].tobytes()


def test_align_batch_with_mixed_samplers():
    src, tgt = list(_pairs())[1]
    plan = [(RAND, 0), (HASH, None), (RAND, 4000), (EV, 123), (HASH, None), (RAND, 2**40)]

    def make(sampler, pos):
        if sampler == EV:
            return _matcher(src, tgt, normals=EV, position=pos)
        return _matcher(src, tgt, sampler=sampler, position=pos)
    singles = []
    for s, p in plan:
        m = make(s, p)
        singles.append((m.Align(np.eye(4)), m.GetFitnessScore(), m.GetRandPosition()))
    ms = [make(s, p) for s, p in plan]
    oks, rb = smb.AlignBatch(ms, [np.eye(4)] * len(plan))
    for k in range(len(plan)):
        (ok, r), score, pos = singles[k]
        assert oks[k] == ok and rb[k].tobytes() == r.tobytes() and ms[k].GetFitnessScore() == score
        assert ms[k].GetRandPosition() == pos
    assert not np.array_equal(rb[0], rb[2])


def test_other_types_and_bad_values_are_rejected():
    lib = _lib.lib()
    src, tgt, _ = scenes.corner_pair()
    tp, tn = O.calculate_normals(tgt)
    f = smb.IcpFast(0)
    f.SetInputSource(smb.EigenCloud(src))
    f.SetInputTarget(smb.EigenCloud(tp, tn))
    _, r0 = f.Align(np.eye(4))
    pos = C.c_int64(-3)
    assert lib.sm_set_pm_reading_sampler(f._h, 1) == -11
    assert lib.sm_get_pm_rand_position(f._h, C.byref(pos)) == -11 and pos.value == -3
    assert lib.sm_set_pm_rand_position(f._h, 5) == -11
    _, r1 = f.Align(np.eye(4))
    assert r1.tobytes() == r0.tobytes()
    for t in (3, 5):
        h = C.c_void_p()
        assert lib.sm_create(t, 0, C.byref(h)) == 0
        assert lib.sm_set_pm_reading_sampler(h, 1) == -11
        assert lib.sm_get_pm_rand_position(h, C.byref(pos)) == -11
        assert lib.sm_set_pm_rand_position(h, 5) == -11
        lib.sm_destroy(h)
    s32, t32 = src.astype(F32), tgt.astype(F32)
    n = _matcher(s32, t32, sampler=RAND, normals=None)
    fresh = _matcher(s32, t32, sampler=RAND)
    for bad in (-1, 2, 7):
        assert lib.sm_set_pm_reading_sampler(n._h, bad) == -1
    assert lib.sm_set_pm_rand_position(n._h, -1) == -1
    assert lib.sm_get_pm_rand_position(n._h, None) == -1
    assert n.GetRandPosition() == 0
    a, b = n.Align(np.eye(4)), fresh.Align(np.eye(4))
    assert a[0] == b[0] and a[1].tobytes() == b[1].tobytes()
    with pytest.raises(smb.CheckFailure):
        n.SetReadingSampler(5)
    with pytest.raises(smb.CheckFailure):
        n.SetRandPosition(-2)
    n.SetRandPosition(2**63 - 10)
    g, res = np.eye(4), np.zeros(16)
    assert lib.sm_align(n._h, g.ctypes.data_as(_lib._DP), res.ctypes.data_as(_lib._DP)) == -1
    assert n.GetRandPosition() == 2**63 - 10


# ------------------------------------------------------------------------------------------------ the adapter
def test_cpp_adapter(tmp_path):
    exe = adapter_exe(tmp_path, "pm_rand_sampling_adapter_run")
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
    n = src.shape[0]
    assert int(out["bad_mode_rc"][0]) == -1 and int(out["bad_position_rc"][0]) == -1
    assert out["positions"].astype(np.int64).tolist() == [0, n, 2 * n, 7, 7 + n]
    for key, position in (("first", 0), ("second", n), ("at_7", 7)):
        o = rand_chain(src, tgt, position=position)
        ok, score, T = out[key][0], out[key][1], out[key][2:].reshape(4, 4).T
        dt, dr = scenes.se3_error(o["result"], T)
        assert dt <= 1e-9 and dr <= 1e-9, (key, dt, dr)
        assert bool(ok) == o["ok"] and abs(score - o["score"]) < 1e-12
