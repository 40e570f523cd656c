"""The IcpUsingPointMatcher stand-in (type 1) on the GPU one stage at a time, against the oracle and numpy.

tests/test_gpu_icp_pm.py checks the whole chain through the pose and the averaged score.  Here the device stages
type 1 owns run through sm_debug_pm_stages, which calls PmStage::sample, FloatTree::build and PmStage::score_pass as
pm_align does, and each output is compared on its own:
  * the reading filter: the kept set is oracle_lib.pm_keep_mask's and the output is the kept points as doubles, bit
    for bit, in input order, at the compaction's tile edges (tiles of 2048), at prob 0 / 1e-9 / 0.5 / 0.9 / the float
    below 1 / 1 / 1.5 and with four seeds;
  * the score pass: the n sorted squared distances of its approximate search (eps 3.16 over the float tree) are the
    oracle's, bit for bit; valid and kept follow the trim rule; the mean is bit-identical to a numpy restatement of
    pm_score_reduce_kernel's 1024-thread order and within 1e-13 of math.fsum.  Sizes straddle the sort's switch to
    the chunked scan (262 144 keys) and the reduction's 1024-thread stride; clouds with exact ties at the limit, all
    distances zero, far points and non-finite points;
  * the target filter (CalculateNormals) at the sizes where its keep array crosses tile edges;
  * type 1's own control paths through the public API: an empty reading or target filter followed by a good Align,
    a new target or new filter options after an Align, and a reading cloud past the sort's switch."""
import ctypes as C
import functools
import math

import numpy as np
import pytest

import oracle_lib as O
import scenes
import staticmapping_b200 as smb
from staticmapping_b200 import _lib, synth

pytestmark = pytest.mark.gpu

EPS = 3.16
RATIOS = (0.0, 0.7, 1.0, 1.5)          # above 1 the quantile index is clamped to the last valid distance
FLOAT_BELOW_1 = float(np.nextafter(np.float32(1.0), np.float32(0.0)))


# ------------------------------------------------------------------------------------------------ hook binding
def device_stages(reading, target, prob=0.9, seed=1, T=np.eye(4), ratio=0.7, eps=EPS):
    r = np.ascontiguousarray(reading, dtype=np.float32)
    t = np.ascontiguousarray(target, dtype=np.float32)
    n = r.shape[0]
    T_cm = np.ascontiguousarray(np.asarray(T, dtype=np.float64).T).ravel()
    kept = C.c_int64(-1)
    sampled = np.zeros((n, 3))
    keys = np.zeros(n)
    out = np.zeros(3)
    rc = _lib.lib().sm_debug_pm_stages(0, r.ctypes.data, n, t.ctypes.data, t.shape[0], prob, seed & 0xFFFFFFFF,
                                       T_cm.ctypes.data, eps, ratio, C.byref(kept), sampled.ctypes.data,
                                       keys.ctypes.data, out.ctypes.data)
    assert rc == 0
    return {"kept_points": sampled[:kept.value], "keys": keys, "mean": out[0], "kept": int(out[1]),
            "valid": int(out[2])}


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


# ------------------------------------------------------------------------------------------------ reading filter
FILTER_SIZES = [1, 2, 2047, 2048, 2049, 4095, 4096, 4097, 262_145, (1 << 20) + 3]
PROBS = [0.0, 1e-9, 0.5, 0.9, FLOAT_BELOW_1, 1.0, 1.5]
SEEDS = [0, 1, 0x7FFFFFFF, -1]        # sample_seed is an int32 the matcher casts to uint32
TINY_TARGET = np.random.default_rng(7).uniform(-5.0, 5.0, size=(16, 3)).astype(np.float32)


@functools.lru_cache(maxsize=None)
def _filter_cloud(n):
    """n float points, a few with a non-finite coordinate or a negative zero: the filter copies whatever it keeps"""
    rng = np.random.default_rng(n)
    p = rng.normal(0.0, 30.0, size=(n, 3)).astype(np.float32)
    bad = rng.choice(n, size=min(n, 5), replace=False)
    p[bad, rng.integers(0, 3, bad.size)] = np.array([np.nan, np.inf, -np.inf, np.nan, -0.0], np.float32)[:bad.size]
    return p


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("prob", PROBS)
@pytest.mark.parametrize("n", FILTER_SIZES)
def test_reading_filter_keeps_the_oracle_set_in_input_order(n, prob, seed):
    src = _filter_cloud(n)
    mask = O.pm_keep_mask(n, prob, seed & 0xFFFFFFFF)
    r = device_stages(src, TINY_TARGET, prob=prob, seed=seed)
    assert r["kept_points"].shape[0] == int(mask.sum()), (n, prob, seed)
    assert np.array_equal(bits(r["kept_points"]), bits(src[mask].astype(np.float64))), (n, prob, seed)
    if prob <= 0.0:
        assert not mask.any()
    if prob >= 1.0:
        assert mask.all()


# ------------------------------------------------------------------------------------------------ score pass
def check_score_pass(reading, target, T, ratios=RATIOS):
    """Every output of the score pass at each trim ratio against the oracle's approximate search and numpy."""
    reading = np.asarray(reading, dtype=np.float32)
    n = reading.shape[0]
    finite = np.isfinite(reading).all(axis=1)
    # the oracle is fed finite queries only; the others must find no match on the device (+inf keys)
    _, d2 = O.knn1(np.asarray(target, np.float32).astype(np.float64), O.pm_moved(reading[finite], T), epsilon=EPS)
    expect_keys = np.concatenate([np.sort(d2), np.full(n - int(finite.sum()), np.inf)])
    for ratio in ratios:
        r = device_stages(reading, target, T=T, ratio=ratio)
        assert np.array_equal(bits(r["keys"]), bits(expect_keys)), ratio
        v, valid, kept = O.pm_score_trim(d2, ratio)
        assert (r["valid"], r["kept"]) == (valid, kept), ratio
        assert valid == int(finite.sum())
        roots = np.sqrt(v[:kept])
        mean = O.pm_score_block_sum(roots) / kept if kept else 0.0
        assert bits([r["mean"]]) == bits([mean]), (ratio, r["mean"], mean)
        if kept:
            ref = math.fsum(roots) / kept
            assert abs(r["mean"] - ref) <= 1e-13 * abs(ref), (ratio, r["mean"], ref)
    return d2


@functools.lru_cache(maxsize=None)
def _lidar(pair=0):
    src, sub, P = scenes.lidar_pair(pair=pair)
    return src.astype(np.float32), sub.astype(np.float32), P


def test_score_pass_lidar_pair_at_its_registered_pose():
    src, sub, P = _lidar()
    d2 = check_score_pass(src, sub, P)
    assert np.median(np.sqrt(d2)) < 0.2                       # the pose registers the scan


def test_score_pass_identical_clouds_keep_every_point_at_distance_zero():
    _, sub, _ = _lidar()
    d2 = check_score_pass(sub, sub, np.eye(4))
    assert not d2.any()                                       # limit 0, every point kept at every ratio


def test_score_pass_lattice_ties_at_the_limit():
    g = np.arange(16, dtype=np.float32)
    target = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)
    r = np.arange(-3, 19, dtype=np.float32)
    reading = np.stack(np.meshgrid(r, r, r, indexing="ij"), axis=-1).reshape(-1, 3) + np.float32([0.25, 0.5, 0.0])
    d2 = check_score_pass(reading, target, np.eye(4))
    v = np.sort(d2)
    for ratio in (0.0, 0.7):                                  # the limit sits inside a run of equal distances
        qi = int(v.size * float(np.float32(ratio)))
        assert v[qi] == v[min(qi + 1, v.size - 1)] and np.count_nonzero(v == v[qi]) > 1


@pytest.mark.parametrize("n", [1, 31, 1023, 1024, 1025, 2049, 262_144, 262_145])
def test_score_pass_sizes(n):
    _, sub, _ = _lidar()
    rng = np.random.default_rng(n)
    world = sub[rng.integers(0, sub.shape[0], n)].astype(np.float64) + rng.normal(0.0, 0.05, size=(n, 3))
    P = synth.perturbation(3)
    reading = synth.apply_se3(np.linalg.inv(P), world).astype(np.float32)
    check_score_pass(reading, sub, P)


def test_score_pass_far_points():
    src, sub, P = _lidar()
    rng = np.random.default_rng(11)
    reading = src.copy()
    far = rng.choice(src.shape[0], size=src.shape[0] // 3, replace=False)
    direction = rng.normal(size=(far.size, 3))
    reading[far] += (1e4 * direction / np.linalg.norm(direction, axis=1, keepdims=True)).astype(np.float32)
    d2 = check_score_pass(reading, sub, P)
    assert np.sqrt(d2).max() > 9e3


def test_score_pass_non_finite_points_count_nowhere():
    src, sub, P = _lidar()
    rng = np.random.default_rng(12)
    reading = src.copy()
    rows = rng.choice(src.shape[0], size=300, replace=False)
    vals = np.array([np.nan, np.inf, -np.inf], np.float32)
    reading[rows, rng.integers(0, 3, rows.size)] = vals[np.arange(rows.size) % 3]
    reading[rows[:10]] = np.nan                                # whole points as well as single coordinates
    check_score_pass(reading, sub, P)
    check_score_pass(reading, sub, np.eye(4))                  # 0 * inf in the transform: NaN queries


# ------------------------------------------------------------------------------------------------ normals target
@pytest.mark.parametrize("n", [2047, 2048, 2049, 4097, 262_145])
def test_normals_target_at_compaction_edges(n):
    rng = np.random.default_rng(n)
    pts = rng.uniform(1.0, 100.0, size=(n, 3))
    op, on = O.calculate_normals(pts)
    g = smb.CalculateNormals(pts)
    assert op.shape[0] > 0
    assert np.array_equal(bits(g.points), bits(op)) and np.array_equal(bits(g.normals), bits(on))


# ------------------------------------------------------------------------------------------------ public API
RESULT_INFO = ("iterations", "status", "solve_path", "kept", "limit", "aux")   # the timings and launch counts vary


def _matcher(src, tgt, **opts):
    m = smb.IcpUsingPointMatcher()
    if opts:
        m.SetEngineOptions(**opts)
    m.SetInputSource(smb.InnerCloud(src))
    m.SetInputTarget(smb.InnerCloud(tgt))
    return m


def assert_same_align(m, ok, res, src, tgt, **opts):
    """(ok, res) and m's score and align info are bit-identical to a fresh matcher's on the same clouds"""
    f = _matcher(src, tgt, **opts)
    ok_f, res_f = f.Align(np.eye(4))
    assert ok == ok_f and np.array_equal(bits(res), bits(res_f))
    assert bits([m.GetFitnessScore()]) == bits([f.GetFitnessScore()])
    a, b = m.GetAlignInfo(), f.GetAlignInfo()
    assert {k: a[k] for k in RESULT_INFO} == {k: b[k] for k in RESULT_INFO}


def test_reading_filter_keeping_no_point_then_a_good_align():
    src, sub, _ = _lidar()
    m = _matcher(src, sub, reading_sample_prob=0.0)
    with pytest.raises(smb.CheckFailure, match="reading filter kept no point"):
        m.Align(np.eye(4))
    m.SetEngineOptions(reading_sample_prob=0.9)
    ok, res = m.Align(np.eye(4))
    assert_same_align(m, ok, res, src, sub)


def test_target_filter_keeping_no_point_then_a_good_target():
    src, sub, _ = _lidar()
    t = np.arange(1, 257, dtype=np.float32) * np.float32(0.25)
    line = np.stack([t, 2 * t, t + 1], axis=1)                # exactly collinear in float: every leaf is rank-deficient
    assert O.calculate_normals(line.astype(np.float64))[0].shape[0] == 0
    m = _matcher(src, line)
    with pytest.raises(smb.CheckFailure, match="no target point survived"):
        m.Align(np.eye(4))
    m.SetInputTarget(smb.InnerCloud(sub))
    ok, res = m.Align(np.eye(4))
    assert_same_align(m, ok, res, src, sub)


def test_new_target_after_align_smaller_then_larger():
    src, sub, _ = _lidar()
    first, smaller = sub[: 3 * sub.shape[0] // 4], sub[: sub.shape[0] // 2]
    m = _matcher(src, first)
    ok, res = m.Align(np.eye(4))
    assert_same_align(m, ok, res, src, first)
    for tgt in (smaller, sub):                                # rebuilt normals, score tree and IcpFast buffers
        m.SetInputTarget(smb.InnerCloud(tgt))
        ok, res = m.Align(np.eye(4))
        assert_same_align(m, ok, res, src, tgt)


@pytest.mark.parametrize("opts", [{"reading_sample_prob": 1.0}, {"sample_seed": 5}])
def test_new_reading_filter_options_after_align(opts):
    src, sub, _ = _lidar()
    m = _matcher(src, sub)
    m.Align(np.eye(4))
    m.SetEngineOptions(**opts)                                # the next Align filters the reading cloud anew
    ok, res = m.Align(np.eye(4))
    assert_same_align(m, ok, res, src, sub, **opts)
    o = O.icp_pm_equivalent(src, sub, prob=opts.get("reading_sample_prob", 0.9), seed=opts.get("sample_seed", 1))
    assert int(m.GetAlignInfo()["aux"][2]) == o["n_source"]


def test_large_reading_cloud_through_the_chunked_sort():
    src, sub, P = _lidar()
    rng = np.random.default_rng(5)
    n = 262_145
    tiles = -(-n // src.shape[0])
    big = (np.tile(src, (tiles, 1))[:n] + rng.normal(0.0, 0.01, size=(n, 3))).astype(np.float32)
    m = _matcher(big, sub)
    ok, res = m.Align(np.eye(4))
    o = O.icp_pm_equivalent(big, sub)
    info = m.GetAlignInfo()
    assert o["rc"] == 1 and ok == o["ok"]
    assert int(info["aux"][2]) == o["n_source"] and int(info["aux"][3]) == o["n_target"]
    assert info["iterations"] == o["iterations"]
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= 1e-4 and dr <= 1e-4, (dt, dr)
    assert abs(m.GetFitnessScore() - o["score"]) < 1e-9
    assert abs(info["aux"][0] - o["icp_fast_score"]) < 1e-9 and int(info["aux"][1]) == o["score_kept"]
    gt_t, gt_r = scenes.se3_error(P, res)
    assert gt_t < 0.05 and gt_r < 0.01
