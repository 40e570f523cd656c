"""sm_align_pairs and sm_align_batch driven the way bench.py drives them: 16 IcpFast instances on caller-owned
torch streams, several host threads at once, device / pinned / pageable inputs, every instance given pairs of
different sizes within one call.  The pipelined layer must not change a pose: every pipelined result is compared
bit for bit with a single sm_align of the same pair on a fresh instance, and every such reference with the CPU
oracle.  A failed pair must report its own rc, a score of 0.0 and an untouched result slot, and no instance's
stream may still be busy with a pair when the call returns.

The distinct pairs straddle the k-NN launch paths: targets up to 16 384 points (11 k-d levels, kKnnSmemLevels) are
searched with the whole inner tree in shared memory, deeper ones through the other kernel instantiation."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

import oracle_lib as O
import scenes
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

pytestmark = pytest.mark.gpu

TOL_T = 1e-4   # metres   (test_gpu_icp.py, test_gpu_full_size.py)
TOL_R = 1e-4   # radians

# instance options: bench.py's, the one-alignment-in-flight search geometry, and the convergence test on
OPTS = {
    "bench": {"max_iteration": 30, "disable_convergence_check": 1, "knn_queries_per_cta": 1024},
    "qpc0": {"max_iteration": 30, "disable_convergence_check": 1, "knn_queries_per_cta": 0},
    "conv": {"max_iteration": 100, "disable_convergence_check": 0, "knn_queries_per_cta": 1024},
}
ORACLE_OPTS = {"bench": dict(max_iteration=30, disable_convergence_check=True),
               "qpc0": dict(max_iteration=30, disable_convergence_check=True),
               "conv": dict(max_iteration=100, disable_convergence_check=False)}

# (source, raw target) builders and the k-d depth of the target after CalculateNormals
PAIRS = (
    (lambda: scenes.corner_pair()[:2], 7),                                                         # 1 024 target points
    (lambda: scenes.lidar_pair()[:2], 11),                                                         # 8 567: deepest all-smem tree
    (lambda: scenes.lidar_pair(n_az=600, submap_points=180_000, pair=1)[:2], 12),                  # 23 308
    (lambda: scenes.lidar_pair(n_az=800, n_beams=48, submap_points=380_000, pair=2)[:2], 13),      # 48 117
    (lambda: scenes.lidar_pair(n_az=1600, n_beams=64, submap_points=560_000, pair=3)[:2], 14),     # 93 924
    (lambda: scenes.full_size_pair(0)[:2], 14),                                                    # 120 000 -> 106 784
)
SMALL, LARGE = (0, 1, 2), (3, 4, 5)
KINDS = ("device", "pinned", "pageable")
SENTINEL = -7.25
KNN_SMEM_LEVELS = 11


def kd_levels(n, bucket=8):
    """kd_num_levels (kdtree.cu)"""
    L = 0
    while n > bucket:
        n = (n + 1) // 2
        L += 1
    return L


def guess_of(d):
    """a non-identity initial guess per distinct pair"""
    a = 0.01 * (d + 1)
    G = np.eye(4)
    G[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    G[:3, 3] = np.array([0.2, -0.12, 0.03]) * (1 + 0.5 * d)
    return G


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


class Cloud:
    """One distinct pair in the three forms sm_align_pairs takes: device tensors, pinned and pageable host memory."""

    def __init__(self, src, tp, tn):
        self.src, self.tp, self.tn = (np.ascontiguousarray(a) for a in (src, tp, tn))
        self.ns, self.nt = self.src.shape[0], self.tp.shape[0]
        self.dev = [torch.from_numpy(a).cuda() for a in (self.src, self.tp, self.tn)]
        self.pin = [torch.from_numpy(a).pin_memory() for a in (self.src, self.tp, self.tn)]

    def ptrs(self, kind):
        if kind == "device":
            return [int(t.data_ptr()) for t in self.dev]
        if kind == "pinned":
            return [int(t.data_ptr()) for t in self.pin]
        return [a.ctypes.data for a in (self.src, self.tp, self.tn)]


@pytest.fixture(scope="module")
def clouds():
    out = []
    for build, levels in PAIRS:
        src, raw = build()
        tp, tn = O.calculate_normals(raw)
        assert kd_levels(tp.shape[0]) == levels, (tp.shape[0], levels)
        out.append(Cloud(src, tp, tn))
    assert out[5].nt == 106_784 and out[5].ns == 120_000       # the benchmark's own pair
    assert kd_levels(out[1].nt) == KNN_SMEM_LEVELS < kd_levels(out[2].nt)
    return out


@pytest.fixture(scope="module")
def refs(clouds):
    """refs(d, opts, guessed): a single sm_align of pair d on a fresh instance, checked once against the oracle"""
    cache = {}

    def get(d, opts, guessed=False):
        key = (d, opts, guessed)
        if key not in cache:
            c = clouds[d]
            g = guess_of(d) if guessed else np.eye(4)
            m = smb.IcpFast()
            m.InitWithXml(OPTS[opts])
            m.SetInputSource(smb.EigenCloud(c.src)); m.SetInputTarget(smb.EigenCloud(c.tp, c.tn))
            res = np.zeros(16)
            gcm = np.ascontiguousarray(g.T).ravel()
            rc = m._lib.sm_align(m._h, gcm.ctypes.data_as(_lib._DP), res.ctypes.data_as(_lib._DP))
            r = {"rc": rc, "pose": res.reshape(4, 4).T.copy(), "score": m.GetFitnessScore(), "info": m.GetAlignInfo()}
            o = O.icp_fast_align(c.src, c.tp, c.tn, g, **ORACLE_OPTS[opts])
            assert rc == 1 and o["rc"] == 1
            assert r["info"]["iterations"] == o["iterations"], key
            dt, dr = scenes.se3_error(o["result"], r["pose"])
            assert dt <= TOL_T and dr <= TOL_R, (key, dt, dr)
            cache[key] = r
        return cache[key]
    return get


def instances(n, opts, streams=True, **extra):
    ms, ss = [], []
    for _ in range(n):
        m = smb.IcpFast()
        m.InitWithXml({**OPTS[opts], **extra})
        if streams:
            s = torch.cuda.Stream()
            m.SetStream(s.cuda_stream)
            ss.append(s)
        ms.append(m)
    return ms, ss


def pair_array(clouds, plan):
    """plan: [(d, kind, guessed)] or with a 4th entry overriding fields: {"n_source": .., "source": ..}"""
    arr = (_lib.Pair * len(plan))()
    keep = []
    for k, step in enumerate(plan):
        d, kind, guessed = step[:3]
        over = step[3] if len(step) > 3 else {}
        c = clouds[d]
        src, tgt, nrm = c.ptrs(kind)
        arr[k].source = over.get("source", src)
        arr[k].target, arr[k].target_normals = tgt, nrm
        arr[k].n_source = over.get("n_source", c.ns)
        arr[k].n_target = c.nt
        arr[k].on_device = 1 if kind == "device" else 0
        if guessed:
            g = np.ascontiguousarray(guess_of(d).T).ravel()
            keep.append(g)
            arr[k].guess = g.ctypes.data
    arr._keep = keep
    return arr


def align_pairs(ms, arr, streams=()):
    """sm_align_pairs through the C ABI (AlignPairs raises on the first bad rc): (ret, rcs, poses, scores, idle),
    result slots and scores filled with a sentinel first; idle = every stream's query() right after the return"""
    n = len(arr)
    hs = (C.c_void_p * len(ms))(*[m._h for m in ms])
    res = np.full((n, 16), SENTINEL)
    scores = np.full(n, SENTINEL)
    rcs = np.full(n, 7, dtype=np.int32)
    ret = _lib.lib().sm_align_pairs(hs, len(ms), arr, n, res.ctypes.data, scores.ctypes.data, rcs.ctypes.data)
    idle = [s.query() for s in streams]
    return ret, rcs, res.reshape(n, 4, 4).transpose(0, 2, 1), scores, idle


def run_threads(ms, streams, clouds, plan, T, batches=1):
    """thread j drives instances j::T with pairs j::T of the plan, `batches` calls in a row, as bench.py's
    run_steps does.  Returns per batch (rets per thread, rcs, poses, scores in plan order, idle flags)."""
    arrs = [pair_array(clouds, plan[j::T]) for j in range(T)]
    out = [[None] * T for _ in range(batches)]
    errors = []
    gate = threading.Barrier(T)

    def body(j):
        try:
            for b in range(batches):
                gate.wait()
                out[b][j] = align_pairs(ms[j::T], arrs[j], streams[j::T])
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=body, args=(j,)) for j in range(T)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    n = len(plan)
    inv = np.argsort(np.concatenate([np.arange(n)[j::T] for j in range(T)]))
    runs = []
    for b in range(batches):
        rets = [out[b][j][0] for j in range(T)]
        rcs, poses, scores = (np.concatenate([out[b][j][i] for j in range(T)])[inv] for i in (1, 2, 3))
        idle = [f for j in range(T) for f in out[b][j][4]]
        runs.append((rets, rcs, poses, scores, idle))
    return runs


def owner(k, n_instances, T):
    """the instance (index into the full list) pair k of a run_threads plan runs on"""
    j, i = k % T, k // T
    H = len(range(j, n_instances, T))
    return j + T * (i % H)


def assert_matches(refs, plan, opts, rcs, poses, scores):
    for k, step in enumerate(plan):
        d, kind, guessed = step[:3]
        r = refs(d, opts, guessed)
        assert rcs[k] == r["rc"], (k, rcs[k])
        assert np.array_equal(bits(poses[k]), bits(r["pose"])), (k, d, kind, guessed)
        assert bits(scores[k]) == bits(r["score"]), (k, scores[k], r["score"])


def bench_plan(n_pairs=64, n_instances=16):
    """pair k runs on instance k % 16 as its (k // 16)-th pair: every instance goes small -> large -> small ->
    large within one call; the input kind rotates device -> pinned -> pageable"""
    plan = []
    for k in range(n_pairs):
        h, r = k % n_instances, k // n_instances
        d = (SMALL, LARGE)[r % 2][(h + r // 2) % 3]
        plan.append((d, KINDS[k % 3], False))
    return plan


@pytest.mark.parametrize("T", [1, 2, 4])
def test_benchmark_regime(clouds, refs, T):
    ms, ss = instances(16, "bench")
    plan = bench_plan()
    for k in range(len(plan)):
        assert owner(k, 16, T) == k % 16
    for rets, rcs, poses, scores, idle in run_threads(ms, ss, clouds, plan, T, batches=3):
        assert rets == [0] * T
        assert all(idle)
        assert_matches(refs, plan, "bench", rcs, poses, scores)


def test_guesses_and_null_guess_in_one_call(clouds, refs):
    # pairs 0-5 with a guess of their own, 6-11 with guess_4x4 = NULL; instance h gets e.g. 0, 4 (guessed), 8 (NULL)
    ms, ss = instances(4, "qpc0")
    plan = [(k % 6, KINDS[k % 3], k < 6) for k in range(12)]
    (rets, rcs, poses, scores, idle), = run_threads(ms, ss, clouds, plan, 1)
    assert rets == [0] and all(idle)
    assert_matches(refs, plan, "qpc0", rcs, poses, scores)


def test_convergence_check_chunks_across_pipelines(clouds, refs):
    # guessed and identity starts stop after 6 .. 39 iterations: sm_align_wait re-enqueues 8-iteration chunks
    # on some instances while the others are in flight
    ms, ss = instances(6, "conv")
    plan = [(k % 6, KINDS[k % 3], (k // 6) % 2 == 0) for k in range(18)]
    iters = {refs(d, "conv", g)["info"]["iterations"] for d, _, g in plan}
    assert len(iters) >= 3 and max(iters) > 16
    T = 2
    (rets, rcs, poses, scores, idle), = run_threads(ms, ss, clouds, plan, T)
    assert rets == [0] * T and all(idle)
    assert_matches(refs, plan, "conv", rcs, poses, scores)
    last = {owner(k, len(ms), T): k for k in range(len(plan))}
    assert sorted(last) == list(range(len(ms)))
    for h, k in last.items():
        d, _, g = plan[k]
        got, want = ms[h].GetAlignInfo(), refs(d, "conv", g)["info"]
        for f in ("iterations", "kept", "limit", "solve_path"):
            assert got[f] == want[f], (h, k, f, got[f], want[f])


def sm_align_rc(opts, src_ptr, n_source, c, **extra):
    """what sm_set_input_target, sm_set_input_source and sm_align return, in that order, on a fresh instance"""
    m = smb.IcpFast()
    m.InitWithXml({**OPTS[opts], **extra})
    lib = m._lib
    rc = lib.sm_set_input_target(m._h, c.tp.ctypes.data, c.tn.ctypes.data, c.nt)
    if rc >= 0:
        rc = lib.sm_set_input_source(m._h, src_ptr, n_source)
    if rc >= 0:
        eye, res = np.eye(4).ravel(), np.zeros(16)
        rc = lib.sm_align(m._h, eye.ctypes.data_as(_lib._DP), res.ctypes.data_as(_lib._DP))
    return rc


def test_failed_pairs_keep_to_themselves(clouds, refs):
    # instances A, B on bench options, C with dist_outlier_ratio 1.5 (refused by the ratio check)
    (a, b), ss_ab = instances(2, "bench")
    (c,), ss_c = instances(1, "bench", dist_outlier_ratio=1.5)
    ms, ss = [a, b, c], ss_ab + ss_c
    nan_src = torch.full((clouds[1].ns, 3), float("nan"), dtype=torch.float64).pin_memory()
    nan = {"source": int(nan_src.data_ptr())}
    plan = [
        (0, "pinned", False),                      # A
        (5, "pinned", False, {"n_source": 0}),     # B: refused by the source count, after the target upload
        (5, "pinned", False),                      # C: refused by the ratio, after both uploads
        (1, "pinned", False, nan),                 # A: all-NaN source, fails in sm_align_wait (-2)
        (1, "pinned", False),                      # B: the pair after a refused one
        (2, "pageable", False),                    # C
        (5, "device", False),                      # A: the pair after a failed one
        (3, "pinned", False),                      # B
        (4, "pinned", False),                      # C: the call's last pair, refused while its copies may run
    ]
    expect = {
        1: sm_align_rc("bench", clouds[5].src.ctypes.data, 0, clouds[5]),
        2: sm_align_rc("bench", clouds[5].src.ctypes.data, clouds[5].ns, clouds[5], dist_outlier_ratio=1.5),
        3: sm_align_rc("bench", int(nan_src.data_ptr()), clouds[1].ns, clouds[1]),
        5: sm_align_rc("bench", clouds[2].src.ctypes.data, clouds[2].ns, clouds[2], dist_outlier_ratio=1.5),
        8: sm_align_rc("bench", clouds[4].src.ctypes.data, clouds[4].ns, clouds[4], dist_outlier_ratio=1.5),
    }
    assert expect == {1: -4, 2: -1, 3: -2, 5: -1, 8: -1}
    arr = pair_array(clouds, plan)
    ret, rcs, poses, scores, idle = align_pairs(ms, arr, ss)
    assert idle == [True, True, True]
    assert ret == min(expect.values())
    for k, step in enumerate(plan):
        if k in expect:
            assert rcs[k] == expect[k], (k, rcs[k])
            assert scores[k] == 0.0, (k, scores[k])
            assert np.all(poses[k] == SENTINEL), k
        else:
            r = refs(step[0], "bench")
            assert rcs[k] == 1
            assert np.array_equal(bits(poses[k]), bits(r["pose"])), k
            assert bits(scores[k]) == bits(r["score"]), k
    # the same instances, the all-NaN pair now the last one its instance (B) is given
    arr2 = pair_array(clouds, [(3, "pinned", False), (0, "device", False), (1, "pinned", False, nan)])
    ret, rcs, poses, scores, idle = align_pairs([b, a], arr2, ss_ab[::-1])
    assert idle == [True, True] and ret == -2 and list(rcs) == [1, 1, -2]
    assert scores[2] == 0.0 and np.all(poses[2] == SENTINEL)
    for k, d in ((0, 3), (1, 0)):
        assert np.array_equal(bits(poses[k]), bits(refs(d, "bench")["pose"])), k
    # a refused pinned pair alone in a call: no other pipeline keeps the call busy while its copies would run
    for inst, s, step, rc in ((c, ss_c, (5, "pinned", False), -1), (b, ss_ab[:1], (5, "pinned", False, {"n_source": 0}), -4)):
        ret, rcs, poses, scores, idle = align_pairs([inst], pair_array(clouds, [step]), s)
        assert idle == [True]
        assert ret == rcs[0] == rc and scores[0] == 0.0 and np.all(poses[0] == SENTINEL)


def test_stream_switching_relaunches_graphs(clouds, refs):
    m = smb.IcpFast()
    m.InitWithXml(OPTS["qpc0"])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def align(d):
        c = clouds[d]
        m.SetInputSource(smb.EigenCloud(c.src)); m.SetInputTarget(smb.EigenCloud(c.tp, c.tn))
        ok, res = m.Align(np.eye(4))
        r = refs(d, "qpc0")
        assert ok and np.array_equal(bits(res), bits(r["pose"])), d
        assert m.GetFitnessScore() == r["score"]

    align(5)                  # graphs captured on the instance's own stream
    m.SetStream(s1.cuda_stream)
    align(5)                  # ... launched on s1
    align(1)                  # captured on s1
    m.SetStream(0)
    align(1)                  # ... launched on the own stream
    m.SetStream(s2.cuda_stream)
    arr = pair_array(clouds, [(5, "pinned", False), (1, "device", False), (4, "pageable", False)])
    ret, rcs, poses, scores, idle = align_pairs([m], arr, [s2])
    assert ret == 0 and idle == [True]
    assert_matches(refs, [(5, "", False), (1, "", False), (4, "", False)], "qpc0", rcs, poses, scores)
    m.SetStream(0)
    align(4)


def test_align_batch_across_types_and_threads(clouds, refs):
    f32 = [tuple(a.astype(np.float32) for a in scenes.lidar_pair(pair=p)[:2]) for p in range(3)]
    icp, icp_ss = instances(4, "bench")
    for m, d in zip(icp, (0, 1, 2, 5)):
        c = clouds[d]
        m.SetInputSource(smb.EigenCloud(c.src)); m.SetInputTarget(smb.EigenCloud(c.tp, c.tn))
    ndt = [smb.Ndt() for _ in range(2)]
    gicp = [smb.NdtWithGicp() for _ in range(3)]
    pm = [smb.IcpUsingPointMatcher() for _ in range(2)]
    for m, normals in zip(pm, (smb.SurfaceNormals.LEAST_SQUARES, smb.SurfaceNormals.EIGENVECTOR)):
        m.SetReadingSampler(smb.ReadingSampler.HASH)
        m.SetSurfaceNormals(normals)
    for ms_, ps in ((ndt, (0, 1)), (gicp, (0, 1, 2)), (pm, (0, 1))):
        for m, p in zip(ms_, ps):
            m.SetInputSource(smb.InnerCloud(f32[p][0])); m.SetInputTarget(smb.InnerCloud(f32[p][1]))
    batch = [icp[0], gicp[0], ndt[0], pm[0], icp[1], gicp[1], icp[2], pm[1], ndt[1], gicp[2], icp[3]]
    n = len(batch)
    # the second host thread: 16 pairs over 8 other IcpFast instances
    others, other_ss = instances(8, "bench")
    plan = [(d, KINDS[k % 3], False) for k, d in enumerate([0, 3, 1, 4, 2, 5, 1, 3] * 2)]
    arr = pair_array(clouds, plan)
    hs = (C.c_void_p * n)(*[m._h for m in batch])
    guesses = np.tile(np.eye(4).ravel(), n)
    res = np.full((n, 16), SENTINEL)
    rcs = np.full(n, 7, dtype=np.int32)
    gate = threading.Barrier(2)
    pairs_out = []

    def pairs_thread():
        gate.wait()
        pairs_out.append(align_pairs(others, arr, other_ss))

    t = threading.Thread(target=pairs_thread)
    t.start()
    gate.wait()
    ret = _lib.lib().sm_align_batch(hs, n, guesses.ctypes.data, res.ctypes.data, rcs.ctypes.data)
    t.join()
    assert pairs_out, "the sm_align_pairs thread raised"
    batch_scores = [m.GetFitnessScore() for m in batch]
    assert ret == 0 and all(rc >= 0 for rc in rcs), list(rcs)
    assert all(s.query() for s in icp_ss)
    for i, m in enumerate(batch):
        one = np.zeros(16)
        rc = m._lib.sm_align(m._h, np.eye(4).ravel().ctypes.data_as(_lib._DP), one.ctypes.data_as(_lib._DP))
        assert rc == rcs[i], (i, rc, rcs[i])
        assert np.array_equal(bits(res[i]), bits(one)), (i, m.GetType())
        assert bits(batch_scores[i]) == bits(m.GetFitnessScore()), i
    pret, prcs, pposes, pscores, pidle = pairs_out[0]
    assert pret == 0 and all(pidle)
    assert_matches(refs, plan, "bench", prcs, pposes, pscores)
    # one NdtWithGicp and one Ndt of the batch against the oracle (test_gpu_full_size.py's bars)
    s32, t32 = f32[0]
    o = O.ndt_gicp_align(s32, t32)
    info = gicp[0].GetAlignInfo()
    dt, dr = scenes.se3_error(o["result"], res[1].reshape(4, 4).T)
    assert o["rc"] == 1 and dt <= TOL_T and dr <= TOL_R, (dt, dr)
    assert info["iterations"] == o["gicp_iterations"] and info["profiled_iterations"] == o["bfgs_evaluations"]
    assert abs(batch_scores[1] - o["score"]) < 1e-9
    o = O.ndt_align(s32, t32)
    info = ndt[0].GetAlignInfo()
    dt, dr = scenes.se3_error(o["result"], res[2].reshape(4, 4).T)
    assert o["rc"] == 1 and dt <= TOL_T and dr <= TOL_R, (dt, dr)
    assert info["iterations"] == o["iterations"]
    assert abs(batch_scores[2] - o["fitness"]) <= 1e-9 * max(1.0, o["fitness"])
