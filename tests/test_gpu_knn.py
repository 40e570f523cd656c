"""sm_knn on an H100: libnabo's k-NN (k = 1..64, epsilon, maxRadius, self-match exclusion) bit for bit against the oracle
(tests/cpp/knn_oracle.cc), on ids and squared distances, order included.  Also: k = 1 against sm_knn1, the device
entry point against the host one, and two host threads on two streams against one."""
import ctypes as C
import threading

import numpy as np
import pytest

import kd_tree_model as M
import oracle_knn as OK
import staticmapping_b200 as smb
from staticmapping_b200 import _lib
from test_search_formulation_model import _adversarial_clouds

pytestmark = pytest.mark.gpu

INF = float("inf")
KS = [1, 2, 3, 7, 8, 9, 16, 20, 32, 33, 64]
EPSILONS = [0.0, 0.5, 3.16]
RADII = [INF, 0.3, 2.0]


def _cloud(n, seed, scale=3.0):
    return np.random.default_rng(seed).normal(size=(n, 3)) * scale


def _queries(T, seed, n):
    rng = np.random.default_rng(seed)
    m = n // 2
    near = T[rng.integers(0, len(T), m)] + rng.normal(size=(m, 3)) * 0.2
    return np.concatenate([near, rng.normal(size=(n - m, 3)) * 4.0, T[:3]])


def _check(T, Q, k, eps, radius, self_match, bucket=8):
    flags = OK.ALLOW_SELF_MATCH if self_match else 0
    ids_o, d2_o = OK.knn(T, Q, k, eps, radius, flags, bucket)
    ids_g, d2_g = smb.knn(T, Q, k, epsilon=eps, max_radius=radius, allow_self_match=self_match, bucket_size=bucket)
    ctx = dict(nt=len(T), nq=len(Q), k=k, eps=eps, radius=radius, self_match=self_match, bucket=bucket)
    assert ids_g.shape == (len(Q), k), ctx
    bad = np.flatnonzero(np.any(ids_g != ids_o, axis=1) | np.any(d2_g.view(np.int64) != d2_o.view(np.int64), axis=1))
    assert bad.size == 0, (ctx, bad[:5], ids_g[bad[:1]], ids_o[bad[:1]], d2_g[bad[:1]], d2_o[bad[:1]])


@pytest.mark.parametrize("k", KS)
def test_every_k_epsilon_radius_and_self_match(k):
    T = _cloud(6000, k)
    Q = np.concatenate([_queries(T, k + 100, 3000), T[::7]])
    for eps in EPSILONS:
        for radius in RADII:
            for self_match in (True, False):
                _check(T, Q, k, eps, radius, self_match)


@pytest.mark.parametrize("bucket", range(2, 9))
def test_every_bucket_past_the_launch_path_changes(bucket):
    cap = M.sub_capacity(bucket)
    sizes = [1, bucket, bucket + 1, cap, cap + 1, 2 * cap, 2 * cap + 1, 262_145]
    for i, nt in enumerate(sizes):
        T = _cloud(nt, nt + bucket)
        Q = _queries(T, nt, 1500)
        for k, eps, radius, self_match in ((KS[i % len(KS)], EPSILONS[i % 3], RADII[i % 3], i % 2 == 0),
                                           (KS[(i + 5) % len(KS)], EPSILONS[(i + 1) % 3], RADII[(i + 2) % 3],
                                            i % 2 == 1),
                                           (64, 0.5, INF, True)):
            _check(T, Q, k, eps, radius, self_match, bucket)


@pytest.mark.parametrize("k,eps,radius", [(1, 3.16, INF), (8, 0.0, INF), (20, 0.5, 2.0), (64, 3.16, 0.3), (33, 0.0, 2.0)])
def test_icp_sizes(k, eps, radius):
    # 120 k queries against a 107 k-point target: the tree is deeper than the levels staged in shared memory
    rng = np.random.default_rng(k)
    T = np.concatenate([rng.uniform(-40, 40, size=(107_000, 3)) * [1.0, 1.0, 0.1]])
    Q = np.concatenate([T[rng.integers(0, len(T), 60_000)] + rng.normal(size=(60_000, 3)) * 0.05,
                        rng.uniform(-45, 45, size=(60_000, 3)) * [1.0, 1.0, 0.1]])
    _check(T, Q, k, eps, radius, True)
    _check(T, Q, k, eps, radius, False)


@pytest.mark.parametrize("name,T", list(_adversarial_clouds()), ids=[n for n, _ in _adversarial_clouds()])
def test_adversarial_scenes(name, T):
    rng = np.random.default_rng(len(name))
    Q = np.concatenate([T + rng.normal(size=T.shape) * 0.3, rng.normal(size=(300, 3)) * np.abs(T).max(), T])
    scale = float(np.abs(T).max()) or 1.0
    for k in KS:
        for eps, radius, self_match in ((0.0, INF, True), (3.16, 0.3 * scale, False), (0.5, 2.0, True)):
            _check(T, Q, k, eps, radius, self_match)


@pytest.mark.parametrize("eps", EPSILONS)
@pytest.mark.parametrize("nt", [1, 9, 5000, 107_000])
def test_k1_equals_knn1(nt, eps):
    T = _cloud(nt, 3)
    Q = _queries(T, 4, 20_000)
    ids, d2 = smb.knn(T, Q, 1, epsilon=eps)
    ids1, d21 = smb.knn1(T, Q, epsilon=eps)
    assert np.array_equal(ids[:, 0], ids1) and np.array_equal(d2[:, 0].view(np.int64), d21.view(np.int64))


def _device_knn(lib, T, Q, k, eps, radius, flags, stream):
    import torch
    t = torch.from_numpy(T).cuda()
    q = torch.from_numpy(Q).cuda()
    ids = torch.empty((len(Q), k), dtype=torch.int32, device="cuda")
    d2 = torch.empty((len(Q), k), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    rc = lib.sm_knn_device(0, t.data_ptr(), len(T), q.data_ptr(), len(Q), k, eps, radius, flags, 8, ids.data_ptr(),
                           d2.data_ptr(), C.c_void_p(stream.cuda_stream))
    assert rc == 0
    return ids.cpu().numpy(), d2.cpu().numpy()


def test_device_entry_point_equals_host_entry_point():
    import torch
    lib = _lib.lib()
    T = _cloud(40_000, 61)
    Q = _queries(T, 62, 30_000)
    s = torch.cuda.Stream()
    for k, eps, radius, flags in ((1, 3.16, INF, 1), (8, 0.0, 2.0, 0), (20, 0.5, INF, 3), (64, 0.0, 0.3, 1)):
        ids_d, d2_d = _device_knn(lib, T, Q, k, eps, radius, flags, s)
        ids_h, d2_h = smb.knn(T, Q, k, eps, radius, bool(flags & 1))
        assert np.array_equal(ids_d, ids_h) and np.array_equal(d2_d.view(np.int64), d2_h.view(np.int64))


def test_two_threads_on_two_streams_equal_one():
    import torch
    lib = _lib.lib()
    jobs = [(_cloud(50_000, 71), 7, 0.5, INF, 1), (_cloud(30_000, 72), 33, 0.0, 2.0, 0)]
    jobs = [(T, _queries(T, 73 + i, 40_000), k, eps, radius, flags) for i, (T, k, eps, radius, flags) in enumerate(jobs)]
    alone = [_device_knn(lib, T, Q, k, eps, radius, flags, torch.cuda.Stream()) for T, Q, k, eps, radius, flags in jobs]
    out = [None, None]
    errors = []

    def run(i):
        try:
            T, Q, k, eps, radius, flags = jobs[i]
            for _ in range(3):
                out[i] = _device_knn(lib, T, Q, k, eps, radius, flags, torch.cuda.Stream())
                assert np.array_equal(out[i][0], alone[i][0]) and np.array_equal(out[i][1], alone[i][1])
        except Exception as e:      # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    host = [smb.knn(T, Q, k, eps, radius, bool(flags & 1)) for T, Q, k, eps, radius, flags in jobs]
    for (ids_t, d2_t), (ids_h, d2_h) in zip(out, host):
        assert np.array_equal(ids_t, ids_h) and np.array_equal(d2_t, d2_h)


def test_python_rejects_bad_arguments():
    T = _cloud(100, 81)
    for kw in (dict(k=0), dict(k=65), dict(k=4, epsilon=-0.1), dict(k=4, max_radius=float("nan")),
               dict(k=4, bucket_size=9)):
        with pytest.raises(ValueError):
            smb.knn(T, T, **kw)
