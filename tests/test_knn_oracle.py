"""libnabo's k-NN (sm_knn) without a GPU: the oracle (tests/cpp/knn_oracle.cc) against an independent Python
restatement (tests/pyref_knn.py), against the oracle's own 1-NN, against scipy's cKDTree and brute force, the radius,
self-match and tie rules, the kernel's search formulation (tests/gpu_knn_k_model.py), and the C ABI's argument checks."""
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

import oracle_knn as OK
import oracle_lib as O
import pyref_knn
from gpu_knn_k_model import GpuKnnKModel
from staticmapping_b200 import _lib
from test_search_formulation_model import _adversarial_clouds

INF = float("inf")
DBL_EPSILON = sys.float_info.epsilon


def _cloud(n, seed, scale=2.0):
    return np.random.default_rng(seed).normal(size=(n, 3)) * scale


def _queries(T, seed, n=60):
    rng = np.random.default_rng(seed)
    near = T[rng.integers(0, len(T), n // 2)] + rng.normal(size=(n // 2, 3)) * 0.2
    return np.concatenate([near, rng.normal(size=(n - n // 2, 3)) * 3.0, T[:3]])


def _brute_d2(T, q):
    d = q[None, :] - T
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


@pytest.mark.parametrize("k", [1, 2, 3, 7, 8, 9, 20, 33, 64])
@pytest.mark.parametrize("eps,radius", [(0.0, INF), (0.5, 1.0), (3.16, INF), (0.0, 0.3)])
def test_oracle_equals_python_restatement(k, eps, radius):
    T = _cloud(350, k)
    Q = _queries(T, k + 1)
    for flags, bucket in ((1, 8), (0, 2), (3, 5)):
        ids_o, d2_o = OK.knn(T, Q, k, eps, radius, flags, bucket)
        ids_p, d2_p = pyref_knn.PyNaboK(T, bucket).knn(Q, k, eps, radius, flags)
        assert np.array_equal(ids_o, ids_p)
        assert np.array_equal(d2_o.view(np.int64), d2_p.view(np.int64))


@pytest.mark.parametrize("bucket", [2, 3, 8])
@pytest.mark.parametrize("eps", [0.0, 0.5, 3.16])
def test_k1_equals_the_oracle_1nn(bucket, eps):
    T = _cloud(2000, 7)
    Q = _queries(T, 8, 400)
    ids, d2 = OK.knn(T, Q, 1, eps, INF, OK.ALLOW_SELF_MATCH, bucket)
    ids1, d21 = O.knn1(T, Q, epsilon=eps, bucket_size=bucket)
    assert np.array_equal(ids[:, 0], ids1) and np.array_equal(d2[:, 0], d21)


@pytest.mark.parametrize("k", [1, 5, 8, 20, 64])
def test_exact_search_equals_ckdtree(k):
    T = _cloud(3000, 11)
    Q = _queries(T, 12, 300)
    ids, d2 = OK.knn(T, Q, k, 0.0)
    dd, ii = cKDTree(T).query(Q, k=k)
    dd, ii = dd.reshape(len(Q), k), ii.reshape(len(Q), k)
    assert np.allclose(d2, dd * dd, rtol=1e-12, atol=0.0)
    for j, q in enumerate(Q):
        b = _brute_d2(T, q)
        # random normal coordinates: no two distances tie, so the sets are equal and the order is the distance order
        assert set(ids[j].tolist()) == set(ii[j].tolist())
        assert np.array_equal(d2[j], b[ids[j]]) and np.all(np.diff(d2[j]) > 0)


@pytest.mark.parametrize("radius", [0.0, 0.25, 0.7, 2.0])
@pytest.mark.parametrize("k", [1, 7, 64])
def test_radius_rule(k, radius):
    T = _cloud(1500, 21, scale=1.0)
    Q = _queries(T, 22, 200)
    ids, d2 = OK.knn(T, Q, k, 0.0, radius)
    for j, q in enumerate(Q):
        b = _brute_d2(T, q)
        inside = np.sort(b[b <= radius * radius])[:k]
        n = len(inside)
        assert np.array_equal(d2[j, :n], inside)
        assert np.all(ids[j, n:] == -1) and np.all(d2[j, n:] == INF)


@pytest.mark.parametrize("eps", [0.0, 3.16])
def test_self_match_rule(eps):
    T = _cloud(800, 31)
    T = np.concatenate([T, T[:5] + 1e-9])          # near-duplicates at d2 ~ 3e-18 <= DBL_EPSILON: dropped too
    ids_on, d2_on = OK.knn(T, T, 4, eps, INF, OK.ALLOW_SELF_MATCH)
    ids_off, d2_off = OK.knn(T, T, 4, eps, INF, 0)
    assert np.all(d2_on[:, 0] == 0.0)
    assert np.all(d2_off > DBL_EPSILON)
    exact_off, _ = OK.knn(T, T, 4, 0.0, INF, 0)
    for j in range(0, len(T), 37):
        b = _brute_d2(T, T[j])
        assert not np.any(exact_off[j] == j)
        assert np.array_equal(np.sort(b[b > DBL_EPSILON])[:4], _brute_d2(T, T[j])[exact_off[j]])


def test_sort_results_flag_changes_nothing():
    T = _cloud(900, 41)
    Q = _queries(T, 42)
    for k in (3, 20):
        a = OK.knn(T, Q, k, 0.5, 1.5, OK.ALLOW_SELF_MATCH)
        b = OK.knn(T, Q, k, 0.5, 1.5, OK.ALLOW_SELF_MATCH | OK.SORT_RESULTS)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert np.all(a[1][:, :-1] <= a[1][:, 1:])


def test_k_above_n_target_pads():
    T = _cloud(5, 51)
    ids, d2 = OK.knn(T, _queries(T, 52, 10), 9)
    assert np.all(ids[:, 5:] == -1) and np.all(d2[:, 5:] == INF)
    assert np.all(np.sort(ids[:, :5], axis=1) == np.arange(5))


def test_tie_order_identical_points():
    # 100 copies of one point: every distance ties, so the list holds the first k points the search visits, in that
    # order, and a tie with the k-th entry is rejected
    T = np.tile([[1.5, -2.0, 0.25]], (100, 1))
    Q = np.array([[1.5, -2.0, 0.25], [0.0, 0.0, 0.0], [10.0, 3.0, -1.0]])
    for k, bucket in ((1, 8), (7, 8), (20, 3), (64, 2)):
        ids, d2 = OK.knn(T, Q, k, 0.0, INF, 1, bucket)
        ids_p, d2_p = pyref_knn.PyNaboK(T, bucket).knn(Q, k)
        assert np.array_equal(ids, ids_p) and np.array_equal(d2, d2_p)
        assert len(set(ids[0].tolist())) == k and np.all(d2[:, 1:] == d2[:, :1])


@pytest.mark.parametrize("k", [6, 27, 64])
def test_tie_order_grid(k):
    g = np.stack(np.meshgrid(np.arange(9.0), np.arange(7.0), np.arange(4.0)), -1).reshape(-1, 3)
    Q = np.concatenate([g[::11], g[::13] + 0.5])
    for eps in (0.0, 0.5):
        ids, d2 = OK.knn(g, Q, k, eps, 2.5)
        ids_p, d2_p = pyref_knn.PyNaboK(g).knn(Q, k, eps, 2.5)
        assert np.array_equal(ids, ids_p) and np.array_equal(d2, d2_p)
        if eps == 0.0:     # the distances are the k smallest within the radius, whichever tied points were kept
            for j, q in enumerate(Q):
                b = _brute_d2(g, q)
                inside = np.sort(b[b <= 6.25])[:k]
                assert np.array_equal(d2[j, :len(inside)], inside)


@pytest.mark.parametrize("name,T", list(_adversarial_clouds()), ids=[n for n, _ in _adversarial_clouds()])
def test_kernel_formulation_equals_the_oracle_on_adversarial_clouds(name, T):
    rng = np.random.default_rng(len(name))
    step = max(1, len(T) // 60)
    Q = np.concatenate([T[::step] + rng.normal(size=(len(T[::step]), 3)) * 0.3,
                        rng.normal(size=(30, 3)) * np.abs(T).max(), T[:2]])
    m = GpuKnnKModel(T)
    r_scale = float(np.abs(T).max()) or 1.0
    for k, eps, radius, flags in ((1, 3.16, INF, 1), (3, 0.0, INF, 0), (8, 0.5, 0.3 * r_scale, 1),
                                  (9, 3.16, 2.0, 0), (33, 0.0, 0.05 * r_scale, 1), (64, 0.5, INF, 1)):
        ids_o, d2_o = OK.knn(T, Q, k, eps, radius, flags)
        ids_m, d2_m = m.knn(Q, k, eps, radius, flags)
        assert np.array_equal(ids_m, ids_o), (k, eps, radius, flags)
        assert np.array_equal(d2_m.view(np.int64), d2_o.view(np.int64)), (k, eps, radius, flags)


@pytest.mark.parametrize("nt,bucket", [(1, 8), (9, 8), (300, 2), (1000, 8), (2049, 5)])
def test_kernel_formulation_equals_the_oracle(nt, bucket):
    T = _cloud(nt, nt)
    Q = _queries(T, nt + 1, 80)
    m = GpuKnnKModel(T, bucket)
    for k, eps, radius, flags in ((1, 0.0, INF, 1), (7, 3.16, INF, 0), (20, 0.5, 1.0, 1), (64, 0.0, 2.0, 0)):
        ids_o, d2_o = OK.knn(T, Q, k, eps, radius, flags, bucket)
        ids_m, d2_m = m.knn(Q, k, eps, radius, flags)
        assert np.array_equal(ids_m, ids_o) and np.array_equal(d2_m, d2_o)


def _abi_call(k=4, eps=0.0, radius=INF, flags=1, bucket=8, nt=10, nq=3, target=True):
    lib = _lib.lib()
    T = np.zeros((max(nt, 1), 3))
    Q = np.zeros((max(nq, 1), 3))
    ids = np.empty(max(nq, 1) * 64, dtype=np.int32)
    d2 = np.empty(max(nq, 1) * 64)
    return lib.sm_knn(0, T.ctypes.data if target else None, nt, Q.ctypes.data, nq, k, eps, radius, flags, bucket,
                      ids.ctypes.data, d2.ctypes.data)


@pytest.mark.parametrize("kw", [dict(k=0), dict(k=65), dict(k=-3), dict(eps=-1e-300), dict(eps=float("nan")),
                                dict(radius=-1.0), dict(radius=float("nan")), dict(bucket=1), dict(bucket=9),
                                dict(flags=4), dict(flags=0x80000000), dict(nt=0), dict(nq=-1), dict(target=False)],
                         ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_abi_rejects_bad_arguments(kw):
    # the checks run before a device is selected, so they hold on a machine without one
    assert _abi_call(**kw) == -1


def test_oracle_rejects_what_the_abi_rejects():
    T = _cloud(10, 1)
    for args in ((0, 0.0, INF, 1, 8), (65, 0.0, INF, 1, 8), (3, -1.0, INF, 1, 8), (3, float("nan"), INF, 1, 8),
                 (3, 0.0, -1.0, 1, 8), (3, 0.0, float("nan"), 1, 8), (3, 0.0, INF, 4, 8), (3, 0.0, INF, 1, 9)):
        with pytest.raises(ValueError):
            OK.knn(T, T, *args)
