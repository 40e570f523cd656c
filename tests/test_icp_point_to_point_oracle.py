"""IcpFast's point-to-point minimizer without a GPU: the C++ oracle (tests/cpp/icp_point_to_point_oracle.cc) against
the numpy restatement (tests/pyref_point_to_point.py) iteration by iteration, the product's Kabsch solve compiled
for the host (sm_debug_kabsch_host) against numpy and the oracle, and the ABI's argument checks."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as O
import oracle_point_to_point as OP
import point_to_point_scenes as S
import pyref_point_to_point as PP
import scenes
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _knn(Q, P):
    return O.knn1(Q, P, epsilon=3.16)


def _is_rotation(R, tol=1e-12):
    return np.abs(R.T @ R - np.eye(3)).max() <= tol and abs(np.linalg.det(R) - 1.0) <= tol


@pytest.mark.parametrize("name", list(S.SCENES))
def test_oracle_matches_numpy_every_iteration(name):
    src, tp, _, guess, mi = S.SCENES[name]()
    o = OP.icp_fast_align(src, tp, guess, max_iteration=mi, trace=True)
    assert o["rc"] == 1
    tr = []
    p = PP.icp_fast_align(src, tp, _knn, guess, max_iteration=mi, trace=tr)
    for k, t in enumerate(o["trace"]):
        assert _is_rotation(t["R"])
        if name not in S.UNIQUE or name == "identical":
            break   # R is not unique, or (identical clouds) d2 ~ 0 ties at the limit fall either way on rounding
        assert t["kept"] == tr[k]["kept"] and abs(t["limit"] - tr[k]["limit"]) <= 1e-12 * max(t["limit"], 1e-300)
        if name in ("corner", "reflection"):   # full-rank M: sign(det(U V^T)) = sign(det M) whichever SVD
            assert (t["path"] == 4) == tr[k]["fix"]
        assert np.abs(t["T_iter"] - tr[k]["T_iter"]).max() <= 1e-9, k
    if name in S.UNIQUE:
        dt, dr = scenes.se3_error(o["result"], p["result"])
        assert dt <= 1e-9 and dr <= 1e-9
    if name in S.UNIQUE and name != "identical":
        assert o["iterations"] == p["iterations"]
        assert abs(o["score"] - p["score"]) <= 1e-12


def test_scene_properties():
    # the corner: with the reference's eps = 3.16 approximate search and its convergence test, point-to-point stops
    # 7 cm / 0.9 deg from the ground truth.  The search is the cause, together with the test stopping a slowly
    # creeping minimizer: with an exact search (eps = 0) and 100 iterations it reaches 8 mm / 0.3 deg.
    src, tp, _, guess, mi = S.corner()
    GT = scenes.corner_pair()[2]
    dt, dr = scenes.se3_error(GT, OP.icp_fast_align(src, tp, guess)["result"])
    assert dt <= 0.08 and dr <= np.radians(1.0), (dt, dr)
    exact = OP.icp_fast_align(src, tp, guess, knn_epsilon=0.0, disable_convergence_check=True)
    dt, dr = scenes.se3_error(GT, exact["result"])
    assert dt <= 0.01 and dr <= np.radians(0.3), (dt, dr)
    # identical clouds: identity
    src, tp, _, guess, mi = S.identical()
    o = OP.icp_fast_align(src, tp, guess, trace=True)
    assert np.abs(o["result"] - np.eye(4)).max() <= 1e-12
    # the mirrored slab takes the reflection fix in its first iteration
    src, tp, _, guess, mi = S.reflection()
    o = OP.icp_fast_align(src, tp, guess, max_iteration=mi, trace=True)
    assert o["trace"][0]["path"] == 4 and o["trace"][0]["kept"] == tp.shape[0]
    # one kept match: M = 0 exactly, R = I, the point moves onto its match
    src, tp, _, guess, mi = S.one_match()
    o = OP.icp_fast_align(src, tp, guess, max_iteration=1, trace=True)
    t0 = o["trace"][0]
    assert t0["kept"] == 1 and not t0["M"].any() and np.array_equal(t0["R"], np.eye(3))
    # collinear: M has rank 1 and the moved source lies on the target's line
    src, tp, _, guess, mi = S.collinear()
    o = OP.icp_fast_align(src, tp, guess, trace=True)
    assert np.linalg.matrix_rank(o["trace"][0]["M"], tol=1e-9 * np.abs(o["trace"][0]["M"]).max()) == 1
    moved = src @ o["result"][:3, :3].T + o["result"][:3, 3]
    d = tp[-1] / np.linalg.norm(tp[-1])
    assert np.linalg.norm(moved - np.outer(moved @ d, d), axis=1).max() <= 1e-3


def _sums(P, Q):
    """The phase-B/C moment record of pairs P, Q: [0..2] sum p, [3..5] sum q, [6 + 3i + j] sum q_i p_j, [27], [28]."""
    s = np.zeros(32)
    s[0:3] = P.sum(axis=0); s[3:6] = Q.sum(axis=0)
    s[6:15] = (Q.T @ P).ravel()
    s[27] = np.sqrt(((P - Q) ** 2).sum(axis=1)).sum(); s[28] = P.shape[0]
    return s


def _kabsch_host(s):
    R, t, path = np.zeros(9), np.zeros(3), C.c_int32(0)
    rc = _lib.lib().sm_debug_kabsch_host(s.ctypes.data, R.ctypes.data, t.ctypes.data, C.byref(path))
    assert rc == 0
    return R.reshape(3, 3), t, path.value


def _pairs(kind, rng):
    P = rng.normal(size=(50, 3)) * [3.0, 2.0, 1.0] + [1.0, -2.0, 0.5]
    if kind == "random":
        R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        R *= np.sign(np.linalg.det(R))
        Q = P @ R.T + [0.3, 0.1, -0.2] + rng.normal(size=P.shape) * 0.01
    elif kind == "reflected":
        Q = P * [1.0, 1.0, -1.0]
    elif kind == "rank1":
        P = np.outer(rng.normal(size=50), [1.0, 2.0, -1.0]) + [0.5, 0.5, 0.5]
        Q = np.outer(rng.normal(size=50), [0.0, 1.0, 1.0]) - [1.0, 0.0, 0.0]
    elif kind == "rank0":
        P = P[:1]; Q = P + [0.2, -0.1, 0.3]
    else:                         # repeated singular values: an isotropic cloud rotated about z
        P = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], float)
        c, s = np.cos(0.3), np.sin(0.3)
        Q = P @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T
    return P, Q


@pytest.mark.parametrize("kind", ["random", "reflected", "rank1", "rank0", "repeated"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_kabsch_host_against_numpy_and_oracle(kind, seed):
    P, Q = _pairs(kind, np.random.default_rng(seed))
    R, t, path = _kabsch_host(_sums(P, Q))
    o = OP.point_to_point(P, Q)
    T, fix = PP.compute_point_to_point(P, Q)
    assert _is_rotation(R) and path in (3, 4)
    assert np.abs(R - o["R"]).max() <= 1e-9 and np.abs(t - o["t"]).max() <= 1e-9 and path == o["path"]
    # the optimal objective, unique or not
    best = PP.kabsch_objective(T[:3, :3], P, Q)
    assert PP.kabsch_objective(R, P, Q) <= best + 1e-9 * max(1.0, best)
    if kind in ("random", "reflected"):
        assert np.abs(R - T[:3, :3]).max() <= 1e-9 and np.abs(t - T[:3, 3]).max() <= 1e-9
        assert (path == 4) == fix == (kind == "reflected")
    if kind == "rank0":
        assert np.array_equal(R, np.eye(3)) and path == 3 and np.allclose(t, Q[0] - P[0], atol=0, rtol=1e-15)


def test_abi_without_device():
    lib = _lib.lib()
    assert lib.sm_set_icp_error_minimizer(None, 0) == -1
    assert int(smb.ErrorMinimizer.POINT_TO_PLANE) == 0 and int(smb.ErrorMinimizer.POINT_TO_POINT) == 1
    with open(os.path.join(ROOT, "include", "sm_b200.h")) as f:
        h = f.read()
    assert "SM_ICP_POINT_TO_PLANE = 0" in h and "SM_ICP_POINT_TO_POINT = 1" in h
    assert "int sm_set_icp_error_minimizer(sm_handle* h, int32_t minimizer);" in h
