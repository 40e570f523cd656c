"""IcpFast with inner compensation on the CPU: the C++ restatement (tests/cpp/icp_compensation_oracle.cc) against
the numpy one (tests/pyref_compensation.py), against a scene with a known answer, against the plain oracle with the flag clear, and the
engine's host build of its per-point arithmetic against the oracle's pieces."""
import ctypes as C

import numpy as np
import pytest

import inner_compensation_scenes as ICS
import oracle_compensation as OC
import oracle_lib as O
import pyref_compensation
import scenes
from staticmapping_b200 import _lib


def _knn(t, P):
    return O.knn1(t, P, epsilon=3.16)


def _scene(name):
    if name == "corner":
        src, _, _ = scenes.corner_pair()
        tp, tn = ICS.corner_target()
        return src, tp, tn, np.eye(4)
    src, sub, P = scenes.lidar_pair(pair=1)
    tp, tn = O.calculate_normals(sub)
    return src, tp, tn, np.linalg.inv(P) @ np.eye(4) @ P   # the identity guess, as the mapper's first try


@pytest.mark.parametrize("disable_convergence", [False, True])
@pytest.mark.parametrize("name", ["corner", "lidar"])
def test_oracle_matches_python_restatement(name, disable_convergence):
    src, tp, tn, guess = _scene(name)
    kw = dict(max_iteration=30 if disable_convergence else 100, disable_convergence_check=disable_convergence)
    o = OC.icp_fast_align(src, tp, tn, guess, inner_compensation=True, trace=True, **kw)
    tr = []
    p = pyref_compensation.icp_fast_align(src, tp, tn, _knn, guess, trace=tr, **kw)
    assert o["rc"] == 1
    assert o["iterations"] == p["iterations"]
    for k, (a, b) in enumerate(zip(o["trace"], tr)):
        assert np.abs(a["T_iter"] - b["T_iter"]).max() <= 1e-12
        assert a["kept"] == b["kept"]
        # the limit is one of the k-NN distances: bit-identical while the iterate is (iteration 1), to rounding
        # afterwards (LAPACK vs the oracle's Eigen-style 6x6 solve)
        if k == 0:
            assert a["limit"] == b["limit"]
        assert abs(a["limit"] - b["limit"]) <= 1e-11 * max(1.0, abs(b["limit"]))
    dt, dr = scenes.se3_error(o["result"], p["result"])
    assert dt <= 1e-9 and dr <= 1e-9
    # the flag changes the answer on these scenes
    plain = O.icp_fast_align(src, tp, tn, guess, **kw)
    assert not np.array_equal(plain["result"], o["result"])


@pytest.mark.parametrize("name", ["corner", "lidar"])
def test_flag_clear_is_the_plain_oracle_bit_for_bit(name):
    src, tp, tn, guess = _scene(name)
    for kw in (dict(), dict(max_iteration=12, disable_convergence_check=True)):
        a = OC.icp_fast_align(src, tp, tn, guess, inner_compensation=False, trace=True, **kw)
        b = O.icp_fast_align(src, tp, tn, guess, trace=True, **kw)
        assert a["rc"] == b["rc"] == 1 and a["iterations"] == b["iterations"]
        assert np.array_equal(a["result"], b["result"]) and a["score"] == b["score"]
        for x, y in zip(a["trace"], b["trace"]):
            assert np.array_equal(x["T_iter"], y["T_iter"]) and x["limit"] == y["limit"] and x["kept"] == y["kept"]
            assert np.array_equal(x["A"], y["A"]) and np.array_equal(x["b"], y["b"])


def test_model_exact_scene_recovers_the_motion():
    src, tp, tn, G, expected = ICS.model_exact()
    comp = OC.icp_fast_align(src, tp, tn, G, inner_compensation=True)
    dt, dr = scenes.se3_error(comp["result"], expected)
    assert dt <= 0.02 and dr <= np.radians(0.2), (dt, np.degrees(dr))
    plain = O.icp_fast_align(src, tp, tn, G)
    pdt, pdr = scenes.se3_error(plain["result"], expected)
    # plain ICP fits one rigid motion to the skewed scan and lands near the middle of the sweep
    assert pdt >= 0.1, (pdt, np.degrees(pdr))
    assert pdt >= 10 * dt


def test_one_point_source_takes_the_zero_jacobian_path():
    tp, tn = ICS.corner_target()
    src = tp[:1] + 0.01
    o = OC.icp_fast_align(src, tp, tn, inner_compensation=True, trace=True)
    assert o["rc"] == 1
    t0 = o["trace"][0]
    assert not t0["A"].any() and not t0["b"].any()             # f_0 = 0: the only match has a zero column
    assert np.array_equal(t0["T_iter"], np.eye(4))             # x = 0
    assert o["iterations"] == 4                                # four identities after the initial one: converged


def _host_hook(T, pts, q, n):
    lib = _lib.lib()
    k = pts.shape[0]
    out_p = np.zeros((k, 3)); out_t = np.zeros((k, 7))
    Tc = np.ascontiguousarray(T.T).ravel()
    rc = lib.sm_debug_inner_compensation_host(Tc.ctypes.data_as(_lib._DP), np.ascontiguousarray(pts).ctypes.data,
                                              np.ascontiguousarray(q).ctypes.data, np.ascontiguousarray(n).ctypes.data,
                                              k, out_p.ctypes.data, out_t.ctypes.data)
    assert rc == 0
    return out_p, out_t


@pytest.mark.parametrize("angle", [0.0, 1e-9, 0.7, 25.0, 179.0])
def test_host_hook_is_bit_identical_to_the_oracle_pieces(angle):
    rng = np.random.default_rng(int(angle * 10) + 3)
    k = 257
    T = ICS.se3(angle, (0.3, -0.5, 0.8), (1.5, -0.7, 0.2)) if angle else np.eye(4)
    if angle:
        T[:3, :3] += rng.normal(scale=1e-12, size=(3, 3))        # T_iter is never re-orthonormalised
    pts = rng.normal(size=(k, 3)) * 20.0
    q = pts + rng.normal(size=(k, 3))
    n = rng.normal(size=(k, 3)); n /= np.linalg.norm(n, axis=1)[:, None]
    got_p, got_t = _host_hook(T, pts, q, n)
    for i in range(k):
        f = i / k
        rc, Ti = O.interpolate_transform(np.eye(4), T, np.float32(f))
        assert rc == 0
        x, y, z = pts[i]
        p = [((Ti[r, 0] * x + Ti[r, 1] * y) + Ti[r, 2] * z) + Ti[r, 3] for r in range(3)]
        assert list(got_p[i]) == p, i
        F = [p[1] * n[i, 2] - p[2] * n[i, 1], p[2] * n[i, 0] - p[0] * n[i, 2], p[0] * n[i, 1] - p[1] * n[i, 0],
             n[i, 0], n[i, 1], n[i, 2]]
        dot = ((p[0] - q[i, 0]) * n[i, 0] + (p[1] - q[i, 1]) * n[i, 1]) + (p[2] - q[i, 2]) * n[i, 2]
        assert list(got_t[i, :6]) == [v * f for v in F] and got_t[i, 6] == dot, i
