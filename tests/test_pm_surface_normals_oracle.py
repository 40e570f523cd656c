"""The eigenvector leaf of libpointmatcher's SamplingSurfaceNormalDataPointsFilter (knn 7), the reference filter type 1
runs with sm_set_pm_surface_normals(EIGENVECTOR), without a GPU.  Three statements of it meet here:
  - the product's leaf (csrc/normals.cu leaf_eigen_normal) compiled for the host, through
    sm_debug_pm_surface_normal_leaf_host;
  - the oracle (oracle/pm_surface_normals_oracle.cc), a twin transcription: the same operation order, no contraction,
    so means, covariances and normals agree bit for bit;
  - tests/pyref.py pm_sampling_surface_normal, the literal numpy restatement (float sums, LAPACK's eigh, numpy's rank),
    which is independent of both: means bit for bit, normals within the conditioning of the eigenproblem, and the
    kept / dropped decision equal away from boxes built on the rank border."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as O
import oracle_pm_surface_normals as PN
import pyref
import scenes
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
U = float(np.finfo(F32).eps) / 2                      # unit roundoff of float


def hook_leaf(members):
    m = np.ascontiguousarray(members, dtype=F32)
    mean = np.zeros(3, F32); cov = np.zeros(9, F32); nrm = np.zeros(3, F32); kept = C.c_int32(-1)
    rc = _lib.lib().sm_debug_pm_surface_normal_leaf_host(m.ctypes.data, m.shape[0], mean.ctypes.data, cov.ctypes.data,
                                                         nrm.ctypes.data, C.byref(kept))
    assert rc == 0
    return bool(kept.value), mean, cov.reshape(3, 3), (nrm if kept.value else None)


def _rng_box(rng, count, kind):
    """One box of `count` float members of the given kind."""
    if kind == "generic":
        return rng.uniform(-1.0, 1.0, size=(count, 3)).astype(F32)
    if kind == "far":                                 # far from the origin: the float mean cancels most digits
        return (rng.uniform(-1e4, 1e4, size=3) + rng.uniform(-0.3, 0.3, size=(count, 3))).astype(F32)
    if kind == "plane":                               # a clear plane with millimetre noise
        uv = rng.uniform(-0.5, 0.5, size=(count, 2))
        n = rng.normal(size=3); n /= np.linalg.norm(n)
        a = np.cross(n, [1.0, 0.0, 0.0] if abs(n[0]) < 0.9 else [0.0, 1.0, 0.0]); a /= np.linalg.norm(a)
        b = np.cross(n, a)
        c = rng.uniform(-20, 20, size=3)
        return (c + uv[:, :1] * a + uv[:, 1:] * b + rng.normal(scale=1e-3, size=(count, 1)) * n).astype(F32)
    if kind == "close":                               # a rod: the two smallest eigenvalues nearly equal
        x = rng.uniform(-1.0, 1.0, size=(count, 1))
        return np.hstack([x, rng.normal(scale=0.05, size=(count, 2))]).astype(F32) + F32(3.0)
    if kind == "axis_line":                           # exactly collinear in float: C has one non-zero entry
        p = np.zeros((count, 3), F32) + rng.uniform(-5, 5, size=3).astype(F32)
        p[:, rng.integers(3)] += rng.uniform(-1, 1, size=count).astype(F32)
        return p
    if kind == "diagonal_line":                       # exactly collinear along (1, 1, 0), integer steps
        t = rng.integers(-8, 8, size=count).astype(F32)
        return np.stack([t + F32(2.0), t - F32(1.0), np.full(count, F32(0.5))], axis=1)
    if kind == "coincident":
        return np.repeat(rng.uniform(-3, 3, size=(1, 3)).astype(F32), count, axis=0)
    raise ValueError(kind)


KINDS = ["generic", "far", "plane", "close", "axis_line", "diagonal_line", "coincident"]
DEGENERATE = {"axis_line", "diagonal_line", "coincident"}


def _boxes():
    rng = np.random.default_rng(20261018)
    for kind in KINDS:
        for count in range(1, 8):
            for _ in range(12):
                yield kind, _rng_box(rng, count, kind)


def test_hook_and_oracle_agree_bit_for_bit():
    seen = {"kept": 0, "dropped": 0}
    for kind, box in _boxes():
        hk, hm, hc, hn = hook_leaf(box)
        ok, om, oc, on = PN.pm_surface_normal_leaf(box)
        assert hk == ok, (kind, box)
        assert hm.tobytes() == om.tobytes() and hc.tobytes() == oc.tobytes(), (kind, box)
        if hk:
            assert hn.tobytes() == on.tobytes(), (kind, box)
            assert abs(float(np.linalg.norm(hn.astype(np.float64))) - 1.0) < 4 * U
            big = int(np.argmax(np.abs(hn)))
            assert hn[big] > 0                         # the sign rule
        seen["kept" if hk else "dropped"] += 1
        if kind in DEGENERATE or box.shape[0] == 1:
            assert not hk, (kind, box)                 # collinear, coincident or one member: rank(C) + 1 < 3
        # two members lie on the rank border: d_0 - mean and d_1 - mean are opposite only up to the float rounding of
        # the mean, so far from the origin C can have rank 2 in float, and the box is kept as libpointmatcher keeps it
    assert seen["kept"] > 200 and seen["dropped"] > 200, seen


def test_against_numpy():
    """pyref on each box alone (a cloud of <= 7 points is one box): means bit for bit; normals up to sign within
    c * u * |C| / (lambda_2 - lambda_1), the first-order bound of an eigenvector's error over its gap; and the same
    boxes kept.  The constructed degenerate boxes lie on the rank border, where the two rank rules may differ."""
    worst = 0.0
    for kind, box in _boxes():
        hk, hm, hc, hn = hook_leaf(box)
        pm, pn = pyref.pm_sampling_surface_normal(box, 7)
        mean_np = box.T.sum(axis=1, dtype=F32) / F32(box.shape[0])
        assert hm.tobytes() == mean_np.tobytes(), (kind, box)
        if kind not in DEGENERATE:
            assert hk == (pm.shape[0] == 1), (kind, box)
        if not (hk and pm.shape[0] == 1):
            continue
        assert pm[0].tobytes() == hm.tobytes()
        w = np.linalg.eigvalsh(hc.astype(np.float64))
        gap = w[1] - w[0]
        scale = max(abs(w[2]), abs(w[0]))
        sin = float(np.linalg.norm(np.cross(hn.astype(np.float64), pn[0].astype(np.float64))))
        if gap > 0:
            ratio = sin / (U * scale / gap + U)
            worst = max(worst, ratio)
            assert ratio < 64, (kind, box, sin, gap, scale)
    assert worst > 0.0


def test_whole_filter_oracle_against_pyref():
    """The whole filter: the same boxes in the same order, the means bit for bit, the normals up to sign and within the
    conditioning bound; and the same boxes as CalculateNormals (whose kept points are double means)."""
    _, tgt, _ = scenes.corner_pair()
    _, sub, _ = scenes.lidar_pair(submap_points=20000)
    for cloud in (tgt.astype(F32), sub.astype(F32)):
        om, on, oi = PN.pm_surface_normals(cloud)
        pm, pn = pyref.pm_sampling_surface_normal(cloud, 7)
        assert om.shape == pm.shape and om.shape[0] > 0.1 * cloud.shape[0] / 7
        assert om.tobytes() == pm.tobytes()
        sin = np.linalg.norm(np.cross(on.astype(np.float64), pn.astype(np.float64)), axis=1)   # sign-free
        assert np.median(sin) < 1e-7 and sin.max() < 1e-4       # observed 1e-9 and 5e-6: float eigh vs double Jacobi
        assert (on[np.arange(on.shape[0]), np.argmax(np.abs(on), axis=1)] > 0).all()
        assert np.all(np.diff(oi) > 0)
        tp, _ = O.calculate_normals(cloud.astype(np.float64))
        assert tp.shape == om.shape and np.allclose(tp, om, rtol=0, atol=1e-4 * max(1.0, np.abs(tp).max()))


def test_reference_filter_modes_of_the_oracle_chain():
    """icp_pm_equivalent(normals=...): the default keeps today's chain, "eigenvector" runs the filter's own leaf."""
    src, tgt, _ = scenes.corner_pair()
    s32, t32 = src.astype(F32), tgt.astype(F32)
    a = O.icp_pm_equivalent(s32, t32)
    b = PN.icp_pm_equivalent(s32, t32, normals="least_squares")
    assert a["result"].tobytes() == b["result"].tobytes() and a["score"] == b["score"]
    e = PN.icp_pm_equivalent(s32, t32, normals="eigenvector")
    assert e["rc"] == 1 and e["ok"] and e["n_target"] == a["n_target"]
    assert not np.array_equal(e["result"], a["result"])
    with pytest.raises(ValueError):
        PN.icp_pm_equivalent(s32, t32, normals="svd")


def test_abi_without_device():
    lib = _lib.lib()
    assert lib.sm_set_pm_surface_normals(None, 0) == -1
    assert int(smb.SurfaceNormals.LEAST_SQUARES) == 0 and int(smb.SurfaceNormals.EIGENVECTOR) == 1
    with open(os.path.join(ROOT, "include", "sm_b200.h")) as f:
        h = f.read()
    assert "SM_PM_NORMALS_LEAST_SQUARES = 0" in h and "SM_PM_NORMALS_EIGENVECTOR = 1" in h
    assert "int sm_set_pm_surface_normals(sm_handle* h, int32_t mode);" in h
    z = np.zeros(3 * 8, F32); out = np.zeros(16, F32); kept = C.c_int32()
    for bad in (0, 8):
        assert lib.sm_debug_pm_surface_normal_leaf_host(z.ctypes.data, bad, out.ctypes.data, out.ctypes.data,
                                                        out.ctypes.data, C.byref(kept)) == -1
    assert lib.sm_debug_pm_surface_normal_leaf_host(None, 3, out.ctypes.data, out.ctypes.data, out.ctypes.data,
                                                    C.byref(kept)) == -1
    m = C.c_int64()
    assert lib.sm_debug_pm_surface_normals(0, 2, None, 0, z.ctypes.data, 8, out.ctypes.data, out.ctypes.data,
                                           out.ctypes.data, C.byref(m)) == -1   # unknown mode, before any device
