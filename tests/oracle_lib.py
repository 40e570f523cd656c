"""ctypes binding of oracle/libsm_oracle.so — the CPU restatement used as the parity
checker.  TEST INFRASTRUCTURE: only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this module."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = os.path.join(_ROOT, "oracle")
_SO = os.path.join(_DIR, "libsm_oracle.so")


class IcpOptions(C.Structure):
    _fields_ = [("max_iteration", C.c_int32), ("dist_outlier_ratio", C.c_float),
                ("knn_epsilon", C.c_double), ("disable_convergence_check", C.c_int32),
                ("tie_mode", C.c_int32)]


class IcpTrace(C.Structure):
    _fields_ = [("T_iter", C.c_double * 16), ("limit", C.c_double), ("kept", C.c_int64),
                ("A", C.c_double * 36), ("b", C.c_double * 6)]


class NdtOptions(C.Structure):
    _fields_ = [("resolution", C.c_float), ("step_size", C.c_double), ("outlier_ratio", C.c_double),
                ("transformation_epsilon", C.c_double), ("max_iterations", C.c_int32)]


class NdtGicpOptions(C.Structure):
    _fields_ = [("voxel_resolution", C.c_float), ("using_voxel_filter", C.c_int32), ("use_ndt", C.c_int32)]


class NdtGicpInfo(C.Structure):
    _fields_ = [("n_source_filtered", C.c_int64), ("n_target_filtered", C.c_int64),
                ("ndt_iterations", C.c_int32), ("gicp_iterations", C.c_int32),
                ("bfgs_evaluations", C.c_int32), ("pad", C.c_int32), ("ndt_score", C.c_double),
                ("gicp_fitness", C.c_double)]


_lib = None


def build():
    subprocess.check_call(["make", "-C", _DIR, "-s"])


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
        _lib.sm_oracle_calculate_normals.restype = C.c_int64
        _lib.sm_oracle_calculate_normals.argtypes = [dp, dp, C.c_int64, C.c_int]
        _lib.sm_oracle_knn1.argtypes = [dp, C.c_int64, dp, C.c_int64, C.c_double, C.c_int,
                                        C.c_int, ip, dp]
        _lib.sm_oracle_knn1_brute.argtypes = [dp, C.c_int64, dp, C.c_int64, ip, dp]
        _lib.sm_oracle_icp_fast_align.argtypes = [
            dp, C.c_int64, dp, dp, C.c_int64, dp, C.POINTER(IcpOptions), dp, dp, ip,
            C.POINTER(IcpTrace), C.c_int32]
        _lib.sm_oracle_solve6.argtypes = [dp, dp, dp, C.POINTER(C.c_int)]
        _lib.sm_oracle_quantile_index.argtypes = [C.c_int64, C.c_float]
        _lib.sm_oracle_check_convergence_inputs.argtypes = [dp, C.c_int, C.POINTER(C.c_int)]
        fp, i64 = C.POINTER(C.c_float), C.c_int64
        _lib.sm_oracle_ndt_voxels.restype = C.c_int64
        _lib.sm_oracle_ndt_voxels.argtypes = [fp, i64, C.c_float, i64, ip, ip, dp, dp, fp, ip]
        _lib.sm_oracle_ndt_derivatives.argtypes = [fp, i64, fp, i64, C.POINTER(NdtOptions), dp, dp, dp, dp, dp]
        _lib.sm_oracle_ndt_derivatives_f64.argtypes = [fp, i64, fp, i64, C.POINTER(NdtOptions), dp, dp, dp, dp, dp]
        _lib.sm_oracle_ndt_align.argtypes = [fp, i64, fp, i64, dp, C.POINTER(NdtOptions), dp, dp, ip, dp, dp]
        _lib.sm_oracle_approx_voxel_grid.restype = C.c_int64
        _lib.sm_oracle_approx_voxel_grid.argtypes = [fp, i64, C.c_float, fp, i64]
        _lib.sm_oracle_gicp_covariances.argtypes = [fp, i64, C.c_int, C.c_double, dp]
        _lib.sm_oracle_ndt_gicp_align.argtypes = [fp, i64, fp, i64, dp, C.POINTER(NdtGicpOptions), dp, dp,
                                                  C.POINTER(NdtGicpInfo)]
        _lib.sm_oracle_gicp_cost.restype = C.c_int64
        _lib.sm_oracle_gicp_cost.argtypes = [fp, i64, fp, i64, fp, fp, dp, dp, dp, dp, ip, ip]
    return _lib


def approx_voxel_grid(points, leaf=0.2):
    p = _fcloud(points)
    out = np.zeros_like(p)
    m = lib().sm_oracle_approx_voxel_grid(_f(p), p.shape[0], leaf, _f(out), p.shape[0])
    return out[:m].copy()


def gicp_covariances(points, k=20, eps=1e-3):
    p = _fcloud(points)
    cov = np.zeros((p.shape[0], 9))
    lib().sm_oracle_gicp_covariances(_f(p), p.shape[0], k, eps, _d(cov))
    return cov.reshape(-1, 3, 3)


def gicp_cost(source, target, guess, transformation, x):
    """GICP correspondence step for (guess, transformation_) and one cost / gradient evaluation at state x
    (test hook sm_oracle_gicp_cost) -> dict(f, g, maha (ns,3,3), si, ti)."""
    s, t = _fcloud(source), _fcloud(target)
    g_cm = np.ascontiguousarray(np.asarray(guess, dtype=np.float32).T).ravel()
    t_cm = np.ascontiguousarray(np.asarray(transformation, dtype=np.float32).T).ravel()
    xx = np.ascontiguousarray(np.asarray(x, dtype=np.float64))
    f = C.c_double(); g = np.zeros(6); maha = np.zeros((s.shape[0], 9))
    si = np.zeros(s.shape[0], np.int32); ti = np.zeros(s.shape[0], np.int32)
    m = lib().sm_oracle_gicp_cost(_f(s), s.shape[0], _f(t), t.shape[0], _f(g_cm), _f(t_cm), _d(xx), C.byref(f), _d(g),
                                  _d(maha), _i(si), _i(ti))
    return {"f": f.value, "g": g, "maha": maha.reshape(-1, 3, 3), "si": si[:m].copy(), "ti": ti[:m].copy()}


def ndt_gicp_align(source, target, guess=None, voxel_resolution=0.2, using_voxel_filter=True, use_ndt=True):
    s, t = _fcloud(source), _fcloud(target)
    g = np.eye(4) if guess is None else np.asarray(guess, dtype=np.float64)
    g_cm = np.ascontiguousarray(g.T).ravel()
    opt = NdtGicpOptions(voxel_resolution, int(using_voxel_filter), int(use_ndt))
    res = np.zeros(16); sc = C.c_double(); info = NdtGicpInfo()
    rc = lib().sm_oracle_ndt_gicp_align(_f(s), s.shape[0], _f(t), t.shape[0], _d(g_cm), C.byref(opt), _d(res),
                                        C.byref(sc), C.byref(info))
    out = {"rc": rc, "result": res.reshape(4, 4).T.copy(), "score": sc.value}
    out.update({k: getattr(info, k) for k, _ in NdtGicpInfo._fields_ if k != "pad"})
    return out


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _fcloud(a):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
    assert a.ndim == 2 and a.shape[1] == 3
    return a


def ndt_options(**kw):
    o = NdtOptions(1.0, 0.1, 0.55, 0.1, 35)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def ndt_voxels(target, resolution=1.0):
    t = _fcloud(target)
    cap = t.shape[0]
    idx = np.zeros(cap, np.int32); npts = np.zeros(cap, np.int32); srch = np.zeros(cap, np.int32)
    mean = np.zeros((cap, 3)); icov = np.zeros((cap, 9)); cen = np.zeros((cap, 3), np.float32)
    k = lib().sm_oracle_ndt_voxels(_f(t), t.shape[0], resolution, cap, _i(idx), _i(npts), _d(mean), _d(icov),
                                   _f(cen), _i(srch))
    if k < 0:
        raise OverflowError("NDT grid: more than INT32_MAX voxels in the target's bounding box")
    return {"idx": idx[:k], "n": npts[:k], "mean": mean[:k], "icov": icov[:k].reshape(-1, 3, 3),
            "centroid": cen[:k], "searchable": srch[:k]}


def ndt_derivatives(source, target, p, f64=False, **opts):
    """computeDerivatives at pose vector p -> (score, g[6], H (6,6), mean neighbours per point); f64 = True: the
    stock-PCL double term math of NdtWithGicp."""
    s, t = _fcloud(source), _fcloud(target)
    o = ndt_options(**opts)
    pp = np.ascontiguousarray(np.asarray(p, dtype=np.float64))
    score = C.c_double(); nb = C.c_double()
    g = np.zeros(6); H = np.zeros(36)
    fn = lib().sm_oracle_ndt_derivatives_f64 if f64 else lib().sm_oracle_ndt_derivatives
    rc = fn(_f(s), s.shape[0], _f(t), t.shape[0], C.byref(o), _d(pp), C.byref(score), _d(g), _d(H), C.byref(nb))
    if rc < 0:
        raise OverflowError("NDT grid: more than INT32_MAX voxels in the target's bounding box")
    return score.value, g, H.reshape(6, 6), nb.value


def ndt_align(source, target, guess=None, **opts):
    s, t = _fcloud(source), _fcloud(target)
    o = ndt_options(**opts)
    g = np.eye(4) if guess is None else np.asarray(guess, dtype=np.float64)
    g_cm = np.ascontiguousarray(g.T).ravel()
    res = np.zeros(16); fit = C.c_double(); it = C.c_int32(); tp = C.c_double(); nb = C.c_double()
    rc = lib().sm_oracle_ndt_align(_f(s), s.shape[0], _f(t), t.shape[0], _d(g_cm), C.byref(o), _d(res),
                                   C.byref(fit), C.byref(it), C.byref(tp), C.byref(nb))
    return {"rc": rc, "result": res.reshape(4, 4).T.copy(), "fitness": fit.value, "iterations": it.value,
            "trans_probability": tp.value, "mean_neighbors": nb.value}


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _i(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _cloud(a):
    """(N,3) array-like -> C-contiguous (N,3) float64 == 3xN column-major."""
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float64))
    assert a.ndim == 2 and a.shape[1] == 3
    return a


def calculate_normals(points, tie_mode=0):
    """EigenPointCloud::CalculateNormals -> (points_kept (M,3), normals (M,3))."""
    p = _cloud(points).copy()
    n = np.zeros_like(p)
    m = lib().sm_oracle_calculate_normals(_d(p), _d(n), p.shape[0], tie_mode)
    return p[:m].copy(), n[:m].copy()


def knn1(target, query, epsilon=3.16, bucket_size=8, tie_mode=0):
    t, q = _cloud(target), _cloud(query)
    ids = np.empty(q.shape[0], dtype=np.int32)
    d2 = np.empty(q.shape[0], dtype=np.float64)
    rc = lib().sm_oracle_knn1(_d(t), t.shape[0], _d(q), q.shape[0], epsilon, bucket_size,
                              tie_mode, _i(ids), _d(d2))
    assert rc == 0
    return ids, d2


def knn1_brute(target, query):
    t, q = _cloud(target), _cloud(query)
    ids = np.empty(q.shape[0], dtype=np.int32)
    d2 = np.empty(q.shape[0], dtype=np.float64)
    lib().sm_oracle_knn1_brute(_d(t), t.shape[0], _d(q), q.shape[0], _i(ids), _d(d2))
    return ids, d2


def icp_fast_align(source, target, target_normals, guess=None, max_iteration=100,
                   dist_outlier_ratio=0.7, knn_epsilon=3.16, disable_convergence_check=False,
                   tie_mode=0, trace=False):
    """IcpFast::Align.  Returns dict(result 4x4, score, iterations, rc[, trace])."""
    s, t, n = _cloud(source), _cloud(target), _cloud(target_normals)
    g = np.eye(4) if guess is None else np.asarray(guess, dtype=np.float64)
    g_cm = np.ascontiguousarray(g.T).ravel()  # column-major
    opt = IcpOptions(max_iteration, dist_outlier_ratio, knn_epsilon,
                     int(disable_convergence_check), tie_mode)
    res = np.zeros(16)
    score = C.c_double(0.0)
    iters = C.c_int32(0)
    cap = max_iteration if trace else 0
    tr = (IcpTrace * max(cap, 1))()
    rc = lib().sm_oracle_icp_fast_align(_d(s), s.shape[0], _d(t), _d(n), t.shape[0], _d(g_cm),
                                        C.byref(opt), _d(res), C.byref(score), C.byref(iters),
                                        tr, cap)
    out = {"rc": rc, "result": res.reshape(4, 4).T.copy(), "score": score.value,
           "iterations": iters.value}
    if trace:
        out["trace"] = [
            {"T_iter": np.array(tr[i].T_iter).reshape(4, 4).T.copy(), "limit": tr[i].limit,
             "kept": tr[i].kept, "A": np.array(tr[i].A).reshape(6, 6),
             "b": np.array(tr[i].b)} for i in range(iters.value)]
    return out


def solve6(A, b):
    A = np.asarray(A, dtype=np.float64)
    a_cm = np.ascontiguousarray(A.T).ravel()
    bb = np.ascontiguousarray(np.asarray(b, dtype=np.float64))
    x = np.zeros(6)
    path = C.c_int(-1)
    lib().sm_oracle_solve6(_d(a_cm), _d(bb), _d(x), C.byref(path))
    return x, path.value


def quantile_index(n, ratio=0.7):
    return lib().sm_oracle_quantile_index(n, ratio)


def num_threads():
    return lib().sm_oracle_num_threads()


def set_num_threads(n):
    lib().sm_oracle_set_num_threads(int(n))


# ---- motion compensation either side of Align (oracle/motion_oracle.cc) -------------------------
def interpolate_transform(t1, t2, factor):
    a = np.ascontiguousarray(np.asarray(t1, dtype=np.float64).T).ravel()
    b = np.ascontiguousarray(np.asarray(t2, dtype=np.float64).T).ravel()
    out = np.zeros(16)
    f = lib().sm_oracle_interpolate_transform
    f.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_float, C.POINTER(C.c_double)]
    rc = f(_d(a), _d(b), float(factor), _d(out))
    return rc, out.reshape(4, 4).T.copy()


def motion_compensation(points5, delta):
    p = np.ascontiguousarray(np.asarray(points5, dtype=np.float32))
    assert p.ndim == 2 and p.shape[1] == 5
    d = np.ascontiguousarray(np.asarray(delta, dtype=np.float64).T).ravel()
    out = np.zeros_like(p)
    f = lib().sm_oracle_motion_compensation
    f.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_double), C.c_void_p]
    rc = f(p.ctypes.data, p.shape[0], _d(d), out.ctypes.data)
    return rc, out


def average_transforms(transforms):
    ts = np.ascontiguousarray(np.stack([np.asarray(t, dtype=np.float64).T.ravel() for t in transforms]))
    out = np.zeros(16)
    f = lib().sm_oracle_average_transforms
    f.argtypes = [C.POINTER(C.c_double), C.c_int32, C.POINTER(C.c_double)]
    rc = f(_d(ts.ravel()), len(transforms), _d(out))
    return rc, out.reshape(4, 4).T.copy()


# ---- IcpUsingPointMatcher stand-in (type 1): composition of the pieces above ---------------------
def pm_keep_mask(n, prob=0.9, seed=1):
    """The engine's reading filter: counter hash of the point index (murmur3 finaliser) below
    prob * 2^32 (staticmapping_b200/csrc/icp_pm.cu pm_keep)."""
    p = float(np.float32(prob))
    if p >= 1.0:
        return np.ones(n, dtype=bool)
    thresh = np.uint32(0) if p <= 0.0 else np.uint32(int(p * 4294967296.0))
    with np.errstate(over="ignore"):
        x = np.arange(n, dtype=np.uint32) * np.uint32(0x9E3779B9) + np.uint32(seed)
        x ^= x >> np.uint32(16)
        x *= np.uint32(0x85EBCA6B)
        x ^= x >> np.uint32(13)
        x *= np.uint32(0xC2B2AE35)
        x ^= x >> np.uint32(16)
    return x < thresh


def icp_pm_equivalent(source_f32, target_f32, guess=None, prob=0.9, seed=1, max_iteration=150,
                      accept_min_score=0.6):
    """Reference-side chain of icp_pointmatcher.cc:166-247 restated with the oracle's pieces:
    CalculateNormals on the target (SamplingSurfaceNormal knn 7), hash subsample of the reading,
    IcpFast::Align capped at 150 iterations, Align() false below score 0.6."""
    src = np.asarray(source_f32, dtype=np.float32)
    tgt = np.asarray(target_f32, dtype=np.float32)
    tp, tn = calculate_normals(tgt.astype(np.float64))
    keep = pm_keep_mask(src.shape[0], prob, seed)
    o = icp_fast_align(src[keep].astype(np.float64), tp, tn, guess, max_iteration=max_iteration)
    o["icp_fast_score"] = o["score"]
    o["n_source"] = int(keep.sum())
    o["n_target"] = int(tp.shape[0])
    # "compute the final score" (icp_pointmatcher.cc:131-148): UNFILTERED reading moved by the result,
    # matched against the UNFILTERED reference (same matcher, eps 3.16), trimmed at 0.7
    _, d2 = knn1(tgt.astype(np.float64), pm_moved(src, o["result"]), epsilon=3.16)
    v, _, kept = pm_score_trim(d2)
    if kept:
        o["score"] = float(np.exp(-(np.sqrt(v[:kept]).sum() / kept)))
        o["score_kept"] = kept
    o["ok"] = o["score"] >= float(np.float32(accept_min_score))
    return o


def pm_moved(source_f32, R):
    """The reading cloud (float) moved by the 4x4 R in double, in the engine's (and cloud_types.cc:288-296)
    accumulation order: ((R00 x + R01 y) + R02 z) + R03 per row."""
    s64 = np.asarray(source_f32, dtype=np.float32).astype(np.float64)
    moved = np.empty_like(s64)
    for r in range(3):
        moved[:, r] = ((R[r, 0] * s64[:, 0] + R[r, 1] * s64[:, 1]) + R[r, 2] * s64[:, 2]) + R[r, 3]
    return moved


def pm_score_trim(d2, ratio=0.7):
    """The score pass's trim (GetDistsQuantile, icp_fast.cc:82-89): over the finite squared distances, the limit is
    element int(valid * ratio) of the sorted values, or the last one when ratio is 1 or that index is past the end,
    and every value <= limit is kept.  Returns (sorted finite values, valid, kept); kept values are the first `kept`."""
    v = np.sort(np.asarray(d2, dtype=np.float64)[np.isfinite(d2)])
    if not v.size:
        return v, 0, 0
    q = float(np.float32(ratio))
    qi = v.size - 1 if q == 1.0 else min(int(v.size * q), v.size - 1)
    return v, int(v.size), int(np.count_nonzero(v <= v[qi]))


def pm_score_block_sum(values, threads=1024):
    """The sum of `values` in the order the score pass adds them (one block of `threads` threads, reduce.cuh
    block_sum): thread t adds values[i] for i = t (mod threads) in ascending i from 0.0, each warp of 32 adds with an
    xor butterfly (offsets 16, 8, 4, 2, 1), and the warp totals are added in warp order from 0.0."""
    v = np.asarray(values, dtype=np.float64)
    rows = -(-v.size // threads)
    grid = np.zeros(rows * threads)
    grid[:v.size] = v
    acc = np.zeros(threads)
    for row in grid.reshape(rows, threads):   # adding the zero padding leaves every partial sum unchanged
        acc = acc + row
    lanes = acc.reshape(threads // 32, 32)
    idx = np.arange(32)
    for off in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, idx ^ off]
    total = 0.0
    for w in lanes[:, 0]:
        total += float(w)
    return total


def voxel_grid_filter(points5, voxel_size, order_mode=0):
    """pre_processers::filter::VoxelGrid::Filter; order_mode 1 = the reference's literal
    unordered_map iteration order."""
    p = np.ascontiguousarray(np.asarray(points5, dtype=np.float32))
    assert p.ndim == 2 and p.shape[1] == 5
    out = np.zeros_like(p)
    f = lib().sm_oracle_voxel_grid_filter
    f.restype = C.c_int64
    f.argtypes = [C.c_void_p, C.c_int64, C.c_float, C.c_int, C.c_void_p]
    m = f(p.ctypes.data, p.shape[0], float(voxel_size), int(order_mode), out.ctypes.data)
    return m, out[:max(m, 0)].copy()


# ---- M2DP descriptor (oracle/m2dp_oracle.cc) --------------------------------------------------------
def m2dp(points, r=0.1, max_distance=100.0, t=16, p=4, q=16, with_matrix=False):
    """descriptor::M2dp::setInputCloud + getFinalDescriptor.  Returns the descriptor (p*q + l*t floats),
    or (descriptor, A counts (p*q, l*t), mean+axes (12,)) with with_matrix."""
    pts = _fcloud(points)
    L = lib()
    L.sm_oracle_m2dp_dims.restype = C.c_int64
    L.sm_oracle_m2dp_dims.argtypes = [C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
    l = C.c_int32(0)
    n = L.sm_oracle_m2dp_dims(r, max_distance, t, p, q, C.byref(l))
    if n < 0:
        raise ValueError("r is too small")
    desc = np.zeros(n, np.float32)
    A = np.zeros((p * q, l.value * t), np.int32)
    axes = np.zeros(12, np.float32)
    L.sm_oracle_m2dp.restype = C.c_int64
    L.sm_oracle_m2dp.argtypes = [C.c_void_p, C.c_int64, C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_void_p]
    got = L.sm_oracle_m2dp(pts.ctypes.data, pts.shape[0], r, max_distance, t, p, q, desc.ctypes.data, A.ctypes.data,
                           axes.ctypes.data)
    if got == 0:
        return (None, None, None) if with_matrix else None
    return (desc, A, axes) if with_matrix else desc


def m2dp_match(P, Q):
    P = np.ascontiguousarray(P, np.float32); Q = np.ascontiguousarray(Q, np.float32)
    if P.shape != Q.shape:
        return -1.0
    L = lib()
    L.sm_oracle_m2dp_match.restype = C.c_double
    L.sm_oracle_m2dp_match.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    return L.sm_oracle_m2dp_match(P.ctypes.data, Q.ctypes.data, P.shape[0])
