"""ctypes binding of oracle/icp_point_to_point_oracle.cc: IcpFast::Align with the point-to-point minimizer
(ComputePointToPoint, icp_fast.cc:326-375), restated on the CPU over libsm_oracle.so's pieces.  TEST
INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O

_lib = None


class P2PTrace(C.Structure):
    _fields_ = [("T_iter", C.c_double * 16), ("limit", C.c_double), ("kept", C.c_int64),
                ("pbar", C.c_double * 3), ("qbar", C.c_double * 3), ("M", C.c_double * 9),
                ("R", C.c_double * 9), ("t", C.c_double * 3), ("path", C.c_int32), ("pad", C.c_int32)]


def lib():
    global _lib
    if _lib is None:
        _lib = O.lib()
        dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
        _lib.sm_oracle_icp_fast_align_point_to_point.argtypes = [
            dp, C.c_int64, dp, C.c_int64, dp, C.POINTER(O.IcpOptions), C.c_int32, dp, dp, ip,
            C.POINTER(P2PTrace), C.c_int32]
        _lib.sm_oracle_point_to_point.argtypes = [dp, dp, C.c_int64, dp, dp, dp, dp, dp]
    return _lib


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def point_to_point(P, Q):
    """ComputePointToPoint over kept pairs P (reading) / Q (reference), (n, 3) each: pbar, qbar, M, R, t, path."""
    P, Q = (np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, 3)) for a in (P, Q))
    pbar, qbar, t = np.zeros(3), np.zeros(3), np.zeros(3)
    M, R = np.zeros(9), np.zeros(9)
    path = lib().sm_oracle_point_to_point(_d(P), _d(Q), P.shape[0], _d(pbar), _d(qbar), _d(M), _d(R), _d(t))
    return {"pbar": pbar, "qbar": qbar, "M": M.reshape(3, 3), "R": R.reshape(3, 3), "t": t, "path": path}


def icp_fast_align(source, target, guess=None, inner_compensation=False, max_iteration=100, dist_outlier_ratio=0.7,
                   knn_epsilon=3.16, disable_convergence_check=False, tie_mode=0, trace=False):
    """IcpFast::Align with the point-to-point minimizer; the output of oracle_lib.icp_fast_align (the target's normals
    are not read, so none are passed)."""
    s, t = (np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, 3)) for a in (source, target))
    g = np.eye(4) if guess is None else np.asarray(guess, dtype=np.float64)
    g_cm = np.ascontiguousarray(g.T).ravel()
    opt = O.IcpOptions(max_iteration, dist_outlier_ratio, knn_epsilon, int(disable_convergence_check), tie_mode)
    res = np.zeros(16)
    score = C.c_double(0.0)
    iters = C.c_int32(0)
    cap = max_iteration if trace else 0
    tr = (P2PTrace * max(cap, 1))()
    rc = lib().sm_oracle_icp_fast_align_point_to_point(
        _d(s), s.shape[0], _d(t), t.shape[0], _d(g_cm), C.byref(opt), int(bool(inner_compensation)),
        _d(res), C.byref(score), C.byref(iters), tr, cap)
    out = {"rc": rc, "result": res.reshape(4, 4).T.copy(), "score": score.value, "iterations": iters.value}
    if trace:
        out["trace"] = [
            {"T_iter": np.array(tr[i].T_iter).reshape(4, 4).T.copy(), "limit": tr[i].limit, "kept": tr[i].kept,
             "pbar": np.array(tr[i].pbar), "qbar": np.array(tr[i].qbar), "M": np.array(tr[i].M).reshape(3, 3),
             "R": np.array(tr[i].R).reshape(3, 3), "t": np.array(tr[i].t), "path": tr[i].path}
            for i in range(min(iters.value, cap))]
    return out


def icp_pm_equivalent(source_f32, target_f32, guess=None, prob=0.9, seed=1, max_iteration=150, accept_min_score=0.6):
    """oracle_lib.icp_pm_equivalent (the IcpUsingPointMatcher stand-in's chain) with the point-to-point minimizer."""
    src = np.asarray(source_f32, dtype=np.float32)
    tgt = np.asarray(target_f32, dtype=np.float32)
    tp, _ = O.calculate_normals(tgt.astype(np.float64))
    keep = O.pm_keep_mask(src.shape[0], prob, seed)
    o = icp_fast_align(src[keep].astype(np.float64), tp, guess, max_iteration=max_iteration)
    o["icp_fast_score"] = o["score"]
    _, d2 = O.knn1(tgt.astype(np.float64), O.pm_moved(src, o["result"]), epsilon=3.16)
    v, _, kept = O.pm_score_trim(d2)
    if kept:
        o["score"] = float(np.exp(-(np.sqrt(v[:kept]).sum() / kept)))
    o["ok"] = o["score"] >= float(np.float32(accept_min_score))
    return o
