"""ctypes binding of tests/cpp/icp_compensation_oracle.cc: IcpFast::Align with EnableInnerCompensation, restated
on the CPU over libsm_oracle.so's pieces.  TEST INFRASTRUCTURE.  The library is compiled on first use into a
per-user temporary directory (keyed by the source's hash), so a read-only tree works."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

import oracle_lib as O

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "tests", "cpp", "icp_compensation_oracle.cc")
_ORACLE_DIR = os.path.join(_ROOT, "oracle")
_lib = None


def lib():
    global _lib
    if _lib is None:
        O.lib()                                          # builds libsm_oracle.so if needed; loaded first
        with open(_SRC, "rb") as f:
            tag = hashlib.sha256(f.read() + _ORACLE_DIR.encode()).hexdigest()[:16]   # the rpath is part of it
        out_dir = os.path.join(tempfile.gettempdir(), f"sm_icp_comp_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        so = os.path.join(out_dir, f"libsm_icp_comp_oracle_{tag}.so")
        if not os.path.exists(so):
            cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
            tmp = so + f".{os.getpid()}.tmp"
            # the flags of oracle/Makefile: no FMA contraction, so the arithmetic is the written one
            subprocess.check_call([cxx, "-O2", "-fopenmp", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared",
                                   "-I", _ORACLE_DIR, _SRC, "-o", tmp, "-L", _ORACLE_DIR, "-l:libsm_oracle.so",
                                   "-Wl,-rpath," + _ORACLE_DIR])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
        dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
        _lib.sm_oracle_icp_fast_align_compensated.argtypes = [
            dp, C.c_int64, dp, dp, C.c_int64, dp, C.POINTER(O.IcpOptions), C.c_int32, dp, dp, ip,
            C.POINTER(O.IcpTrace), C.c_int32]
    return _lib


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def icp_fast_align(source, target, target_normals, guess=None, inner_compensation=True, max_iteration=100,
                   dist_outlier_ratio=0.7, knn_epsilon=3.16, disable_convergence_check=False, tie_mode=0,
                   trace=False):
    """IcpFast::Align with the inner-compensation flag; the output of oracle_lib.icp_fast_align."""
    s, t, n = (np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, 3)) for a in
               (source, target, target_normals))
    g = np.eye(4) if guess is None else np.asarray(guess, dtype=np.float64)
    g_cm = np.ascontiguousarray(g.T).ravel()
    opt = O.IcpOptions(max_iteration, dist_outlier_ratio, knn_epsilon, int(disable_convergence_check), tie_mode)
    res = np.zeros(16)
    score = C.c_double(0.0)
    iters = C.c_int32(0)
    cap = max_iteration if trace else 0
    tr = (O.IcpTrace * max(cap, 1))()
    rc = lib().sm_oracle_icp_fast_align_compensated(
        _d(s), s.shape[0], _d(t), _d(n), t.shape[0], _d(g_cm), C.byref(opt), int(bool(inner_compensation)),
        _d(res), C.byref(score), C.byref(iters), tr, cap)
    out = {"rc": rc, "result": res.reshape(4, 4).T.copy(), "score": score.value, "iterations": iters.value}
    if trace:
        out["trace"] = [
            {"T_iter": np.array(tr[i].T_iter).reshape(4, 4).T.copy(), "limit": tr[i].limit,
             "kept": tr[i].kept, "A": np.array(tr[i].A).reshape(6, 6),
             "b": np.array(tr[i].b)} for i in range(iters.value)]
    return out
