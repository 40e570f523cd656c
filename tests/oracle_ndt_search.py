"""ctypes binding of tests/cpp/ndt_search_oracle.cc: registrator::Ndt with each of pclomp's neighbour searches
(KDTREE, DIRECT26, DIRECT7, DIRECT1), restated on the CPU over libsm_oracle.so's pieces.  TEST INFRASTRUCTURE.  The
library is compiled on first use into a per-user temporary directory (keyed by the source's hash), so a read-only
tree works."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

import oracle_lib as O

KDTREE, DIRECT26, DIRECT7, DIRECT1 = 0, 1, 2, 3
METHODS = (KDTREE, DIRECT26, DIRECT7, DIRECT1)

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "tests", "cpp", "ndt_search_oracle.cc")
_ORACLE_DIR = os.path.join(_ROOT, "oracle")
_lib = None


def lib():
    global _lib
    if _lib is None:
        O.lib()                                          # builds libsm_oracle.so if needed; loaded first
        h = hashlib.sha256()
        for path in (_SRC, os.path.join(_ORACLE_DIR, "ndt_math.h"), os.path.join(_ORACLE_DIR, "linalg.h")):
            with open(path, "rb") as f:
                h.update(f.read())
        tag = hashlib.sha256(h.digest() + _ORACLE_DIR.encode()).hexdigest()[:16]   # the rpath is part of it
        out_dir = os.path.join(tempfile.gettempdir(), f"sm_ndt_search_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        so = os.path.join(out_dir, f"libsm_ndt_search_oracle_{tag}.so")
        if not os.path.exists(so):
            cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
            tmp = so + f".{os.getpid()}.tmp"
            # the flags of oracle/Makefile: no FMA contraction, so the arithmetic is the written one
            subprocess.check_call([cxx, "-O2", "-fopenmp", "-fPIC", "-std=c++17", "-ffp-contract=off", "-shared",
                                   "-I", _ORACLE_DIR, _SRC, "-o", tmp, "-L", _ORACLE_DIR, "-l:libsm_oracle.so",
                                   "-Wl,-rpath," + _ORACLE_DIR])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
        fp, dp, ip, i64 = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int32), C.c_int64
        _lib.sm_oracle_ndt_search_neighbors.argtypes = [fp, i64, C.c_float, C.c_int32, fp, i64, ip, ip]
        _lib.sm_oracle_ndt_search_derivatives.argtypes = [fp, i64, fp, i64, C.POINTER(O.NdtOptions), C.c_int32, dp,
                                                          dp, dp, dp, dp]
        _lib.sm_oracle_ndt_search_align.argtypes = [fp, i64, fp, i64, dp, C.POINTER(O.NdtOptions), C.c_int32, dp, dp,
                                                    ip, ip, dp, dp]
    return _lib


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _i(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def neighbors(target, points, method, resolution=1.0):
    """-> list of int arrays: per point, the neighbour leaf indices in the order computeDerivatives uses them."""
    t, p = O._fcloud(target), O._fcloud(points)
    counts = np.zeros(p.shape[0], np.int32)
    keys = np.zeros((p.shape[0], 27), np.int32)
    rc = lib().sm_oracle_ndt_search_neighbors(_f(t), t.shape[0], resolution, method, _f(p), p.shape[0], _i(counts),
                                              _i(keys))
    if rc < 0:
        raise OverflowError("NDT grid: more than INT32_MAX voxels in the target's bounding box")
    return [keys[i, :counts[i]].copy() for i in range(p.shape[0])]


def ndt_derivatives(source, target, p, method, **opts):
    """computeDerivatives at pose vector p -> (score, g[6], H (6,6), mean neighbours per point)."""
    s, t = O._fcloud(source), O._fcloud(target)
    o = O.ndt_options(**opts)
    pp = np.ascontiguousarray(np.asarray(p, dtype=np.float64))
    score = C.c_double(); nb = C.c_double()
    g = np.zeros(6); H = np.zeros(36)
    rc = lib().sm_oracle_ndt_search_derivatives(_f(s), s.shape[0], _f(t), t.shape[0], C.byref(o), method, _d(pp),
                                                C.byref(score), _d(g), _d(H), C.byref(nb))
    if rc < 0:
        raise OverflowError("NDT grid: more than INT32_MAX voxels in the target's bounding box")
    return score.value, g, H.reshape(6, 6), nb.value


def ndt_align(source, target, method, guess=None, **opts):
    """Ndt::Align with the method: the output of oracle_lib.ndt_align plus the evaluation count."""
    s, t = O._fcloud(source), O._fcloud(target)
    o = O.ndt_options(**opts)
    g = np.eye(4) if guess is None else np.asarray(guess, dtype=np.float64)
    g_cm = np.ascontiguousarray(g.T).ravel()
    res = np.zeros(16); fit = C.c_double(); it = C.c_int32(); ev = C.c_int32(); tp = C.c_double(); nb = C.c_double()
    rc = lib().sm_oracle_ndt_search_align(_f(s), s.shape[0], _f(t), t.shape[0], _d(g_cm), C.byref(o), method, _d(res),
                                          C.byref(fit), C.byref(it), C.byref(ev), C.byref(tp), C.byref(nb))
    return {"rc": rc, "result": res.reshape(4, 4).T.copy(), "fitness": fit.value, "iterations": it.value,
            "evaluations": ev.value, "trans_probability": tp.value, "mean_neighbors": nb.value}
