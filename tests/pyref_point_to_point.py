"""Second, independent restatement of IcpFast::Align with the point-to-point minimizer, in numpy, written from the
reference sources (registrators/icp_fast.cc:455-529 with ComputePointToPoint, :326-375, at :506-510).  It reuses
the plain restatement's pieces (tests/pyref.py) and numpy's SVD (LAPACK), not the product's."""
from __future__ import annotations

import math

import numpy as np

import pyref
import pyref_compensation
from pyref import INF


def compute_point_to_point(P, Q):
    """ComputePointToPoint (icp_fast.cc:326-375), all weights 1: centre both sets on their means, M = Qc^T Pc
    (target x source^T), R = U V^T from numpy's SVD with the last row of V^T negated when det R < 0,
    t = qbar - R pbar.  Returns the 4x4 and whether the reflection fix ran."""
    pbar, qbar = P.mean(axis=0), Q.mean(axis=0)
    M = (Q - qbar).T @ (P - pbar)
    U, _, Vt = np.linalg.svd(M)
    R = U @ Vt
    fix = bool(np.linalg.det(R) < 0.0)
    if fix:
        Vt = Vt.copy()
        Vt[2] *= -1.0
        R = U @ Vt
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = qbar - R @ pbar
    return T, fix


def kabsch_objective(R, P, Q):
    """The point-to-point cost at rotation R with its optimal translation: sum |(q - qbar) - R (p - pbar)|^2."""
    Pc, Qc = P - P.mean(axis=0), Q - Q.mean(axis=0)
    return float(((Qc - Pc @ R.T) ** 2).sum())


def icp_fast_align(source, target, knn, guess=None, inner_compensation=False, max_iteration=100,
                   dist_outlier_ratio=0.7, disable_convergence_check=False, trace=None):
    """IcpFast::Align with the point-to-point minimizer.  knn(target_centred, P) -> (ids, d2)."""
    S = np.asarray(source, dtype=np.float64)
    Qt = np.asarray(target, dtype=np.float64).copy()
    guess = np.eye(4) if guess is None else np.asarray(guess, dtype=np.float64)
    target_mean = Qt.sum(axis=0) / Qt.shape[0]
    T_mean = np.eye(4); T_mean[:3, 3] = target_mean
    Qt -= target_mean
    G0 = np.linalg.inv(T_mean) @ guess
    S0 = pyref._apply_transform(G0, S)
    T_iter = np.eye(4)
    rotations, translations = [np.array([1.0, 0.0, 0.0, 0.0])], [np.zeros(3)]
    it = 0
    while True:
        P = pyref_compensation.motion_compensation(T_iter, S0) if inner_compensation else pyref._apply_transform(T_iter, S0)
        ids, d2 = knn(Qt, P)
        limit = pyref._quantile_limit(d2, dist_outlier_ratio)
        keep = np.nonzero((d2 != INF) & (d2 <= limit))[0]
        assert keep.size > 0
        dT, fix = compute_point_to_point(P[keep], Qt[ids[keep]])
        T_iter = dT @ T_iter
        it += 1
        rotations.append(pyref._quat_from_matrix(T_iter[:3, :3]))
        translations.append(T_iter[:3, 3].copy())
        if trace is not None:
            trace.append({"limit": limit, "kept": int(keep.size), "T_iter": T_iter.copy(), "fix": fix})
        conv = (not disable_convergence_check) and pyref._check_convergence(rotations, translations)
        if conv or it >= max_iteration:
            score = math.exp(-float(np.sqrt(d2[keep]).sum()) / keep.size)
            break
    return {"result": T_mean @ T_iter @ G0, "iterations": it, "score": score, "kept": int(keep.size)}
