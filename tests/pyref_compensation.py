"""Second, independent restatement of IcpFast::Align with Interface::EnableInnerCompensation, in numpy, written from
the reference sources (registrators/icp_fast.cc:455-529 with :487-491, :506-510, :284-289; builder/data/cloud_types.cc
:306-318, :340-344; common/math.h:198-211).  It reuses the plain restatement's pieces (tests/pyref.py) and differs
from it in two steps only: the per-point de-skew and the factor-scaled Jacobian."""
from __future__ import annotations

import math

import numpy as np

import pyref
from pyref import INF


def motion_compensation(T, P):
    """EigenPointCloud::ApplyMotionCompensation(T) (cloud_types.cc:306-318, interpolating towards the parameter T:
    the reference's local shadows it and is read uninitialised) with factors[i] = i / N (:340-344): point i moves by
    common::InterpolateTransform(Identity, T, float(f_i)), i.e. Eigen 3.3's slerp from the identity quaternion plus
    a linear translation, then R * p + t in Eigen's order."""
    n = P.shape[0]
    t = np.arange(n, dtype=np.float64) / np.float64(n)
    t = t.astype(np.float32).astype(np.float64)                     # InterpolateTransform takes a float
    qa, qb = np.array([1.0, 0.0, 0.0, 0.0]), pyref._quat_from_matrix(T[:3, :3])
    d = float(qa[1] * qb[1] + qa[2] * qb[2] + qa[3] * qb[3] + qa[0] * qb[0])
    if abs(d) >= 1.0 - 2.220446049250313e-16:
        s0, s1 = 1.0 - t, t
    else:
        theta = math.acos(abs(d))
        s0, s1 = np.sin((1.0 - t) * theta) / math.sin(theta), np.sin(t * theta) / math.sin(theta)
    if d < 0.0:
        s1 = -s1
    w, x, y, z = (s0 * qa[k] + s1 * qb[k] for k in range(4))
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z                           # QuaternionBase::toRotationMatrix
    R = [[1.0 - (ty * y + tz * z), ty * x - tz * w, tz * x + ty * w],
         [ty * x + tz * w, 1.0 - (tx * x + tz * z), tz * y - tx * w],
         [tz * x - ty * w, tz * y + tx * w, 1.0 - (tx * x + ty * y)]]
    return np.stack([((R[r][0] * P[:, 0] + R[r][1] * P[:, 1]) + R[r][2] * P[:, 2]) + T[r, 3] * t
                     for r in range(3)], axis=1)


def compute_point_to_plane(P, Q, N, factors):
    """ComputePointToPlane(..., compensation = true) (icp_fast.cc:256-324), all weights 1: the columns of wF and F
    are scaled by the kept points' factors (:284-289), the residual is not."""
    F = np.concatenate([np.cross(P, N), N], axis=1) * factors[:, None]
    A = F.T @ F
    b = -(F.T @ np.einsum("ij,ij->i", P - Q, N))
    x = pyref._solve_possibly_underdetermined(A, b)
    T = np.eye(4)
    angle = float(np.linalg.norm(x[:3]))
    with np.errstate(invalid="ignore", divide="ignore"):
        axis = x[:3] / angle
    if angle > 0.0 and np.all(np.isfinite(axis)):
        K = np.array([[0.0, -axis[2], axis[1]], [axis[2], 0.0, -axis[0]], [-axis[1], axis[0], 0.0]])
        T[:3, :3] = np.eye(3) + math.sin(angle) * K + (1.0 - math.cos(angle)) * (K @ K)
    T[:3, 3] = x[3:6]
    if not np.all(np.isfinite(T)):                                  # :315-321 hasNaN -> identity rotation
        T[:3, :3] = np.eye(3)
    return T


def icp_fast_align(source, target, target_normals, knn, guess=None, max_iteration=100, dist_outlier_ratio=0.7,
                   disable_convergence_check=False, trace=None):
    """IcpFast::Align with inner compensation.  knn(target_centred, P) -> (ids, d2)."""
    S = np.asarray(source, dtype=np.float64)
    Qt = np.asarray(target, dtype=np.float64).copy()
    Nq = np.asarray(target_normals, dtype=np.float64)
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
        P = motion_compensation(T_iter, S0)
        ids, d2 = knn(Qt, P)
        limit = pyref._quantile_limit(d2, dist_outlier_ratio)
        keep = np.nonzero((d2 != INF) & (d2 <= limit))[0]
        assert keep.size > 0
        fk = keep.astype(np.float64) / np.float64(P.shape[0])       # the factors travel with the kept points
        T_iter = compute_point_to_plane(P[keep], Qt[ids[keep]], Nq[ids[keep]], fk) @ T_iter
        it += 1
        rotations.append(pyref._quat_from_matrix(T_iter[:3, :3]))
        translations.append(T_iter[:3, 3].copy())
        if trace is not None:
            trace.append({"limit": limit, "kept": int(keep.size), "T_iter": T_iter.copy()})
        conv = (not disable_convergence_check) and pyref._check_convergence(rotations, translations)
        if conv or it >= max_iteration:
            score = math.exp(-float(np.sqrt(d2[keep]).sum()) / keep.size)
            break
    return {"result": T_mean @ T_iter @ G0, "iterations": it, "score": score, "kept": int(keep.size)}
