"""MultiviewRegistratorLumPcl's LUM restated in numpy, from PCL 1.8.1's lum.hpp, CorrespondenceEstimation and
transforms.h, independently of the product (csrc/lum_host.h) and of oracle/lum_oracle.cc.  TEST INFRASTRUCTURE.

The per-point geometry is float32 as PCL's (getTransformation with the C library's cosf / sinf, transformPointCloud, the compounded pair, its average
and difference, the 15 terms of M'M / M'Z); everything after the per-edge sums is float64: the sums (math.fsum),
D = M'M^-1 M'Z, s^2, cinv / cinvd, G / B, X (numpy lstsq) and the pose update.  Compared with the oracle to rounding.

  correspondences(src, tgt, metric)   brute-force 1-NN of each finite point of src among the finite points of tgt,
                                      the smallest index among equal distances, kept iff d2 <= 0.25^2; metric
                                      "float" is FLANN's ((dx^2 + dy^2) + dz^2) in float32, "double" the same over the
                                      coordinates widened to float64
  compute_edge(...)                   LUM::computeEdge of one edge under given poses
  step(...)                           one LUM::compute iteration: every edge, G and B, X, the pose update, the sum
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math

import numpy as np

F32, F64 = np.float32, np.float64
MAX_D2 = 0.25 * 0.25

# getTransformation calls the C library's cosf / sinf, which round differently from float(cos(double)) now and then
_libm = ctypes.CDLL(ctypes.util.find_library("m"))
for _f in ("cosf", "sinf"):
    getattr(_libm, _f).restype = ctypes.c_float
    getattr(_libm, _f).argtypes = [ctypes.c_float]


def get_transformation(pose):
    """pcl::getTransformation(x, y, z, roll, pitch, yaw) -> 3x4 float32"""
    x, y, z, roll, pitch, yaw = (F32(v) for v in pose)
    A, B = F32(_libm.cosf(yaw)), F32(_libm.sinf(yaw))
    C, D = F32(_libm.cosf(pitch)), F32(_libm.sinf(pitch))
    E, F = F32(_libm.cosf(roll)), F32(_libm.sinf(roll))
    DE, DF = D * E, D * F
    return np.array([[A * C, A * DF - B * E, B * F + A * DE, x],
                     [B * C, A * E + B * DF, B * DE - A * F, y],
                     [-D, C * F, C * E, z]], F32)


def apply(T, p):
    """((m0 x + m1 y) + m2 z) + m3 per row, float32; p (n, 3)"""
    p = p.astype(F32)
    out = np.empty_like(p)
    for r in range(3):
        out[:, r] = ((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3]
    return out


def transform_cloud(T, p):
    """transformPointCloud of a cloud that is not dense: points with a non-finite coordinate are copied"""
    out = apply(T, p)
    bad = ~np.isfinite(p).all(1)
    out[bad] = p[bad]
    return out


def correspondences(src, tgt, metric):
    """(k, 2) int32 (query, match), ascending in query"""
    qi = np.nonzero(np.isfinite(src).all(1))[0]
    ti = np.nonzero(np.isfinite(tgt).all(1))[0]
    out = []
    if len(ti) == 0:
        return np.zeros((0, 2), np.int32)
    t = tgt[ti]
    for lo in range(0, len(qi), 256):
        q = src[qi[lo:lo + 256]]
        if metric == "float":
            d = (q[:, None, :].astype(F32) - t[None].astype(F32)).astype(F32)
            d2 = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(F64)
        else:
            d = q[:, None, :].astype(F64) - t[None].astype(F64)
            d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        m = d2.argmin(1)                           # the first (smallest index) among equal minima
        best = d2[np.arange(len(q)), m]
        keep = best <= MAX_D2
        out.append(np.c_[qi[lo:lo + 256][keep], ti[m[keep]]])
    return np.concatenate(out).astype(np.int32) if out else np.zeros((0, 2), np.int32)


def incidence_correction(pose):
    """LUM::incidenceCorrection, float64"""
    x, y, z, roll, pitch = (float(v) for v in pose[:5])
    cx, sx, cy, sy = math.cos(roll), math.sin(roll), math.cos(pitch), math.sin(pitch)
    J = np.eye(6)
    J[0, 4] = y * sx - z * cx
    J[0, 5] = y * cx * cy + z * sx * cy
    J[1, 3] = z
    J[1, 4] = -x * sx
    J[1, 5] = -x * cx * cy + z * sy
    J[2, 3] = -y
    J[2, 4] = x * cx
    J[2, 5] = -x * sx * cy - y * sy
    J[3, 5] = sy
    J[4, 4] = sx
    J[4, 5] = cx * cy
    J[5, 4] = cx
    J[5, 5] = -sx * cy
    return J


def compute_edge(src_cloud, tgt_cloud, src_pose, tgt_pose, corr):
    """LUM::computeEdge -> dict(pairs, sums[15], abs_sums[15] (sums of |term|), D[6], ss, cinv (6, 6), cinvd[6]); the sums in float64 (fsum)"""
    s = apply(get_transformation(src_pose), src_cloud[corr[:, 0]]) if len(corr) else np.zeros((0, 3), F32)
    t = apply(get_transformation(tgt_pose), tgt_cloud[corr[:, 1]]) if len(corr) else np.zeros((0, 3), F32)
    ok = np.isfinite(s).all(1) & np.isfinite(t).all(1)
    s, t = s[ok], t[ok]
    a = F32(0.5) * (s + t)
    d = s - t
    terms = [a[:, 0], a[:, 1], a[:, 2], a[:, 0] * a[:, 2], a[:, 0] * a[:, 1], a[:, 1] * a[:, 2],
             a[:, 1] * a[:, 1] + a[:, 2] * a[:, 2], a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1],
             a[:, 0] * a[:, 0] + a[:, 2] * a[:, 2], d[:, 0], d[:, 1], d[:, 2],
             a[:, 1] * d[:, 2] - a[:, 2] * d[:, 1], a[:, 0] * d[:, 1] - a[:, 1] * d[:, 0],
             a[:, 2] * d[:, 0] - a[:, 0] * d[:, 2]]
    S = [math.fsum(x.astype(F64).tolist()) for x in terms]
    absS = [math.fsum(np.abs(x.astype(F64)).tolist()) for x in terms]
    n = int(ok.sum())
    res = dict(pairs=n, sums=np.array(S), abs_sums=np.array(absS), D=np.zeros(6), ss=0.0, cinv=np.zeros((6, 6)), cinvd=np.zeros(6))
    if n < 3:
        return res
    # M'M of lum.hpp: each row of M for a pair with average (x, y, z) is [I | [[0, -y, z], [-z, x, 0], [y, 0, -x]]]
    MM = np.zeros((6, 6))
    MM[0, 4], MM[0, 5], MM[1, 3], MM[1, 4], MM[2, 3], MM[2, 5] = -S[1], S[2], -S[2], S[0], S[1], -S[0]
    MM[3, 4], MM[3, 5], MM[4, 5] = -S[3], -S[4], -S[5]
    MM[3, 3], MM[4, 4], MM[5, 5] = S[6], S[7], S[8]
    MM[0, 0] = MM[1, 1] = MM[2, 2] = n
    MM = np.triu(MM) + np.triu(MM, 1).T
    MZ = np.array(S[9:15])
    try:
        D = np.linalg.solve(MM, MZ)
    except np.linalg.LinAlgError:      # a singular M'M: PCL's inverse yields inf / NaN, and so s^2
        D = np.full(6, np.nan)
    A, Dd = a.astype(F64), d.astype(F64)
    r0 = Dd[:, 0] - (D[0] + A[:, 2] * D[5] - A[:, 1] * D[4])
    r1 = Dd[:, 1] - (D[1] + A[:, 0] * D[4] - A[:, 2] * D[3])
    r2 = Dd[:, 2] - (D[2] + A[:, 1] * D[3] - A[:, 0] * D[5])
    ss = math.fsum((r0 * r0 + r1 * r1 + r2 * r2).tolist())
    res.update(D=D, ss=ss)
    if ss < 1e-13 or not math.isfinite(ss):
        return res
    res.update(cinv=MM / ss, cinvd=MZ / ss)
    return res


def step(clouds, vertex_frame, edges, poses, connected_only):
    """One LUM::compute iteration.  clouds: the transformed frames; vertex_frame[v]: the frame of vertex v's cloud;
    edges: {(s, t): corr}; poses (n, 6) before the iteration.  connected_only: solve only the vertices joined to
    vertex 0 through edges with a non-zero cinv (the others get X = 0), else all vertices by least squares.
    Returns (edge results by (s, t), X (6(n - 1)), poses after, sum of the pose changes' norms, the vertices joined to
    vertex 0)."""
    n = len(poses)
    er = {k: compute_edge(clouds[vertex_frame[k[0]]], clouds[vertex_frame[k[1]]], poses[k[0]], poses[k[1]], c)
          for k, c in edges.items()}
    G = np.zeros((6 * (n - 1), 6 * (n - 1)))
    B = np.zeros(6 * (n - 1))
    for (s, t), r in er.items():       # edge s -> t: forward for vi = s, backward for vi = t
        for vi, vj, sign in ((s, t, 1.0), (t, s, -1.0)):
            if vi == 0:
                continue
            bi = slice(6 * (vi - 1), 6 * vi)
            G[bi, bi] += r["cinv"]
            if vj > 0:
                G[bi, 6 * (vj - 1):6 * vj] = -r["cinv"]
            B[bi] += sign * r["cinvd"]
    joined, todo = {0}, [0]
    while todo:
        v = todo.pop()
        for (s, t), r in er.items():
            if r["cinv"].any() and v in (s, t):
                w = t if v == s else s
                if w not in joined:
                    joined.add(w)
                    todo.append(w)
    solve = sorted(joined - {0}) if connected_only else list(range(1, n))
    X = np.zeros(6 * (n - 1))
    if solve:
        idx = np.concatenate([np.arange(6 * (v - 1), 6 * v) for v in solve])
        X[idx] = np.linalg.lstsq(G[np.ix_(idx, idx)], B[idx], rcond=None)[0]
    out = np.array(poses, F64)
    total = 0.0
    for vi in range(1, n):
        dp = -np.linalg.solve(incidence_correction(poses[vi]), X[6 * (vi - 1):6 * vi])
        total += float(np.linalg.norm(dp))
        out[vi] = out[vi] + dp
    return er, X, out, total, sorted(joined)
