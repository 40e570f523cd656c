"""Scenes for MultiviewRegistratorLumPcl: frames of one structured world seen from known poses, each given with a
perturbed pose, plus small clouds built against single rules.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import numpy as np


def rot(roll, pitch, yaw):
    cr, sr, cp, sp, cy, sy = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    return (np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]]) @ np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
            @ np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]]))


def pose(x, y, z, roll, pitch, yaw):
    T = np.eye(4)
    T[:3, :3] = rot(roll, pitch, yaw)
    T[:3, 3] = (x, y, z)
    return T


def world(n, rng):
    """A room: floor, four walls and two pillars, n points, in a 10 m x 8 m x 3 m box."""
    parts = []
    k = n // 7
    parts.append(np.c_[rng.uniform(-5, 5, 2 * k), rng.uniform(-4, 4, 2 * k), np.zeros(2 * k)])
    for x in (-5.0, 5.0):
        parts.append(np.c_[np.full(k, x), rng.uniform(-4, 4, k), rng.uniform(0, 3, k)])
    for y in (-4.0, 4.0):
        parts.append(np.c_[rng.uniform(-5, 5, k), np.full(k, y), rng.uniform(0, 3, k)])
    rest = n - sum(len(p) for p in parts)
    a = rng.uniform(0, 2 * np.pi, rest)
    cx = np.where(np.arange(rest) % 2 == 0, 1.5, -2.0)
    parts.append(np.c_[cx + 0.3 * np.cos(a), 0.5 + 0.3 * np.sin(a), rng.uniform(0, 3, rest)])
    return np.concatenate(parts)


def frames(n_frames=3, n_points=6000, seed=0, step=0.4, perturb=(0.04, 0.01), noise=0.005, cols=4):
    """n_frames (cloud (n, cols) float32 with x y z first and the rest an index pattern, given 4x4 pose, true pose).
    Frame k sees the world from true pose T_k (a walk along x with a slow turn); its given pose is T_k with a random
    error of about perturb = (metres, radians)."""
    rng = np.random.default_rng(seed)
    W = world(n_points * 2, rng)
    out = []
    for k in range(n_frames):
        T = pose(step * k, 0.1 * k, 0.0, 0.0, 0.0, 0.05 * k)
        sel = rng.choice(len(W), n_points, replace=False)
        local = (W[sel] - T[:3, 3]) @ T[:3, :3]
        local += rng.normal(0, noise, local.shape)
        cloud = np.zeros((n_points, cols), np.float32)
        cloud[:, :3] = local
        if cols > 3:
            cloud[:, 3:] = (np.arange(n_points)[:, None] * 7 + np.arange(cols - 3)[None] + k * 1000) % 9973
        e = rng.normal(0, 1, 6)
        E = pose(*(perturb[0] * e[:3]), *(perturb[1] * e[3:]))
        out.append((cloud, (T @ E).astype(np.float32), T))
    return out


def pairwise_misalignment(clouds):
    """Mean distance from each point of cloud j to its nearest point of cloud i over all pairs j < i, counting pairs
    closer than 0.25 m."""
    from scipy.spatial import cKDTree
    tot, cnt = 0.0, 0
    for i in range(len(clouds)):
        t = cKDTree(clouds[i][:, :3].astype(np.float64))
        for j in range(i):
            d, _ = t.query(clouds[j][:, :3].astype(np.float64))
            d = d[d < 0.25]
            tot += d.sum()
            cnt += d.size
    return tot / max(cnt, 1)
