"""Scenes of IcpFast with inner compensation (Interface::EnableInnerCompensation), shared by the CPU and GPU tests."""
from __future__ import annotations

import functools
import math

import numpy as np

import oracle_lib as O
import scenes
from staticmapping_b200 import synth


def se3(angle_deg, axis, t):
    """Rotation by angle_deg about axis, then translation t."""
    a = np.asarray(axis, dtype=np.float64); a = a / np.linalg.norm(a)
    th = math.radians(angle_deg)
    K = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + math.sin(th) * K + (1.0 - math.cos(th)) * (K @ K)
    T[:3, 3] = t
    return T


@functools.lru_cache(maxsize=None)
def corner_target():
    """The config-1 corner target through CalculateNormals."""
    _, tgt, _ = scenes.corner_pair()
    return O.calculate_normals(tgt)


@functools.lru_cache(maxsize=None)
def model_exact():
    """A scan taken while the platform moved by T_star: source point i (f_i = i / N) is a surface point q_i seen
    from Interp(T_star, f_i), i.e. s_i = G0^-1 Interp(T_star, f_i)^-1 (q_i - mu) + 1 cm noise, G0 = T_mean^-1 G.
    IcpFast with inner compensation models exactly this, so it returns T_mean T_star T_mean^-1 G.
    Returns (source, target points, target normals, guess, expected result)."""
    tp, tn = corner_target()
    mu = scenes.target_mean(tp)
    T_mean = np.eye(4); T_mean[:3, 3] = mu
    G = se3(1.0, (0.0, 0.0, 1.0), (0.05, -0.03, 0.0))
    G0 = np.linalg.inv(T_mean) @ G
    T_star = se3(2.0, (0.2, 0.1, 1.0), (0.4, 0.1, 0.02))
    q = synth.corner_scene_cloud(5000, 4242).astype(np.float64)
    n = q.shape[0]
    rng = np.random.default_rng(7)
    src = np.empty_like(q)
    G0_inv = np.linalg.inv(G0)
    for i in range(n):
        _, Ti = O.interpolate_transform(np.eye(4), T_star, np.float32(i / n))
        p = np.linalg.inv(Ti) @ np.append(q[i] - mu, 1.0)
        src[i] = (G0_inv @ p)[:3]
    src += rng.normal(scale=0.01, size=src.shape)
    return src, tp, tn, G, T_mean @ T_star @ np.linalg.inv(T_mean) @ G
