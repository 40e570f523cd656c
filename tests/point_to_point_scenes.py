"""Scenes of IcpFast with the point-to-point minimizer, shared by the CPU and GPU tests.  Each returns
(source, target points, target normals, guess, max_iteration); the normals are required by SetInputTarget but the
minimizer does not read them."""
from __future__ import annotations

import functools

import numpy as np

import inner_compensation_scenes as ICS
import oracle_lib as O
import scenes


@functools.lru_cache(maxsize=None)
def corner():
    """Config 1: the 3-plane corner pair, target through CalculateNormals; the ground truth is scenes.corner_pair's."""
    src, tgt, _ = scenes.corner_pair()
    tp, tn = O.calculate_normals(tgt)
    return src, tp, tn, np.eye(4), 100


@functools.lru_cache(maxsize=None)
def identical():
    """Source == target: every match has d2 = 0, M is symmetric positive semi-definite, so R = I and t = 0."""
    _, tp, tn, _, _ = corner()
    return tp.copy(), tp, tn, np.eye(4), 100


@functools.lru_cache(maxsize=None)
def plane():
    """A single plane z = 0 (3 600 seeded uniform points on 3 m x 3 m: a regular grid would put source points at equal
    distance from several targets), the source rotated 2 deg about z and shifted in the plane: every centred match
    lies in the plane, so M has rank 2."""
    rng = np.random.default_rng(3)
    tp = np.stack([rng.uniform(0, 3, 3600), rng.uniform(0, 3, 3600), np.zeros(3600)], axis=1)
    tn = np.tile([0.0, 0.0, 1.0], (tp.shape[0], 1))
    T = ICS.se3(2.0, (0, 0, 1), (0.03, -0.02, 0.0))
    src = tp[::3] @ T[:3, :3].T + T[:3, 3]
    return src, tp, tn, np.eye(4), 100


@functools.lru_cache(maxsize=None)
def reflection():
    """A 12 x 8 grid of 1 m at z = +-0.2 m whose source is its mirror image in z: each source point's nearest target
    point is its own partner (0.4 m against >= 1 m), so the kept matches correlate z negatively and det(U V^T) < 0."""
    gx, gy = np.meshgrid(np.arange(12) * 1.0, np.arange(8) * 1.0)
    z = np.where(np.random.default_rng(7).random(gx.size) < 0.5, 0.2, -0.2)
    tp = np.stack([gx.ravel(), gy.ravel(), z], axis=1)
    tn = np.tile([0.0, 0.0, 1.0], (tp.shape[0], 1))
    return tp * np.array([1.0, 1.0, -1.0]), tp, tn, np.eye(4), 3


@functools.lru_cache(maxsize=None)
def one_match():
    """One source point: one kept match, M = 0 exactly, R = I and t = q - p."""
    _, tp, tn, _, _ = corner()
    return tp[:1] + np.array([0.01, -0.02, 0.005]), tp, tn, np.eye(4), 100


@functools.lru_cache(maxsize=None)
def collinear():
    """Target and source on one line (the source shifted along and across it): every centred match is collinear,
    M has rank 1 and R is not unique."""
    s = np.arange(200) * 0.05
    d = np.array([1.0, 2.0, 0.5]) / np.linalg.norm([1.0, 2.0, 0.5])
    tp = s[:, None] * d
    tn = np.tile([0.0, 0.0, 1.0], (tp.shape[0], 1))
    src = tp[::2] + np.array([0.012, -0.004, 0.003])
    return src, tp, tn, np.eye(4), 100


SCENES = {"corner": corner, "identical": identical, "plane": plane, "reflection": reflection,
          "one_match": one_match, "collinear": collinear}
# scenes whose rotation is unique in every iteration: product, oracle and numpy must agree on R itself
UNIQUE = ("corner", "identical", "plane", "reflection", "one_match")
