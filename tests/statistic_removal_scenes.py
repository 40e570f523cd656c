"""Clouds shared by the StatisticRemoval tests (tests/test_statistic_removal_oracle.py, tests/test_gpu_statistic_removal.py):
(N,5) InnerPointType records built to exercise the filter's neighbour ties, non-finite points and planted outliers."""
import numpy as np

from filter_scenes import records, scan  # noqa: F401
from test_search_formulation_model import _adversarial_clouds

F = np.float32


def planted(n=3000, n_out=12, seed=5):
    """a dense cluster with n_out far points planted among it; returns (records, planted indices)"""
    rng = np.random.default_rng(seed)
    xyz = rng.normal(size=(n, 3)) * 0.5
    at = np.sort(rng.choice(n, n_out, replace=False))
    dirs = rng.normal(size=(n_out, 3))
    xyz[at] = dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * rng.uniform(20, 40, (n_out, 1))
    return records(xyz), at


def ties():
    """duplicated points, a grid and a line: many neighbours at the same distance, the K-th one included"""
    rng = np.random.default_rng(7)
    base = rng.normal(size=(400, 3))
    dup = np.concatenate([base, base[::3], base[::5]])
    grid = np.stack(np.meshgrid(np.arange(10.0), np.arange(8.0), np.arange(6.0)), -1).reshape(-1, 3) * 0.5
    line = np.stack([np.linspace(-3, 3, 701), np.zeros(701), np.zeros(701)], 1)
    return {"duplicates": records(dup), "grid": records(grid), "line": records(line)}


def non_finite():
    """NaN and inf coordinates among finite points (each of x, y, z, and intensity, which does not matter)"""
    rng = np.random.default_rng(9)
    r = records(rng.normal(size=(2500, 3)))
    r[5, 0] = np.nan
    r[17, 1] = np.inf
    r[400, 2] = -np.inf
    r[401:420, :3] = np.nan
    r[1000, 3] = np.nan
    r[-1, 2] = np.nan
    return r


def adversarial():
    """the k-NN tests' adversarial clouds as records"""
    return {name: records(T) for name, T in _adversarial_clouds()}
