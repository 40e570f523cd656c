"""Clouds shared by the RandomSamplerWithPlaneDetect tests (tests/test_plane_sampler_oracle.py,
tests/test_gpu_plane_sampler.py): (N,5) InnerPointType records, each built against one rule of the sampler
(include/sm_b200.h), with the parameters to run it at.  scenes() -> {name: (records, [params, ...])}, params =
(sampling_rate, leaf_size, min_point_num_in_voxel) as after the setters.  At leaf 0.8 a voxel with 1.6 <= z < 2.4 has
iz = 2, so it runs RANSAC."""
import numpy as np

from filter_scenes import records, scan  # noqa: F401

F = np.float32
NAN = float("nan")
DEFAULT = (0.5, 0.8, 10)


def _plane(center, count, normal_axis=2, noise=0.0, seed=0, half=0.3):
    """count points on the plane through `center` across `normal_axis`, spread +-half along the other two axes, with
    a uniform offset of +-noise along the normal"""
    rng = np.random.default_rng(seed)
    p = np.tile(np.asarray(center, np.float64), (count, 1))
    for a in range(3):
        p[:, a] += rng.uniform(-noise, noise, count) if a == normal_axis else rng.uniform(-half, half, count)
    return p


def flat_ground():
    """voxels with iz = 0 and iz = -1: flat ones (z range <= 0.2) are plane points, one 0.5 m deep is not, a small
    one is skipped"""
    parts = [_plane((0.4 + 0.8 * k, 0.4, 0.1), 30, noise=0.05, seed=k) for k in range(6)]
    parts += [_plane((0.4, 2.0, -1.2), 25, noise=0.09, seed=7), _plane((3.0, 2.0, 0.35), 25, noise=0.25, seed=8),
              _plane((5.0, 2.0, 0.1), 9, seed=9)]
    return records(np.concatenate(parts))


def walls():
    """vertical planes above iz = 0: RANSAC passes, so their points are plane points"""
    parts = [_plane((4.4 + 0.8 * k, 1.2, 2.0), 60, normal_axis=0, noise=0.01, seed=k) for k in range(3)]
    parts += [_plane((2.0, 4.4, 2.0), 80, normal_axis=1, noise=0.02, seed=5)]
    return records(np.concatenate(parts))


def noisy_planes():
    """horizontal planes at z = 2 whose inlier share is 0.9, 0.85 (the float 0.85f passes > 0.85), 0.84 and 0.8; the
    outliers lie 0.3 m off the plane"""
    parts = []
    for j, (good, bad) in enumerate([(90, 10), (85, 15), (84, 16), (80, 20), (170, 30)]):
        c = (0.4 + 0.8 * (j + 2), 0.4, 2.0)
        on = _plane(c, good, noise=0.01, seed=10 + j)
        off = _plane((c[0], c[1], 2.3), bad, noise=0.005, seed=20 + j)
        parts += [on, off]
    return records(np.concatenate(parts))


def degenerate():
    """two voxels of identical points (zero normal: every sample passes the 0 / 0 test and every point is an inlier):
    at (8.4, 0.4, 2) the float covariance is not exactly zero and the refined plane keeps them all, at (11, 0.5, 2)
    it is, and the refined plane is NaN; a collinear voxel (1000 rejected draws, no model); voxels of exactly 2 min
    and 2 min - 1 points (min 10)"""
    same = np.tile([8.4, 0.4, 2.0], (25, 1))
    exact = np.tile([11.0, 0.5, 2.0], (25, 1))
    j = np.arange(25)[:, None]
    line = np.array([8.25, 1.75, 1.625]) + j * np.array([1 / 256, 1 / 128, 1 / 64])
    parts = [same, exact, line, _plane((10.0, 0.4, 2.0), 20, seed=1), _plane((10.0, 2.0, 2.0), 19, seed=2)]
    return records(np.concatenate(parts))


def nan_x():
    """points with a NaN x and iz > 0 share voxel (INT_MIN, iy, 2): every distance is NaN, so the best count is 0 and
    the loop runs its 51 iterations; NaN points next to a plane voxel"""
    a = _plane((0.0, 0.4, 2.0), 25, seed=3)
    a[:, 0] = NAN
    b = _plane((2.0, 0.4, 2.0), 30, seed=4)
    b[::7, 0] = NAN
    return records(np.concatenate([a, b]))


def big_voxel(count=3000, seed=6):
    """one RANSAC voxel of `count` points (past the one-warp size) with 10 % outliers, next to small ones"""
    on = _plane((2.0, 2.0, 2.0), count - count // 10, noise=0.03, seed=seed, half=0.39)
    off = _plane((2.0, 2.0, 2.3), count // 10, noise=0.05, seed=seed + 1, half=0.39)
    rng = np.random.default_rng(seed + 2)
    mixed = np.concatenate([on, off])[rng.permutation(count)]
    return records(np.concatenate([mixed, _plane((4.0, 2.0, 2.0), 40, seed=seed + 3)]))


def scenes():
    return {
        "flat_ground": (flat_ground(), [DEFAULT, (0.1, 0.8, 10), (0.5, 0.8, 30)]),
        "walls": (walls(), [DEFAULT, (0.25, 0.8, 5)]),
        "noisy_planes": (noisy_planes(), [DEFAULT, (0.1, 0.8, 10)]),
        "degenerate": (degenerate(), [DEFAULT, (0.5, 0.8, 11)]),
        "nan_x": (nan_x(), [DEFAULT]),
        "leaf_at_or_below_threshold": (walls(), [(0.5, 0.2, 10), (0.5, 0.1, 10), (0.5, -0.8, 10),
                                                 (0.5, float(np.nextafter(F(0.2), F(1))), 10)]),
        "copy": (walls(), [(1.0, 0.8, 10), (float(np.nextafter(F(0.999999), F(1))), 0.8, 10)]),
        "near_copy": (walls(), [(float(np.nextafter(F(0.999999), F(0))), 0.8, 10), (0.999999, 0.8, 10)]),
        "big_voxel": (big_voxel(), [DEFAULT]),
    }
