"""Clouds shared by the GroundRemoval tests (tests/test_ground_removal_oracle.py, tests/test_gpu_ground_removal.py):
(N,5) InnerPointType records, each built against one rule of the filter (include/sm_b200.h), with the parameters to
run it at.  scenes() -> {name: (records, [params, ...])}, params = (min_point_num_in_voxel, leaf_size,
height_threshold)."""
import numpy as np

from filter_scenes import records, scan  # noqa: F401

F = np.float32
NAN, INF = float("nan"), float("inf")
DEFAULT = (10, 0.8, 0.15)


def _flat(center, count, dz=0.0, seed=0):
    """count points around `center`, z spread over [cz, cz + dz]"""
    rng = np.random.default_rng(seed)
    p = np.tile(np.asarray(center, np.float64), (count, 1))
    p[:, :2] += rng.uniform(-0.05, 0.05, (count, 2))
    p[:, 2] += np.linspace(0.0, dz, count)
    return p


def trunc_not_floor():
    """+-0.5 leaf share voxel 0 (floor would split them into two voxels of 5); z just below leaf_size is tested, z equal
    to it is not; z = -leaf lands in iz = -1, tested"""
    below = float(np.nextafter(F(0.8), F(0)))
    parts = [np.array([[0.4 * s, 0.1, 0.05] for s in (1, -1)] * 5),
             _flat((5.0, 5.0, below), 10), _flat((9.0, 5.0, 0.8), 10), _flat((13.0, 5.0, -0.8), 10, -0.1),
             _flat((5.0, -5.0, -0.4), 10, 0.5)]
    return records(np.concatenate(parts))


def rounding():
    """coordinates within a few ulps of k * leaf: float division rounds some quotients onto k and some just below"""
    pts = []
    for leaf in (0.8, 0.1, 0.3, 0.7):
        lf = F(leaf)
        for k in (-7, -3, -1, 1, 2, 3, 5, 10, 29):
            c = F(k) * lf
            for u in range(-3, 4):
                x = F(c)
                for _ in range(abs(u)):
                    x = np.nextafter(x, F(np.sign(u) * np.inf))
                pts.append([x, 0.25, float(x) * 0.5])
    return records(np.array(pts))


def non_finite():
    """NaN, +-inf and 1e12 coordinates land in the INT_MIN voxel of their axis; the (INT_MIN, INT_MIN, INT_MIN) voxel
    sorts first"""
    bad = [NAN, INF, -INF, 1e12, -1e12]
    pts = [[a, b, c] for a in bad for b in bad for c in (NAN, 1e12, 0.1)]
    pts += [[0.1, 0.1, z] for z in bad] * 3 + [[a, 0.1, 0.1] for a in bad] * 3 + [[NAN, NAN, NAN]] * 12
    return records(np.array(pts))


def z_rules():
    """a NaN z among finite ones of the same (ix, iy, INT_MIN) voxel, a voxel whose z are all NaN, z below -1e9 (max_z
    stays -1e9), signed zeros"""
    parts = [np.array([[0.1, 0.1, z] for z in (NAN, 1e12, -5e9, NAN, 3e12)] * 2),
             np.array([[2.1, 0.1, NAN]] * 10),
             np.array([[4.1, 0.1, z] for z in (-2e9, -3e9, -2e9 - 256, -1e10, -4e9)] * 2),
             np.array([[6.1, 0.1, z] for z in (0.0, -0.0)] * 5), np.array([[-0.0, -0.0, z] for z in (-0.0, 0.0)] * 5),
             np.array([[8.1, 0.1, z] for z in (-0.0, 0.15)] * 5)]
    return records(np.concatenate(parts))


def sizes():
    """voxels of 1 .. 12 points: min_point_num_in_voxel - 1 and min_point_num_in_voxel at every tested minimum"""
    return records(np.concatenate([_flat((2.0 * c + 0.1, 0.1, 0.1), c, 0.01, seed=c) for c in range(1, 13)]))


def delta_at_threshold():
    """delta == height_threshold exactly (ground), and the next float delta above it (kept)"""
    thr = F(0.15)
    parts = []
    for i, lo in enumerate((F(0.0), F(-0.5), F(-0.2), F(0.25), F(-1.1))):
        hi = F(lo + thr)
        if F(hi - lo) != thr:
            continue
        above = np.nextafter(hi, F(1))
        while F(above - lo) <= thr:
            above = np.nextafter(above, F(1))
        for j, top in enumerate((hi, above)):
            z = np.r_[lo, np.full(8, (lo + top) / 2), top]
            parts.append(np.stack([np.full(10, 2.0 * i + 0.1), np.full(10, 2.0 * j + 0.1), z], 1))
    return records(np.concatenate(parts))


def duplicates():
    """every point written three times, interleaved"""
    base = _flat((0.3, 0.3, -0.5), 4, 0.02)
    return records(np.concatenate([base, base[::-1], base]))


def spread(n=5000, seed=3):
    """a scene over a few metres around the ground, for the parameter sweeps (one voxel holds it all at leaf 1000)"""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform([-6, -6, -1.8], [6, 6, 1.5], (n, 3))
    xyz[: n // 2, 2] = -1.73 + rng.normal(size=n // 2) * 0.03
    return records(xyz)


def scenes():
    return {
        "trunc_not_floor": (trunc_not_floor(), [DEFAULT, (5, 0.8, 0.15)]),
        "rounding": (rounding(), [(1, 0.8, 0.15), (1, 0.1, 0.15), (1, 0.3, 0.15), (1, 0.7, 0.15), (2, 0.1, 0.15)]),
        "non_finite": (non_finite(), [(1, 0.8, 0.15), (3, 0.8, 0.15), (1, 0.8, 1e13)]),
        "z_rules": (z_rules(), [DEFAULT, (10, 0.8, 3.1e12), (10, 0.8, 6e9), (10, 0.8, -0.0), (10, 0.8, 0.0)]),
        "sizes": (sizes(), [DEFAULT, (1, 0.8, 0.15), (7, 0.8, 0.15), (12, 0.8, 0.15), (13, 0.8, 0.15)]),
        "delta_at_threshold": (delta_at_threshold(), [DEFAULT]),
        "duplicates": (duplicates(), [DEFAULT, (12, 0.8, 0.15), (13, 0.8, 0.15)]),
        "parameters": (spread(), [(0, 0.8, 0.15), (-4, 0.8, 0.15), (10, 0.8, -0.1), (10, 0.8, NAN), (3, 0.0, 0.15),
                                  (3, -0.8, 0.15), (3, -0.0, 0.15), (10, 1000.0, 5.0), (10, 1000.0, 0.15),
                                  (10, 0.2, 0.15), (10, 2.0, 0.3)]),
    }


def span_limit():
    """(records, leaf, fits): per axis the indices other than INT_MIN may span 2^21 - 1 voxels, not 2^21"""
    lim = (1 << 21) - 1
    cases = []
    for axis in range(3):
        for lo, hi, fits in ((0, lim - 1, True), (-(lim // 2), lim // 2, True), (0, lim, False), (-5, lim, False)):
            p = np.zeros((14, 3))
            p[:6, axis] = lo
            p[6:12, axis] = hi
            p[12, axis] = NAN
            p[13, axis] = 1e12                               # INT_MIN: its own slot, outside the span
            cases.append((records(p), 1.0, fits))
    cases.append((records(np.stack([np.linspace(0, 3000, 4000), np.zeros(4000), np.zeros(4000)], 1)), 1e-3, False))
    return cases
