"""Clouds and configurations shared by the filter-chain tests (tests/test_filters_oracle.py, tests/test_gpu_filters.py):
a synthetic 64-beam scan as (N,5) InnerPointType records, the two chains of the reference's shipped configuration
(config/lidar_only_kitti.xml:18-41 and :55-71) and clouds built to sit on the filters' decision borders."""
import numpy as np

from staticmapping_b200 import synth

F = np.float32
FLT_MAX = float(np.finfo(np.float32).max)


def scan(n_az=1875, seed=2):
    """lidar_scan in firing order with intensity and factor filled in; the ground lies near z = -1.73."""
    xyz = synth.lidar_scan(synth.make_scene(0), (0.0, 0.0, 0.0), seed=seed, n_beams=64, n_az=n_az)
    # the firing azimuths are exact fractions of a turn and some fall exactly on segment and column borders, where one
    # ulp of atan2f decides: turn the scan off that lattice
    c, s = np.cos(0.01234), np.sin(0.01234)
    xyz = np.stack([c * xyz[:, 0] - s * xyz[:, 1], s * xyz[:, 0] + c * xyz[:, 1], xyz[:, 2]], axis=1).astype(F)
    rng = np.random.default_rng(seed + 100)
    n = xyz.shape[0]
    return np.concatenate([xyz, rng.uniform(0, 255, (n, 1)).astype(F), (np.arange(n, dtype=F) / F(n))[:, None]], axis=1)


def records(xyz):
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    n = xyz.shape[0]
    return np.concatenate([xyz, np.arange(n, dtype=F)[:, None], np.linspace(0, 1, n, dtype=F)[:, None]], axis=1)


# the scan matcher's GroundRemoval2 of the shipped configuration, the ground height moved to this scene's
GROUND = dict(r_min=0.1, start_ground_height=-1.73, long_line_threshold=10, max_slope=0.12, max_error=0.1,
              max_dist_to_line=0.10, max_start_height=0.6, thread_num=4)
RANGE_IMAGE = dict(top_angle=30.0, btm_angle=-20.0, vertical_line_num=60)
CHAIN_SCAN = [("Range", dict(min_range=5.0)), ("AxisRange", dict(min=-2.0)), ("RandomSampler", dict(sampling_rate=0.5))]
CHAIN_MATCHER = [("GroundRemoval2", GROUND), ("RangeImage", RANGE_IMAGE)]
SINGLE = [("Range", dict(min_range=5.0, max_range=60.0)), ("AxisRange", dict(min=-1.0)),
          ("AxisRange", dict(min=-10.0, max=10.0, axis_index=0)),
          ("BoundingBoxRemoval", dict(min_x=-5, max_x=5, min_y=-5, max_y=5, min_z=-3, max_z=3)),
          ("RandomSampler", dict(sampling_rate=0.5)), ("RangeImage", RANGE_IMAGE), ("GroundRemoval2", GROUND)]


def predicate_edges():
    """points exactly on min / max, NaN and inf coordinates"""
    nan, inf = np.nan, np.inf
    return records([[3, 4, 0], [3, 4, 12], [0, 0, 0], [6, 8, 0], [5, 0, 0], [60, 0, 0], [0, 0, -2], [0, 0, 2],
                    [-10, 1, 1], [10, 1, 1], [nan, 1, 1], [1, nan, 1], [1, 1, nan], [inf, 0, 0], [0, -inf, 1],
                    [5, 5, 3], [5, 5, 3.0000002], [-5, -5, -3], [4.9999995, 0, 0], [1e20, 1e20, 1e20]])


def range_image_edges(p=None):
    """d_xy at 0.01, a row value of -0.5 and one at the top edge, a column rounding to W, pixels hit twice"""
    p = dict(top_angle=30.0, btm_angle=-15.0, vertical_line_num=40, horizontal_line_num=1800, **(p or {}))
    vres = np.deg2rad((p["top_angle"] - p["btm_angle"]) / p["vertical_line_num"])
    btm, top = np.deg2rad(p["btm_angle"]), np.deg2rad(p["top_angle"])
    d = 10.0
    e3, e6 = np.hypot(d, 0.3), np.hypot(d, 0.6)
    pts = [[0.01, 0, 0], [0.0099, 0, 0], [0.0, 0.0, 1.0],
           [d, 0.3, e3 * np.tan(btm - 0.5 * vres)], [d, 0.3, e3 * np.tan(btm - 1.5 * vres)],
           [d, 0.6, e6 * np.tan(top - 0.01 * vres)], [d, 0.6, e6 * np.tan(top + 0.01 * vres)],
           [d, -1e-4, 0.5], [d, 1e-4, 0.5],                 # h just below 2 pi -> column W -> 0, shared with h just above 0
           [7, 7, 1], [7.0001, 7.0001, 1.0001], [-3, 2, 0.2], [-3.0001, 2.0001, 0.2],
           [np.nan, 1, 1], [np.inf, 1, 1], [1, 1, np.inf]]
    fwd = records(pts)
    return [fwd, np.ascontiguousarray(fwd[::-1])]            # two points in one pixel, in both orders


def polar(seg, r, z, segment_num=180, frac=0.5):
    a = (np.asarray(seg, float) + frac) * 2 * np.pi / segment_num
    return np.stack([r * np.cos(a), r * np.sin(a), np.broadcast_to(z, np.shape(r))], axis=-1)


def ground_edges():
    """One cloud per GroundRemoval2 case, with the shipped parameters (ground at -1.73)."""
    g = -1.73
    r = np.arange(2.0, 20.0, 0.5)
    flat = lambda s, z=g, rr=r: polar(np.full(len(rr), s), rr, z)       # noqa: E731
    out = {}
    # a cell whose minimum drops by more than 0.5 after members joined: the earlier members stay
    out["min_drops"] = records(np.concatenate([flat(3), polar([4, 4, 4], np.array([6.01, 6.02, 6.03]), np.array([-1.0, -0.9, -1.72])),
                                               polar([4], np.array([6.04]), np.array([-0.95]))]))
    # segments 10..12 empty between populated ones; a segment whose only occupied bin is the last one
    out["empty_and_last_bin"] = records(np.concatenate([flat(9), flat(13), polar([11, 11], np.array([150.0, 170.0]), g)]))
    # a gap of more than long_line_threshold inside a line, the far part 0.3 above the extrapolation
    far = np.arange(32.0, 40.0, 0.5)
    out["long_line_break"] = records(np.concatenate([flat(20), polar(np.full(len(far), 20), far, g + 0.3),
                                                     flat(21), polar(np.full(len(far), 21), far, g + 0.02)]))
    # points exactly on the fitted line (distance 0 is "not ground") beside points slightly off it
    out["on_the_line"] = records(np.concatenate([flat(30, z=-1.75), polar([30, 30], np.array([4.1, 4.2]), np.array([-1.75, -1.70]))]))
    # a point whose own segment has no line: only the neighbour explains it
    out["neighbour_only"] = records(np.concatenate([flat(40), polar([41, 41], np.array([5.0, 9.0]), np.array([g + 0.03, g + 0.5]))]))
    # +k before -k (k = 5 at 180 segments): the lone point of segment 50 is ground by segment 55 (45 would say 0.13 away); that of
    # segment 70 is not, by segment 75 (65 would say ground)
    out["plus_k_first"] = records(np.concatenate([flat(55), flat(45, z=g + 0.10), polar([50], np.array([8.0]), np.array([g - 0.03])),
                                                  flat(65), flat(75, z=g + 0.10), polar([70], np.array([8.0]), np.array([g - 0.03]))]))
    # the wrap of the neighbour search across segment 0 and non-finite points
    out["wrap_and_nan"] = records(np.concatenate([flat(178), polar([1], np.array([6.0]), np.array([g + 0.02])),
                                                  [[np.nan, 1, g], [1, 1, np.nan], [np.inf, 2, g]]]))
    return out
