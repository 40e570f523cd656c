"""numpy restatement of the reference's scan pre-processing filters (pre_processors/filter_*.cc), written from the
reference sources independently of tests/cpp/filters_oracle.cc.  TEST INFRASTRUCTURE: a transcription error shared by
the GPU chain and the C++ restatement does not pass both.  float32 arithmetic is numpy's (IEEE, no contraction); the
line fit is numpy.linalg.lstsq in float64, cast to float32 as FitLocalLine does; atan2 is taken in float64 and rounded
to float32."""
from __future__ import annotations

import numpy as np

F = np.float32
FLT_MAX = F(np.finfo(np.float32).max)
INT_MIN = -2 ** 31

DEFAULTS = {
    "Range": dict(min_range=0.0, max_range=FLT_MAX),
    "AxisRange": dict(min=-FLT_MAX, max=FLT_MAX, axis_index=2),
    "BoundingBoxRemoval": dict(min_x=-FLT_MAX, min_y=-FLT_MAX, min_z=-FLT_MAX, max_x=FLT_MAX, max_y=FLT_MAX, max_z=FLT_MAX),
    "RandomSampler": dict(sampling_rate=1.0),
    "RangeImage": dict(top_angle=30.0, btm_angle=-15.0, offset_x=0.0, offset_y=0.0, offset_z=0.0, vertical_line_num=40,
                       horizontal_line_num=1800),
    "GroundRemoval2": dict(r_max=100.0, r_min=1.0, bin_num=200, segment_num=180, start_ground_height=-0.25,
                           long_line_threshold=1.0, max_long_line_height=0.1, max_start_height=0.2, max_error=0.05,
                           max_slope=np.tan(np.pi / 12.0), max_b=0.1, max_dist_to_line=0.05, search_angle=10.0,
                           thread_num=4),
}
INT_PARAMS = {"axis_index", "vertical_line_num", "horizontal_line_num", "bin_num", "segment_num", "thread_num"}


class CheckFailed(RuntimeError):
    pass


def _params(name, params):
    p = dict(DEFAULTS[name])
    for k, v in (params or {}).items():
        if k not in p:
            raise KeyError(k)
        p[k] = v
    return {k: (int(v) if k in INT_PARAMS else F(v)) for k, v in p.items()}


def _trunc(q):
    """C's (int)q for an array of floats; INT_MIN where the conversion is undefined (x86's answer)."""
    q = np.asarray(q, np.float64)
    ok = np.isfinite(q) & (q > -2147483649.0) & (q < 2147483648.0)
    return np.where(ok, np.trunc(np.where(ok, q, 0.0)), INT_MIN).astype(np.int64)


def _atan2f(y, x):
    return np.arctan2(np.asarray(y, np.float64), np.asarray(x, np.float64)).astype(F)


def valid(name, params=None):
    p = _params(name, params)
    if name == "AxisRange":
        return bool(p["max"] > p["min"] and 0 <= p["axis_index"] <= 2)
    if name == "BoundingBoxRemoval":
        return bool(p["min_x"] < p["max_x"] and p["min_y"] < p["max_y"] and p["min_z"] < p["max_z"])
    if name == "RandomSampler":
        return bool(F(0) <= p["sampling_rate"] <= F(1))
    return True


def fmix32(h):
    h = np.asarray(h, np.uint32).copy()
    h ^= h >> np.uint32(16); h *= np.uint32(0x85EBCA6B); h ^= h >> np.uint32(13); h *= np.uint32(0xC2B2AE35)
    h ^= h >> np.uint32(16)
    return h


def sampler_keep(scan_index, rate, seed):
    x = np.asarray(scan_index).astype(np.uint32) * np.uint32(0x9E3779B9) + np.uint32(seed)
    return fmix32(x).astype(np.float64) <= np.float64(F(rate)) * 4294967296.0


def range_image_pixels(p, c):
    """-> (row, col) int arrays, -1 where the point is an outlier before the pixel test."""
    x, y, z = c[:, 0] + p["offset_x"], c[:, 1] + p["offset_y"], c[:, 2] + p["offset_z"]
    H, W = p["vertical_line_num"], p["horizontal_line_num"]
    hres = F(np.pi * 2 / np.float64(F(W)))
    vres = F(np.float64((p["top_angle"] - p["btm_angle"]) / F(H) / F(180)) * np.pi)
    with np.errstate(all="ignore"):
        dxy = np.sqrt(x * x + y * y)
        v = _atan2f(z, dxy)
        row = _trunc((v.astype(np.float64) - np.float64(p["btm_angle"] / F(180)) * np.pi) / np.float64(vres))
        h = _atan2f(y, x)
        h = np.where(h < 0, (h.astype(np.float64) + np.pi * 2).astype(F), h)
        q = (h / hres).astype(F)
        # lround: half away from zero; q >= 0 wherever it is used
        col = np.where(np.isfinite(q), np.floor(np.where(np.isfinite(q), q, 0).astype(np.float64) + 0.5), -1).astype(np.int64)
    col = np.where(col >= W, col - W, col)
    ok = ~(dxy < F(0.01)) & (row >= 0) & (row < H) & (col >= 0) & (col < W)
    return np.where(ok, row, -1), np.where(ok, col, -1)


def gr2_cells(p, c):
    two_pi = F(np.pi * 2)
    delta_alpha = two_pi / F(p["segment_num"])
    delta_bin = (p["r_max"] - p["r_min"]) / F(p["bin_num"])
    with np.errstate(all="ignore"):
        rng = np.sqrt(c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1])
        rad = _atan2f(c[:, 1], c[:, 0])
        rad = np.where(rad < 0, rad + two_pi, rad).astype(F)
        s = np.clip(_trunc(rad / delta_alpha), 0, p["segment_num"] - 1)
        b = np.clip(_trunc((rng - p["r_min"]) / delta_bin), 0, p["bin_num"] - 1)
    return s, b, rng


def fit_line(pts):
    a = np.asarray(pts, np.float64)
    X = np.stack([a[:, 0], np.ones(len(a))], axis=1)
    sol = np.linalg.lstsq(X, a[:, 1], rcond=None)[0]
    return F(sol[0]), F(sol[1])


def vertical_distance(point, seg):
    margin, dist = F(0.1), F(-1.0)
    for (d0, z0, d1, z1) in seg:
        if not d0 < d1:
            raise CheckFailed("line.start[0] < line.end[0]")
        if d0 - margin < point[0] and d1 + margin > point[0]:
            dist = abs(point[1] - ((point[0] - d0) / (d1 - d0) * (z1 - z0) + z0))
    return dist


def _fit_segment(p, mins):
    """mins: [(d, z)] of the occupied bins in bin order with their bin numbers -> the segment's lines."""
    lines = []
    if not mins or mins[0][0] >= p["bin_num"] - 1:
        return lines
    pts = [mins[0][1]]
    cur = (F(0), F(0))
    long_line, ground_h = False, p["start_ground_height"]
    i = 1
    while i < len(mins):
        cp = mins[i][1]
        if cp[0] - pts[-1][0] >= p["long_line_threshold"]:
            long_line = True
        expected = FLT_MAX
        if long_line and len(pts) > 2:
            expected = cur[0] * cp[0] + cur[1]
        if len(pts) >= 2:
            pts.append(cp)
            cur = fit_line(pts)
            err = max(abs(cur[0] * q[0] + cur[1] - q[1]) for q in pts)
            if err > p["max_error"] or abs(cur[0]) > p["max_slope"] or \
                    (long_line and abs(expected - cp[1]) > p["max_long_line_height"]):
                pts.pop()
                if len(pts) >= 3:
                    m, b = fit_line(pts)
                    lines.append((pts[0][0], m * pts[0][0] + b, pts[-1][0], m * pts[-1][0] + b))
                    ground_h = m * pts[-1][0] + b
                long_line = False
                pts = [pts[-1]]
                continue            # the reference's --i: the same bin again
        elif not long_line and abs(pts[-1][1] - ground_h) < p["max_start_height"]:
            pts.append(cp)
        else:
            pts = [cp]
        i += 1
    if len(pts) > 2:
        m, b = fit_line(pts)
        lines.append((pts[0][0], m * pts[0][0] + b, pts[-1][0], m * pts[-1][0] + b))
    return lines


def ground_removal2(p, c, stages=None):
    S, B = p["segment_num"], p["bin_num"]
    s, b, rng = gr2_cells(p, c)
    cell = s * B + b
    z = c[:, 2]
    members = {}
    cmin = {}
    with np.errstate(all="ignore"):
        for i in range(len(c)):
            k = int(cell[i])
            if k not in members or z[i] < cmin[k][1]:
                cmin[k] = (rng[i], z[i])
            if np.float64(z[i]) <= np.float64(cmin[k][1]) + 0.5:
                members.setdefault(k, []).append(i)
        segs = []
        for si in range(S):
            mins = [(bi, cmin[si * B + bi]) for bi in range(B) if (si * B + bi) in members]
            segs.append(_fit_segment(p, mins))
        k_max = int(_trunc(np.float64(p["search_angle"]) / 180.0 * np.pi / np.float64(F(np.pi * 2 / S))))
        cand = [sign * k for k in range(k_max, 0, -1) for sign in (1, -1)]
        ground = np.zeros(len(c), bool)
        for k, idx in members.items():
            si = k // B
            for i in idx:
                pt = (rng[i], z[i])
                d = vertical_distance(pt, segs[si])
                if d < 0:
                    for o in cand:
                        d = vertical_distance(pt, segs[(si + o) % S])
                        if d > 0:
                            break
                ground[i] = d > 0 and d <= p["max_dist_to_line"]
    if stages is not None:
        stages.update(cell=cell, members=members, cell_min=cmin, segments=segs)
    return ~ground


def filter_flags(name, params, cloud, scan_index=None, seed=1):
    c = np.ascontiguousarray(cloud, F)
    p = _params(name, params)
    n = len(c)
    with np.errstate(all="ignore"):
        if name == "Range":
            r = np.sqrt(c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1] + c[:, 2] * c[:, 2])
            return (r >= p["min_range"]) & (r <= p["max_range"])
        if name == "AxisRange":
            if (p["min"] == -FLT_MAX and p["max"] == FLT_MAX) or not 0 <= p["axis_index"] <= 2:
                return np.ones(n, bool)
            v = c[:, p["axis_index"]]
            return ~((v < p["min"]) | (v > p["max"]))
        if name == "BoundingBoxRemoval":
            if not valid(name, params):
                raise CheckFailed("BoundingBox")
            inside = np.ones(n, bool)
            for a, ax in enumerate("xyz"):
                inside &= (c[:, a] >= p["min_" + ax]) & (c[:, a] <= p["max_" + ax])
            return ~inside
        if name == "RandomSampler":
            if np.float64(p["sampling_rate"]) > 0.999:
                return np.ones(n, bool)
            return sampler_keep(np.arange(n) if scan_index is None else scan_index, p["sampling_rate"], seed)
        if name == "RangeImage":
            if p["vertical_line_num"] <= 0 or p["horizontal_line_num"] <= 0:
                raise ValueError("RangeImage size")
            row, col = range_image_pixels(p, c)
            px = np.where(row >= 0, row * p["horizontal_line_num"] + col, -1)
            keep = np.zeros(n, bool)
            first = {}
            for i in np.nonzero(px >= 0)[0]:
                if first.setdefault(int(px[i]), i) == i:
                    keep[i] = True
            return keep
        if name == "GroundRemoval2":
            return ground_removal2(p, c)
    raise KeyError(name)


def chain(filters, cloud, seed=1):
    r = np.ascontiguousarray(cloud, F)
    index = np.arange(len(r), dtype=np.int32)
    for name, params in filters:
        if len(r) == 0:
            break
        keep = filter_flags(name, params, r, index, seed)
        r, index = r[keep], index[keep]
    return r, index
