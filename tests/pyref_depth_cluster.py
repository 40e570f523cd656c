"""numpy restatement of RangeImage::DepthCluster (pre_processors/filter_range_image.cc:143-173, :245-309), written from
the reference independently of tests/cpp/depth_cluster_oracle.cc.  TEST INFRASTRUCTURE.

The image comes from pyref_filters.range_image_pixels (first point per pixel).  The edge mask is computed for the whole
image at once in float32 (numpy, no contraction); sin, cos and atan2 are taken in float64 and rounded to float32.  The
order is a breadth-first search that marks a pixel when it is first pushed: the reference marks at the first pop and
pushes duplicates, which pop in the same order, so the two agree exactly when the reference is restated right."""
from __future__ import annotations

from collections import deque

import numpy as np

import pyref_filters as PF

F = np.float32
STEPS = ((0, 1), (0, -1), (0, 2), (0, -2), (1, 0), (-1, 0))
THRESHOLD = F(10 / 180.0 * np.pi)


def resolutions(p):
    """(sin, cos) of the horizontal and the vertical resolution as LabelOneComponent derives them (:255-259)"""
    V, H = p["vertical_line_num"], p["horizontal_line_num"]
    hres = F(np.pi * 2 / np.float64(F(H)))
    vres = F(np.float64((p["top_angle"] - p["btm_angle"]) / F(V)) / 180.0 * np.pi)
    sc = lambda a: (F(np.sin(np.float64(a))), F(np.cos(np.float64(a))))   # noqa: E731
    return sc(hres), sc(vres)


def edge(a, b, sin_a, cos_a):
    """beta > threshold for ranges a, b (arrays), and beta"""
    a, b = np.asarray(a, F), np.asarray(b, F)
    d1, d2 = np.maximum(a, b), np.minimum(a, b)
    with np.errstate(all="ignore"):
        beta = np.arctan2(np.float64(d2 * sin_a), np.float64(d1 - d2 * cos_a)).astype(F)
    return beta > THRESHOLD, beta


def image(params, cloud):
    """-> (V*H float32 ranges, V*H int owners (-1 empty)), row-major"""
    p = PF._params("RangeImage", params)
    c = np.ascontiguousarray(cloud, F)
    V, H = p["vertical_line_num"], p["horizontal_line_num"]
    row, col = PF.range_image_pixels(p, c)
    ok = np.nonzero(row >= 0)[0]
    px = row[ok] * H + col[ok]
    owner = np.full(V * H, -1, np.int64)
    uniq, first = np.unique(px, return_index=True)          # first occurrence = smallest input index
    owner[uniq] = ok[first]
    rng = np.zeros(V * H, F)
    i = owner[uniq]
    x, y, z = c[i, 0] + p["offset_x"], c[i, 1] + p["offset_y"], c[i, 2] + p["offset_z"]
    with np.errstate(all="ignore"):
        rng[uniq] = np.sqrt(x * x + y * y + z * z)
    return rng, owner


def mask(params, rng):
    """6-bit edge mask per pixel, bit k for STEPS[k]"""
    p = PF._params("RangeImage", params)
    V, H = p["vertical_line_num"], p["horizontal_line_num"]
    img = np.asarray(rng, F).reshape(V, H)
    occ = ~(img.astype(np.float64) < 1e-6)
    (sh, ch), (sv, cv) = resolutions(p)
    out = np.zeros((V, H), np.uint8)
    for k, (dr, dc) in enumerate(STEPS):
        nb = np.zeros((V, H), F)
        nocc = np.zeros((V, H), bool)
        rows = np.arange(V) + dr
        inside = (rows >= 0) & (rows < V)
        cols = (np.arange(H) + dc) % H                      # one wrap suffices for H >= 2
        nb[inside] = img[rows[inside]][:, cols]
        nocc[inside] = occ[rows[inside]][:, cols]
        e, _ = edge(img, nb, sh if dr == 0 else sv, ch if dr == 0 else cv)
        out |= ((occ & nocc & e).astype(np.uint8) << k)
    return out.ravel()


def cluster(V, H, owner, msk, cloud):
    """labels, order and output from an image's owners and edge mask -> dict as oracle_depth_cluster"""
    c = np.ascontiguousarray(cloud, F)
    owner = np.asarray(owner).ravel()
    msk = np.asarray(msk).ravel()
    label = np.zeros(V * H, np.uint32)
    level = np.full(V * H, -1, np.int32)
    clusters = []
    nxt = 1
    for seed in np.nonzero(owner >= 0)[0]:                  # row-major
        if label[seed]:
            continue
        label[seed], level[seed] = nxt, 0
        order, queue = [], deque([int(seed)])
        while queue:
            q = queue.popleft()
            order.append(q)
            r, col = divmod(q, H)
            m = int(msk[q])
            for k, (dr, dc) in enumerate(STEPS):
                if not m >> k & 1:
                    continue
                t = (r + dr) * H + (col + dc) % H
                if not label[t]:
                    label[t], level[t] = nxt, level[q] + 1
                    queue.append(t)
        if len(order) >= 20:
            clusters.append((nxt, order))
        nxt += 1
    px = np.array([q for _, o in clusters for q in o], np.int64)
    index = owner[px].astype(np.int32) if len(px) else np.zeros(0, np.int32)
    return {"xyz": c[index, :3].copy(), "label": label[px] if len(px) else np.zeros(0, np.uint32), "index": index,
            "pixel_label": label, "level": level, "components": nxt - 1}


def depth_cluster(params, cloud):
    p = PF._params("RangeImage", params)
    V, H = p["vertical_line_num"], p["horizontal_line_num"]
    if len(cloud) == 0:
        raise PF.CheckFailed("inner_cloud_ != nullptr")
    if V <= 0 or H < 2:
        raise ValueError("RangeImage: a grid DepthCluster cannot run")
    rng, owner = image(params, cloud)
    msk = mask(params, rng)
    out = cluster(V, H, owner, msk, cloud)
    out.update(image=rng, owner=owner.astype(np.int32), mask=msk)
    return out
