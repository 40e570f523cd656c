"""Clouds for RangeImage::DepthCluster (tests/test_depth_cluster_oracle.py, tests/test_gpu_depth_cluster.py): points
placed at pixel centres of a given grid, so each lands in the pixel it was built for, and shapes built to reach the
cases of the labelling and of the visiting order."""
import numpy as np

import filter_scenes as FS

F = np.float32


def grid(V, H, top=30.0, btm=-15.0):
    return dict(top_angle=top, btm_angle=btm, vertical_line_num=V, horizontal_line_num=H)


def at_pixels(params, pixels, ranges):
    """records at the centres of (row, col) pixels with the given ranges"""
    V, H = params["vertical_line_num"], params["horizontal_line_num"]
    top, btm = params.get("top_angle", 30.0), params.get("btm_angle", -15.0)
    px = np.asarray(pixels, np.float64).reshape(-1, 2)
    el = np.deg2rad(btm + (px[:, 0] + 0.5) * (top - btm) / V)
    az = px[:, 1] * 2 * np.pi / H
    r = np.broadcast_to(np.asarray(ranges, np.float64), (len(px),))
    return FS.records(np.stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)], axis=1))


def serpentine(V, H, r=10.0):
    """one path: every third column full height, joined at alternate ends through the two columns between; each
    column step is a new level, so the BFS runs about V * H / 3 levels deep"""
    px = []
    cols = list(range(0, H - 2, 3))
    for j, c in enumerate(cols):
        rows = range(V) if j % 2 == 0 else range(V - 1, -1, -1)
        px += [(row, c) for row in rows]
        if j + 1 < len(cols):
            end = V - 1 if j % 2 == 0 else 0
            px += [(end, c + 1), (end, c + 2)]
    return at_pixels(grid(V, H), px, r)


def cases():
    """name -> (RangeImage parameters, cloud)"""
    out = {}
    g = grid(16, 360)
    # a wall across column 0, and a second object in front of it (range jump: no edge)
    wall = [(r, c % 360) for r in range(4, 9) for c in range(350, 372)]
    front = [(r, c) for r in range(5, 8) for c in range(100, 110)]
    out["wrap"] = (g, np.concatenate([at_pixels(g, wall, 20.0), at_pixels(g, front, 5.0), at_pixels(g, front, 30.0)]))
    # one row with column 20 missing: only the +-2 hop joins the halves
    out["hop_two"] = (g, at_pixels(g, [(2, c) for c in range(10, 31) if c != 20], 8.0))
    # two lines of 19 and 20 pixels (the smaller one dropped), a single pixel and a pair
    out["sizes_19_20"] = (g, np.concatenate([at_pixels(g, [(3, c) for c in range(40, 59)], 9.0),
                                             at_pixels(g, [(6, c) for c in range(40, 60)], 9.0),
                                             at_pixels(g, [(10, 200)], 4.0), at_pixels(g, [(11, 5), (11, 6)], 4.0)]))
    # V = 1, H = 2: (0, +-1) both reach the other column, (0, +-2) the pixel itself
    g12 = grid(1, 2)
    out["v1_h2"] = (g12, at_pixels(g12, [(0, 0), (0, 1), (0, 0)], [5.0, 5.5, 7.0]))
    # a block: most pixels of level >= 2 have two parents on the level before, in (r, k) order
    block = [(r, c) for r in range(2, 8) for c in range(60, 75)]
    rng = 12.0 + 0.05 * np.arange(len(block))
    out["two_parents"] = (g, at_pixels(g, block, rng))
    # a serpentine several hundred levels deep
    out["serpentine"] = (grid(16, 300), serpentine(16, 300))
    # a range step inside a surface: the criterion splits it; inf / NaN coordinates beside it
    step = [(r, c) for r in range(8, 12) for c in range(150, 175)]
    ranges = np.where(np.array([c for _, c in step]) < 162, 10.0, 13.0)
    bad = FS.records([[np.inf, 0, 0], [np.nan, 1, 0], [1, np.nan, 0], [3, 3, np.nan], [-np.inf, 1, 0.1],
                      [np.inf, np.inf, 0]])
    out["split_and_nonfinite"] = (g, np.concatenate([bad[:3], at_pixels(g, step, ranges), bad[3:]]))
    out["many_clusters"] = (grid(60, 1800), many_clusters())
    return out


def many_clusters(seed=3):
    """2 700 blocks of 4 x 5 pixels at range 10 (each exactly 20 points, more kept components than the BFS grid has
    CTAs), three columns apart so no +-2 hop joins them; every other pixel holds a point at a random range in
    [30, 100], which makes thousands of components more, most of them dropped"""
    V, H = 60, 1800
    g = grid(V, H)
    inside = np.zeros((V, H), bool)
    for r0 in range(0, V, 5):
        for c0 in range(0, H, 8):
            inside[r0:r0 + 4, c0:c0 + 5] = True
    rows, cols = np.nonzero(inside)
    noise_r, noise_c = np.nonzero(~inside)
    rng = np.random.default_rng(seed)
    return np.concatenate([at_pixels(g, np.stack([rows, cols], 1), 10.0),
                           at_pixels(g, np.stack([noise_r, noise_c], 1), rng.uniform(30, 100, len(noise_r)))])
