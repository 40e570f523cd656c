"""pclomp's neighbour searches of Ndt (KDTREE, DIRECT26, DIRECT7, DIRECT1) without a GPU: the product's direct
searches (csrc/ndt.cu for_each_direct_cell and its leaf test, compiled for the host through
sm_debug_ndt_direct_neighbors), the oracle (oracle/ndt_search_oracle.cc) and the numpy restatement
(tests/pyref_ndt_search.py) on hand-built grids with known answers, on lidar scenes and on degenerate leaves."""
import numpy as np
import pytest

import oracle_lib as O
import oracle_ndt_search as OS
import pyref
import pyref_ndt_search as PS
import scenes
from staticmapping_b200 import _lib
from test_gpu_ndt_gicp_stages import grid_degenerate, grid_faces_and_signs, grid_invalid_leaf

F32 = np.float32
DIRECT = (PS.DIRECT26, PS.DIRECT7, PS.DIRECT1)


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=F32))


def product_neighbors(target, points, method, resolution=1.0):
    """The product's direct neighbour lists (host build of the kernel's search) over the oracle's leaves."""
    grid = PS.SearchGrid(target, resolution, method)
    p = _f32(points)
    min_b = np.ascontiguousarray(grid.min_b, np.int32)
    div_b = np.ascontiguousarray(grid.max_b - grid.min_b + 1, np.int32)
    keys = np.ascontiguousarray(grid.leaf_idx_arr, np.int32)
    npts = np.ascontiguousarray(grid.n, np.int32)
    counts = np.zeros(p.shape[0], np.int32)
    out = np.zeros((p.shape[0], 26), np.int32)
    rc = _lib.lib().sm_debug_ndt_direct_neighbors(method, p.ctypes.data, p.shape[0], resolution, min_b.ctypes.data,
                                                  div_b.ctypes.data, keys.ctypes.data, npts.ctypes.data, keys.size,
                                                  counts.ctypes.data, out.ctypes.data)
    assert rc == 0
    return [out[i, :counts[i]].copy() for i in range(p.shape[0])]


def all_neighbors(target, points, method, resolution=1.0):
    """-> (oracle, pyref, product) lists; the product's only for the direct methods."""
    o = OS.neighbors(target, points, method, resolution)
    p = PS.SearchGrid(target, resolution, method).neighbor_lists(_f32(points))
    d = product_neighbors(target, points, method, resolution) if method != PS.KDTREE else p
    return o, p, d


def assert_lists_equal(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(np.asarray(x, np.int64), np.asarray(y, np.int64)), (i, x, y)


# --------------------------------------------------------------------------------------- known-answer grids
def _cube_target(counts=None, skip=()):
    """A 3 x 3 x 3 block of unit cells at (2..4, 2..4, 2..4), each with 8 box-corner points (searchable, valid),
    except the cells in `counts` (cell -> number of points, a prefix of the corners plus jittered extras)."""
    rng = np.random.default_rng(3)
    corners = np.array([[x, y, z] for x in (0.25, 0.75) for y in (0.25, 0.75) for z in (0.25, 0.75)])
    pts = []
    for i in range(3):
        for j in range(3):
            for k in range(3):
                c = (2 + i, 2 + j, 2 + k)
                if c in skip:
                    continue
                n = (counts or {}).get(c, 8)
                extra = rng.uniform(0.1, 0.9, (max(n - 8, 0), 3))
                pts.append(np.asarray(c, np.float64) + np.concatenate([corners, extra])[:n])
    return _f32(np.concatenate(pts))


def _key(grid, cell):
    return int((np.asarray(cell, np.int64) - grid.min_b) @ grid.divb_mul)


def test_offset_lists_are_pclomps():
    half = PS.OFFSETS[PS.DIRECT26][:13]
    assert np.array_equal(PS.OFFSETS[PS.DIRECT26][13:], -half)
    assert not (PS.OFFSETS[PS.DIRECT26] == 0).all(axis=1).any()          # no centre cell
    assert len({tuple(o) for o in PS.OFFSETS[PS.DIRECT26]}) == 26
    assert PS.OFFSETS[PS.DIRECT7].tolist() == [[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1],
                                               [0, 0, -1]]


@pytest.mark.parametrize("method", DIRECT)
def test_full_block_gives_the_offsets_in_list_order(method):
    target = _cube_target()
    grid = PS.SearchGrid(target, 1.0, method)
    q = _f32([[3.5, 3.5, 3.5], [3.01, 3.99, 3.5]])                        # two points in the centre cell
    expected = [_key(grid, (3, 3, 3) + d) for d in PS.OFFSETS[method]]
    for lists in all_neighbors(target, q, method):
        assert_lists_equal(lists, [expected, expected])
    if method == PS.DIRECT26:
        assert _key(grid, (3, 3, 3)) not in expected


def test_leaf_with_five_points_is_never_a_neighbour_six_is():
    target = _cube_target(counts={(3, 3, 3): 5, (4, 3, 3): 6})
    grid = PS.SearchGrid(target, 1.0, PS.DIRECT7)
    centre, six = _key(grid, (3, 3, 3)), _key(grid, (4, 3, 3))
    for method in DIRECT:
        for lists in all_neighbors(target, _f32([[3.5, 3.5, 3.5], [4.5, 3.5, 3.5]]), method):
            flat = np.concatenate(lists)
            assert centre not in flat
            assert six in flat
    o, p, d = all_neighbors(target, _f32([[4.5, 3.5, 3.5]]), PS.DIRECT1)
    assert o[0].tolist() == p[0].tolist() == d[0].tolist() == [six]


def test_failed_covariance_leaf_is_excluded_by_the_direct_searches_only():
    target = grid_invalid_leaf()
    grid = PS.SearchGrid(target, 1.0, PS.KDTREE)
    assert grid.n.tolist() == [-1] and grid.searchable.tolist() == [1]
    c = grid.centroid[0].astype(np.float64)
    q = _f32([c + (0.5, 0.0, 0.0), c + (0.0, -0.5, 0.25)])
    o, p, _ = all_neighbors(target, q, PS.KDTREE)
    assert [x.tolist() for x in o] == [x.tolist() for x in p] == [[grid.leaf_idx[0]]] * 2
    for method in DIRECT:
        for lists in all_neighbors(target, q, method):
            assert all(x.size == 0 for x in lists)


def _division_differs(resolution, rng, n=200000):
    """Points where floorf(x / r) != floorf(x * (1 / r)) in float32."""
    x = (rng.integers(-3000, 3000, n) * F32(resolution)).astype(F32)
    r = F32(resolution)
    return x[np.floor(x / r) != np.floor(x * (F32(1.0) / r))]


def test_query_cell_uses_the_division_at_resolution_0_3():
    rng = np.random.default_rng(21)
    xs = _division_differs(0.3, rng)
    assert xs.size >= 10
    xs = xs[np.abs(xs) < 60][:40]
    r = F32(0.3)
    # a target with a valid leaf in every cell of a box that holds the query points
    cells = np.stack(np.meshgrid(np.arange(-210, 210), [0], [0], indexing="ij"), -1).reshape(-1, 3)
    corners = np.array([[x, y, z] for x in (0.2, 0.8) for y in (0.2, 0.8) for z in (0.2, 0.8)])
    target = _f32(((cells[:, None, :] + corners[None]) * 0.3).reshape(-1, 3))
    q = _f32(np.stack([xs, np.full(xs.size, 0.15, F32), np.full(xs.size, 0.15, F32)], 1))
    grid = PS.SearchGrid(target, 0.3, PS.DIRECT1)
    div = np.floor(q[:, 0] / r).astype(np.int64)
    mul = np.floor(q[:, 0] * (F32(1.0) / r)).astype(np.int64)
    assert np.all(div != mul)
    expected = [[_key(grid, (c, 0, 0))] if grid.min_b[0] <= c <= grid.max_b[0] else [] for c in div]
    assert sum(len(e) for e in expected) >= 10
    for lists in all_neighbors(target, q, PS.DIRECT1, resolution=0.3):
        assert_lists_equal(lists, expected)


def test_points_outside_the_box_get_the_in_box_offsets_only():
    target = _cube_target()
    grid = PS.SearchGrid(target, 1.0, PS.DIRECT26)
    q = _f32([[1.5, 3.5, 3.5], [5.5, 5.5, 5.5], [0.5, 3.5, 3.5], [3.5, 6.5, 3.5], [-0.0, 2.0, 2.0]])
    for method in DIRECT:
        exp = []
        for p in q:
            cell = np.floor(p / F32(1.0)).astype(np.int64)
            exp.append([_key(grid, cell + d) for d in PS.OFFSETS[method]
                        if np.all(cell + d >= grid.min_b) and np.all(cell + d <= grid.max_b)])
        for lists in all_neighbors(target, q, method):
            assert_lists_equal(lists, exp)
        if method == PS.DIRECT26:
            assert [len(e) for e in exp] == [9, 1, 0, 0, 0]


def test_nan_and_huge_points_have_no_neighbours():
    target = _cube_target()
    q = _f32([[np.nan, 3.5, 3.5], [3.5, 3.5, np.inf], [1e12, 3.5, 3.5], [3.5, -1e12, 3.5], [3.5, 3.5, 3.5]])
    for method in DIRECT:
        for lists in all_neighbors(target, q, method):
            assert [x.size for x in lists[:4]] == [0, 0, 0, 0] and lists[4].size > 0


# --------------------------------------------------------------------------------------- scenes
def _lidar(pair):
    s, t, _ = scenes.lidar_pair(pair=pair)
    return _f32(s), _f32(t)


SCENES = {
    "lidar-0": lambda: _lidar(0),
    "lidar-2": lambda: _lidar(2),
    "degenerate": lambda: (grid_degenerate()[::3] + F32(0.3), grid_degenerate()),
    "faces-and-signs": lambda: (grid_faces_and_signs()[::2], grid_faces_and_signs()),
}


@pytest.mark.parametrize("method", PS.METHODS)
@pytest.mark.parametrize("scene", list(SCENES))
def test_neighbour_lists_oracle_pyref_product(scene, method):
    src, tgt = SCENES[scene]()
    p = np.array([0.12, 0.05, -0.04, 0.004, 0.006, -0.03])
    q = pyref._transform_cloud_f32(pyref._ndt_pose_matrix_f32(p), src)
    o, py, d = all_neighbors(tgt, q, method)
    assert_lists_equal(o, py)
    assert_lists_equal(d, py)
    assert sum(x.size for x in o) > 0


@pytest.mark.parametrize("method", PS.METHODS)
@pytest.mark.parametrize("scene", ["lidar-0", "degenerate"])
def test_derivatives_oracle_vs_pyref(scene, method):
    src, tgt = SCENES[scene]()
    for p in (np.zeros(6), np.array([0.2, -0.15, 0.05, 0.01, -0.008, 0.03])):
        so, go, Ho, nbo = OS.ndt_derivatives(src, tgt, p, method)
        sp, gp, Hp, nbp = PS.ndt_derivatives(src, tgt, p, method)
        sa, ga, Ha, _ = PS.ndt_derivatives(src, tgt, p, method, absolute=True)
        assert nbp == nbo
        assert abs(sp - so) <= 2e-5 * sa
        assert np.all(np.abs(gp - go) <= 2e-5 * ga.max())
        assert np.all(np.abs(Hp - Ho) <= 2e-5 * Ha.max())


def test_kdtree_restatement_is_the_oracles_ndt_align():
    src, tgt = _lidar(1)
    a = O.ndt_align(src, tgt)
    b = OS.ndt_align(src, tgt, OS.KDTREE)
    assert a["rc"] == b["rc"] == 1
    for k in ("result", "fitness", "iterations", "trans_probability", "mean_neighbors"):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


@pytest.mark.parametrize("method", PS.METHODS)
@pytest.mark.parametrize("pair", [0, 2])
def test_align_oracle_vs_pyref(pair, method):
    src, tgt = _lidar(pair)
    o = OS.ndt_align(src, tgt, method)
    p = PS.ndt_align(src, tgt, method)
    assert o["rc"] == 1
    assert p["iterations"] == o["iterations"] and p["evaluations"] == o["evaluations"]
    dt, dr = scenes.se3_error(o["result"], p["result"])
    assert dt < 1e-4 and dr < 1e-4, (dt, dr)
    assert abs(p["mean_neighbors"] - o["mean_neighbors"]) < 1e-3
