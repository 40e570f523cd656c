"""Second, independent restatement of registrator::Ndt with each of pclomp's neighbour searches
(setNeighborhoodSearchMethod, registrators/pclomp/ndt_omp.h:184; switch at ndt_omp_impl.hpp:233-246), in numpy,
written from the pclomp sources.  It reuses the plain restatement's pieces (tests/pyref.py) and differs from it in
the neighbour search only:

* KDTREE: pyref.NdtGrid.radius_search, unchanged.
* DIRECT26 / DIRECT7 / DIRECT1: VoxelGridCovariance::getNeighborhoodAtPoint / 7 / 1
  (voxel_grid_covariance_omp_impl.hpp:373-441).  The query cell is int(floor(x / leaf_size_)) in float32 (a division,
  :379-381; the grid itself is built with a multiplication by 1 / leaf_size_); offsets are taken in list order when
  min_b <= ijk + d <= max_b (:385-390), and their leaf is kept when it exists with nr_points >= 6 (:394-395), so a
  leaf whose covariance failed (nr_points = -1) is not a neighbour.  No distance test, no sort.
  DIRECT26's list is pcl::getAllNeighborCellIndices() of stock PCL, which is not vendored: restated from upstream PCL
  (getHalfNeighborCellIndices, then its negatives); it holds no (0, 0, 0).
  A point whose floor(x / leaf_size_) is not finite or lies outside [min_b - 1, max_b + 1] on some axis has no
  neighbour (static_cast<int> is undefined there in the reference)."""
from __future__ import annotations

import contextlib

import numpy as np

import pyref

F32 = np.float32
KDTREE, DIRECT26, DIRECT7, DIRECT1 = 0, 1, 2, 3
METHODS = (KDTREE, DIRECT26, DIRECT7, DIRECT1)
MIN_POINTS_PER_VOXEL = 6


def _all_neighbor_cell_indices():
    half = [(i, j, -1) for i in (-1, 0, 1) for j in (-1, 0, 1)]     # getHalfNeighborCellIndices: (i, j, -1), i outer
    half += [(i, -1, 0) for i in (-1, 0, 1)]                         # then (i, -1, 0)
    half += [(-1, 0, 0)]                                             # then (-1, 0, 0)
    return half + [(-a, -b, -c) for a, b, c in half]                 # getAllNeighborCellIndices: half, then -half


OFFSETS = {
    DIRECT26: np.array(_all_neighbor_cell_indices(), dtype=np.int64),
    DIRECT7: np.array([(0, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)], dtype=np.int64),
    DIRECT1: np.zeros((1, 3), dtype=np.int64),
}


class SearchGrid(pyref.NdtGrid):
    """pyref.NdtGrid whose radius_search is the given method's neighbour search (pyref.ndt_derivatives calls it)."""

    def __init__(self, target_f32, resolution=1.0, method=KDTREE):
        super().__init__(target_f32, resolution)
        t = np.ascontiguousarray(target_f32, dtype=F32)
        inv = F32(1.0) / F32(resolution)
        self.min_b = np.floor(t.min(axis=0) * inv).astype(np.int64)
        self.max_b = np.floor(t.max(axis=0) * inv).astype(np.int64)
        div_b = self.max_b - self.min_b + 1
        self.divb_mul = np.array([1, div_b[0], div_b[0] * div_b[1]], dtype=np.int64)
        self.leaf_idx_arr = np.asarray(self.leaf_idx, dtype=np.int64)   # ascending (std::map order)
        self.method = method

    def radius_search(self, pts_f32):
        if self.method == KDTREE:
            return super().radius_search(pts_f32)
        return self.direct_search(pts_f32)

    def direct_search(self, pts_f32):
        """-> (point index, leaf position) pairs, per point in offset order."""
        pts = np.ascontiguousarray(pts_f32, dtype=F32)
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            f = np.floor(pts / F32(self.resolution))                        # float32 division
            ok = (np.isfinite(f).all(axis=1) & (f >= self.min_b - 1).all(axis=1) & (f <= self.max_b + 1).all(axis=1))
        ijk = np.where(ok[:, None], f, 0.0).astype(np.int64)
        L = self.leaf_idx_arr
        pis, lis, ks = [], [], []
        for k, d in enumerate(OFFSETS[self.method]):
            c = ijk + d
            inb = ok & ((c >= self.min_b) & (c <= self.max_b)).all(axis=1)
            key = (c - self.min_b) @ self.divb_mul
            pos = np.minimum(np.searchsorted(L, key), L.size - 1)
            keep = inb & (L[pos] == key)
            keep &= self.n[pos] >= MIN_POINTS_PER_VOXEL
            pi = np.flatnonzero(keep)
            pis.append(pi); lis.append(pos[pi]); ks.append(np.full(pi.size, k))
        pi, li, kk = np.concatenate(pis), np.concatenate(lis), np.concatenate(ks)
        o = np.lexsort((kk, pi))
        return pi[o], li[o]

    def neighbor_lists(self, pts_f32):
        """-> per point, the neighbour leaf indices (voxel index of the grid) in the order they are used."""
        pi, li = self.radius_search(np.ascontiguousarray(pts_f32, dtype=F32))
        n = np.asarray(pts_f32).shape[0]
        bounds = np.searchsorted(pi, np.arange(n + 1))
        keys = self.leaf_idx_arr[li]
        return [keys[bounds[i]:bounds[i + 1]] for i in range(n)]


def ndt_derivatives(source_f32, target_f32, p, method, resolution=1.0, outlier_ratio=0.55, absolute=False):
    """computeDerivatives at pose vector p with the method's search -> (score, g[6], H[6,6], mean neighbours)."""
    src = np.ascontiguousarray(source_f32, dtype=F32)
    grid = SearchGrid(target_f32, resolution, method)
    trans = pyref._transform_cloud_f32(pyref._ndt_pose_matrix_f32(p), src)
    return pyref.ndt_derivatives(grid, src, trans, p, outlier_ratio, absolute=absolute)


@contextlib.contextmanager
def _pyref_grid(method):
    # pyref.ndt_align builds its grid as pyref.NdtGrid(target, resolution); hand it this search's grid instead
    plain = pyref.NdtGrid
    pyref.NdtGrid = lambda target, resolution: SearchGrid(target, resolution, method)
    try:
        yield
    finally:
        pyref.NdtGrid = plain


def ndt_align(source_f32, target_f32, method, guess=None, **kw):
    """Ndt::Align with the method's search: pyref.ndt_align's Newton loop over this module's grid."""
    with _pyref_grid(method):
        return pyref.ndt_align(source_f32, target_f32, guess, **kw)
