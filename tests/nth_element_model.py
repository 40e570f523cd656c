"""Python models of CalculateNormals in std::nth_element's order (SM_NORMALS_ORDER_NTH_ELEMENT).  TEST INFRASTRUCTURE.

  introselect          a sequential restatement of libstdc++'s std::nth_element (introselect: median of three moved to
                       the front, Hoare's unguarded partition, a heap select once 2 * floor(log2 n) rounds are spent,
                       an insertion sort of the last <= 3 elements), written from the algorithm
  introselect_parallel the GPU's formulation of the same rounds (csrc/nth_element.cu): each partition computed from
                       stopper counts instead of two scans
  counts_partition     that partition alone
  normals_perm         the index array the whole BuildNormals recursion (builder/data/cloud_types.cc:105-144) leaves
  normals_from_perm    the leaf routine (cloud_types.cc:73-103) over that array, vectorised over the leaves: kept
                       means and unit normals in the reference's column order (ascending representative index)

Every function works on an index array `perm` and compares keys[perm[i]] with '<' only, as the reference's CompareDim
does, so -0.0 and +0.0 are equal."""
from __future__ import annotations

import numpy as np


def lg(n):
    return int(n).bit_length() - 1


# ---- the sequential restatement --------------------------------------------------------------------------------------

def _median_to_first(p, k, first, a, b, c):
    """swap p[first] with the median of p[a], p[b], p[c] (comparison order as libstdc++'s __move_median_to_first)"""
    ka, kb, kc = k[p[a]], k[p[b]], k[p[c]]
    if ka < kb:
        m = b if kb < kc else (c if ka < kc else a)
    elif ka < kc:
        m = a
    elif kb < kc:
        m = c
    else:
        m = b
    p[first], p[m] = p[m], p[first]


def _unguarded_partition(p, k, lo, hi, pivot_key):
    while True:
        while k[p[lo]] < pivot_key:
            lo += 1
        hi -= 1
        while pivot_key < k[p[hi]]:
            hi -= 1
        if not lo < hi:
            return lo
        p[lo], p[hi] = p[hi], p[lo]
        lo += 1


def _adjust_heap(p, k, base, hole, n, value):
    top, child = hole, hole
    while child < (n - 1) // 2:
        child = 2 * (child + 1)
        if k[p[base + child]] < k[p[base + child - 1]]:
            child -= 1
        p[base + hole] = p[base + child]
        hole = child
    if (n & 1) == 0 and child == (n - 2) // 2:
        child = 2 * (child + 1)
        p[base + hole] = p[base + child - 1]
        hole = child - 1
    parent = (hole - 1) // 2
    while hole > top and k[p[base + parent]] < k[value]:
        p[base + hole] = p[base + parent]
        hole = parent
        parent = (hole - 1) // 2
    p[base + hole] = value


def heap_select(p, k, first, middle, last):
    """max-heap of [first, middle), then every later element below the top replaces it (libstdc++'s __heap_select)"""
    n = middle - first
    if n >= 2:
        parent = (n - 2) // 2
        while True:
            _adjust_heap(p, k, first, parent, n, p[first + parent])
            if parent == 0:
                break
            parent -= 1
    for i in range(middle, last):
        if k[p[i]] < k[p[first]]:
            v = p[i]
            p[i] = p[first]
            _adjust_heap(p, k, first, 0, n, v)


def insertion_sort(p, k, first, last):
    for i in range(first + 1, last):
        v = p[i]
        if k[v] < k[p[first]]:
            p[first + 1:i + 1] = p[first:i]
            p[first] = v
        else:
            j = i
            while k[v] < k[p[j - 1]]:
                p[j] = p[j - 1]
                j -= 1
            p[j] = v


def introselect(keys, nth, perm=None, first=0, last=None, rounds=None):
    """std::nth_element(perm + first, perm + nth, perm + last) in place (perm: list; default iota over keys).
    Returns (perm, took_heap_select).  `rounds`, if a list, receives (first, last, cut, perm snapshot) per round."""
    k = keys
    p = list(range(len(keys))) if perm is None else perm
    last = len(p) if last is None else last
    if first == last or nth == last:
        return p, False
    depth = 2 * lg(last - first)
    while last - first > 3:
        if depth == 0:
            heap_select(p, k, first, nth + 1, last)
            p[first], p[nth] = p[nth], p[first]
            return p, True
        depth -= 1
        _median_to_first(p, k, first, first + 1, first + (last - first) // 2, last - 1)
        cut = _unguarded_partition(p, k, first + 1, last, k[p[first]])
        if rounds is not None:
            rounds.append((first, last, cut, list(p)))
        if cut <= nth:
            first = cut
        else:
            last = cut
    insertion_sort(p, k, first, last)
    return p, False


# ---- the GPU's formulation -------------------------------------------------------------------------------------------

def counts_partition(pk, lo, hi):
    """Hoare's unguarded partition of [lo + 1, hi) around the pivot pk[lo], from counts (pk: the keys in array order).
    A left stopper is an x with !(x < p), met scanning up; a right stopper an x with !(p < x), met scanning down.  The
    a-th left stopper L_a swaps with the a-th right stopper R_a while L_a < R_a, i.e. iff at least a right stoppers lie
    above L_a; K such pairs swap.  The scan then stops at min(L_{K+1}, R_K) (R_0 = hi, L_{K+1} = hi if none).
    Returns (left positions, right positions, cut): swapping pk[L[a]] with pk[R[a]] for all a is the partition."""
    x = pk[lo + 1:hi]
    p = pk[lo]
    isl = ~(x < p)
    isr = ~(p < x)
    pos = np.arange(lo + 1, hi)
    r_above = int(isr.sum()) - np.cumsum(isr)          # right stoppers strictly above each position
    a = np.cumsum(isl)                                  # rank of each left stopper, from 1
    l_swap = isl & (r_above >= a)
    L = pos[l_swap]
    K = len(L)
    R = pos[isr][::-1][:K]                              # the K highest right stoppers, from the top
    rest = pos[isl & ~l_swap]
    cut = min(int(rest[0]) if len(rest) else hi, int(R[K - 1]) if K else hi)
    return L, R, cut


def introselect_parallel(keys, nth, perm=None, first=0, last=None, rounds=None):
    """introselect with every partition from counts_partition; the same arguments and results as introselect"""
    keys = np.asarray(keys, np.float64)
    p = np.arange(len(keys), dtype=np.int64) if perm is None else np.asarray(perm, np.int64).copy()
    last = len(p) if last is None else last
    if first == last or nth == last:
        return list(p), False
    depth = 2 * lg(last - first)
    while last - first > 3:
        if depth == 0:
            q = list(p)
            heap_select(q, keys, first, nth + 1, last)
            q[first], q[nth] = q[nth], q[first]
            return q, True
        depth -= 1
        at = [first, first + 1, first + (last - first) // 2, last - 1]   # distinct while last - first > 3
        q = [int(v) for v in p[at]]
        _median_to_first(q, keys, 0, 1, 2, 3)
        p[at] = q
        pk = keys[p]
        L, R, cut = counts_partition(pk, first, last)
        p[L], p[R] = p[R], p[L].copy()
        if rounds is not None:
            rounds.append((first, last, cut, [int(v) for v in p]))
        if cut <= nth:
            first = cut
        else:
            last = cut
    q = [int(v) for v in p]
    insertion_sort(q, keys, first, last)
    return q, False


# ---- the whole recursion ---------------------------------------------------------------------------------------------

def _arg_max3(ext):
    mv, mi = 0.0, 0
    for i in range(3):
        if ext[i] > mv:
            mv, mi = ext[i], i
    return mi


def normals_perm(points, small=48):
    """BuildNormals' index array after the recursion; segments above `small` points use the counts formulation"""
    pts = np.ascontiguousarray(np.asarray(points, np.float64))
    n = len(pts)
    perm = np.arange(n, dtype=np.int64)
    cols = [pts[:, d].copy() for d in range(3)]
    stack = [(0, n, pts.min(axis=0), pts.max(axis=0))]
    while stack:
        first, last, mn, mx = stack.pop()
        count = last - first
        if count <= 7:
            continue
        dim = _arg_max3(mx - mn)
        left = count - count // 2
        keys = cols[dim]
        seg = perm[first:last]
        if count > small:
            q, _ = introselect_parallel(keys, left, seg)
        else:
            q, _ = introselect(keys, left, [int(v) for v in seg])
        perm[first:last] = q
        cut = keys[perm[first + left]]
        lmx, rmn = mx.copy(), mn.copy()
        lmx[dim] = cut
        rmn[dim] = cut
        stack.append((first + left, last, rmn, mx))
        stack.append((first, first + left, mn, lmx))
    return perm


def leaf_spans(n):
    """(first, count) of every leaf of the median-split recursion over n points, in leaf order"""
    out, stack = [], [(0, n)]
    while stack:
        first, count = stack.pop()
        if count <= 7:
            out.append((first, count))
            continue
        left = count - count // 2
        stack.append((first + left, count - left))
        stack.append((first, left))
    return out


def normals_from_perm(points, perm):
    """the leaf routine over the members in perm order, representative = first member: (points (M,3), normals (M,3),
    representatives (M,)) in ascending representative order, as CalculateNormals compacts them.  The sums are numpy's
    (equal to the reference's to rounding)."""
    pts = np.asarray(points, np.float64)
    reps, means, nrms = [], [], []
    for first, count in leaf_spans(len(pts)):
        d = pts[perm[first:first + count]]
        mean = d.sum(axis=0) / count
        e = d - mean
        C = e.T @ e
        if np.linalg.matrix_rank(C) + 1 < 3:
            continue
        try:
            nrm = np.linalg.solve(d.T @ d, d.sum(axis=0))
            nrm = nrm / np.linalg.norm(nrm)
        except np.linalg.LinAlgError:                   # M singular: the reference's inverse is not finite either
            nrm = np.full(3, np.nan)
        reps.append(int(perm[first]))
        means.append(mean)
        nrms.append(nrm)
    o = np.argsort(reps)
    return np.asarray(means)[o], np.asarray(nrms)[o], np.asarray(reps)[o]
