"""numpy model of the two device stages every matcher builds on: the k-d tree build (csrc/kdtree.cu kd_build and the
layouts its owners fill) and the stable LSD radix sort (csrc/radix_sort.cu).

TEST INFRASTRUCTURE ONLY.  The tree is libnabo's KDTREE_LINEAR_HEAP build (tests/pyref.py PyNabo restates it node by
node, recursively) with the project's tie rule, computed level by level for all nodes at once so that clouds of
millions of points take seconds:
  * widest axis of the node's implicit bounds, first strictly greater spread from axis 0 (spread 0 -> axis 0);
  * leftCount = count - count / 2; the cut is the RAW coordinate of the point at first + leftCount of the node's
    points ordered by (coordinate + 0.0, original index), so -0.0 and +0.0 are equal coordinates;
  * children of heap node h are 2h + 1 / 2h + 2; a node of <= bucket points is a leaf holding its ids ascending;
  * levels = kd_num_levels(n, bucket): halving with ceil until the largest node fits a bucket.
From that heap it derives what the owners store: the blocked node array (common.cuh blocked_index), the leaf order,
the compact search layout (KdCompact in csrc/kernels.h) and FloatTree's bucket points."""
from __future__ import annotations

import numpy as np

LEAF = 3


def num_levels(n, bucket):
    """kd_num_levels: all nodes of the returned level are leaves."""
    levels, c = 0, int(n)
    while c > bucket:
        c = (c + 1) // 2
        levels += 1
    return levels


def sub_capacity(bucket):
    """kd_sub_capacity: the largest segment kd_subtree_kernel finishes in one CTA."""
    return min(2048, 256 * bucket)


def blocked_index(h):
    """common.cuh blocked_index, vectorised: heap index -> slot of the 3-levels-per-128-byte-line node array."""
    h = np.asarray(h, dtype=np.int64)
    lvl = np.floor(np.log2(h + 1)).astype(np.int64)
    lvl += ((h + 1) >> (lvl + 1)) != 0                  # guard the float log2 at exact powers of two
    lvl -= ((h + 1) >> lvl) == 0
    j = h + 1 - (np.int64(1) << lvl)
    bl, sl = lvl // 3, lvl % 3
    base = ((np.int64(1) << (3 * bl)) - 1) // 7
    B = base + (j >> sl)
    p = (np.int64(1) << sl) - 1 + (j & ((np.int64(1) << sl) - 1))
    return B * 8 + p


def blocked_node_slots(levels):
    nbl = levels // 3 + 1
    return (((1 << (3 * nbl)) - 1) // 7) * 8


def sortable_key(v):
    """common.cuh sortable_key: float64 -> u64 whose unsigned order is the total order of the doubles."""
    u = np.ascontiguousarray(v, dtype=np.float64).view(np.uint64)
    return np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))


def float_key(v):
    """kd_keys_kernel's 32-bit key of a coordinate that is exactly a float."""
    u = np.ascontiguousarray(v, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u >> np.uint64(31), (~u) & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))


def tree_keys(coord, keys32=False):
    """kd_keys_kernel: per axis the key of coordinate + 0.0 (-0.0 becomes +0.0), (3, n) u64."""
    c = np.asarray(coord, dtype=np.float64).T + 0.0
    return np.stack([float_key(c[d]) if keys32 else sortable_key(c[d]) for d in range(3)])


def radix_sort(keys, vals, passes):
    """radix_sort_pairs_u64 on one array: stable order of the low 8 * passes key bits, whole words permuted."""
    keys = np.asarray(keys, dtype=np.uint64)
    mask = np.uint64(0xFFFFFFFFFFFFFFFF) if passes >= 8 else np.uint64((1 << (8 * passes)) - 1)
    perm = np.argsort(keys & mask, kind="stable")
    return keys[perm], np.asarray(vals)[perm]


class Tree:
    """The tree of an (n, 3) cloud.  Heap arrays of 2^(levels+1) - 1 entries: dim (0..2 inner, 3 leaf, -1 no node),
    cut (inner), first / count (leaves); leaf_order[n]."""

    def __init__(self, cloud, bucket=8):
        pts = np.ascontiguousarray(np.asarray(cloud, dtype=np.float64))
        n = pts.shape[0]
        assert n >= 1 and pts.ndim == 2 and pts.shape[1] == 3
        self.pts, self.n, self.bucket = pts, n, bucket
        self.levels = L = num_levels(n, bucket)
        total = (1 << (L + 1)) - 1
        self.dim = np.full(total, -1, np.int64)
        self.cut = np.zeros(total)
        self.first = np.zeros(total, np.int64)
        self.count = np.zeros(total, np.int64)
        # per axis the ids ordered by (coordinate + 0.0, id); every level keeps each node's range ordered so
        lists = [np.argsort(pts[:, d] + 0.0, kind="stable").astype(np.int64) for d in range(3)]
        # the nodes still to split: heap index, first, count, bounds (min[3], max[3])
        h = np.zeros(1, np.int64)
        f = np.zeros(1, np.int64)
        c = np.full(1, n, np.int64)
        lo = np.array([[pts[lists[d][0], d] for d in range(3)]])
        hi = np.array([[pts[lists[d][n - 1], d] for d in range(3)]])
        side = np.zeros(n, np.int8)
        while h.size:
            leaf = c <= bucket
            self.dim[h[leaf]] = LEAF
            self.first[h[leaf]], self.count[h[leaf]] = f[leaf], c[leaf]
            h, f, c, lo, hi = h[~leaf], f[~leaf], c[~leaf], lo[~leaf], hi[~leaf]
            if not h.size:
                break
            spread = hi - lo
            d = np.zeros(h.size, np.int64)
            best = np.zeros(h.size)
            for a in range(3):                            # argmax3: strict '>' from axis 0, starting at 0.0
                take = spread[:, a] > best
                d[take], best[take] = a, spread[take, a]
            left = c - c // 2
            stacked = np.stack(lists)
            pivot = stacked[d, f + left]
            cut = pts[pivot, d]
            self.dim[h], self.cut[h] = d, cut
            # positions inside the nodes of this level
            seg = np.repeat(np.arange(h.size), c)
            pos = f[seg] + (np.arange(seg.size) - np.repeat(np.cumsum(c) - c, c))
            rel = pos - f[seg]
            side[stacked[d[seg], pos]] = (rel >= left[seg]).astype(np.int8)
            for a in range(3):                            # stable partition of every list inside every node
                ids = lists[a][pos]
                isleft = side[ids] == 0
                excl = np.cumsum(isleft) - isleft
                start = np.repeat(np.cumsum(c) - c, c)
                rank_left = excl - excl[start]
                new = np.where(isleft, f[seg] + rank_left, f[seg] + left[seg] + (rel - rank_left))
                out = lists[a].copy()
                out[new] = ids
                lists[a] = out
            # children
            lo_l, hi_l, lo_r, hi_r = lo.copy(), hi.copy(), lo.copy(), hi.copy()
            r = np.arange(h.size)
            hi_l[r, d] = cut
            lo_r[r, d] = cut
            h = np.stack([2 * h + 1, 2 * h + 2], 1).ravel()
            f = np.stack([f, f + left], 1).ravel()
            c = np.stack([left, c // 2], 1).ravel()
            lo = np.stack([lo, lo_r], 1).reshape(-1, 3)
            hi = np.stack([hi_l, hi], 1).reshape(-1, 3)
        # leaves hold their ids ascending
        leaves = np.nonzero(self.dim == LEAF)[0]
        owner_first = np.empty(n, np.int64)             # position -> first position of its leaf
        for_pos = np.repeat(self.first[leaves], self.count[leaves])
        owner_first[for_pos + (np.arange(n) - np.repeat(np.cumsum(self.count[leaves]) - self.count[leaves],
                                                        self.count[leaves]))] = for_pos
        self.leaf_order = lists[0][np.lexsort((lists[0], owner_first))]
        self.leaves = leaves

    # ---- what the owners store -------------------------------------------------------------------------------------
    def exists(self):
        return self.dim >= 0

    def leaf_sets(self):
        """the id sets of the leaves, in heap order"""
        return [self.leaf_order[f:f + c] for f, c in zip(self.first[self.leaves], self.count[self.leaves])]

    def blocked_nodes(self):
        """-> (slots, records): the blocked slot of every existing node and its 16-byte KdNode as 2 u64 words
        (cut or {first | count << 32}, dim | pad << 32)."""
        h = np.nonzero(self.exists())[0]
        w0 = np.where(self.dim[h] == LEAF,
                      (self.first[h].astype(np.uint64) | (self.count[h].astype(np.uint64) << np.uint64(32))),
                      np.ascontiguousarray(self.cut[h]).view(np.uint64))
        w1 = self.dim[h].astype(np.uint64)
        return blocked_index(h), np.stack([w0, w1], 1)

    def compact(self, normals=None):
        """The KdCompact layout: heap nodes above the deepest level (mask of existing ones), cut / dim, node[h + 1]
        records (2 u64 words), padded buckets pb (8 << levels, 3, 8 per bucket -> flat), pid and pn."""
        L = self.levels
        top = (1 << L) - 1
        mask = self.dim[:top] >= 0
        dim = self.dim[:top].copy()
        cut = self.cut[:top].copy()
        node = np.zeros((top, 2), np.uint64)
        inner = dim < LEAF
        node[inner, 0] = np.ascontiguousarray(cut[inner]).view(np.uint64)
        node[:, 1] = np.where(dim < 0, 0, dim).astype(np.uint64)
        entries = 8 << L
        pb = np.full((1 << L, 3, 8), np.inf)
        pid = np.full(entries, -1, np.int64)
        pn = np.zeros((entries, 4))
        lvl = np.floor(np.log2(self.leaves + 1)).astype(np.int64)
        lvl += ((self.leaves + 1) >> (lvl + 1)) != 0
        lvl -= ((self.leaves + 1) >> lvl) == 0
        j = self.leaves + 1 - (np.int64(1) << lvl)
        slot = j << (L - lvl)                               # a leaf above the deepest level owns its left-most slot
        co = self.count[self.leaves]
        s = np.repeat(slot, co)                             # every point: its bucket slot and entry k
        k = np.arange(self.n) - np.repeat(np.cumsum(co) - co, co)
        ids = self.leaf_order[np.repeat(self.first[self.leaves], co) + k]
        for a in range(3):
            pb[s, a, k] = self.pts[ids, a]
        pid[8 * s + k] = ids
        if normals is not None:
            pn[8 * s + k, :3] = np.asarray(normals, dtype=np.float64)[ids]
        return {"mask": mask, "dim": dim, "cut": cut, "node": node, "pb": pb.reshape(-1), "pid": pid, "pn": pn}

    def bucket_points(self):
        """FloatTree's bpts: {x, y, z, id} of leaf_order[s] for every slot s"""
        return self.pts[self.leaf_order], self.leaf_order.copy()

    def global_levels(self):
        """kd_build's Lg: the levels split by the per-level kernels before kd_subtree_kernel takes over"""
        cap, lg, c = sub_capacity(self.bucket), 0, self.n
        while lg < self.levels and c > cap:
            c = (c + 1) // 2
            lg += 1
        return lg


def heap_from_pynabo(nodes):
    """pyref.PyNabo's pre-order node list -> {heap index: node}"""
    out, stack = {}, [(0, 0)]
    while stack:
        pos, h = stack.pop()
        dim, a, rc = nodes[pos]
        out[h] = nodes[pos]
        if dim != LEAF:
            stack.append((pos + 1, 2 * h + 1))
            stack.append((rc, 2 * h + 2))
    return out
