"""A CPU model of the GPU kernels' k-NN FORMULATION (staticmapping_b200/csrc/kdtree.cu, knn_smem.cuh).

TEST INFRASTRUCTURE ONLY.  The CUDA search is not a recursion: it is an implicit-heap tree (children of h are
2h+1 / 2h+2, leaves carry no payload, a leaf's bucket is addressed from its heap index), a root visit that keeps
FLOAT lower bounds of the plane distances of its path and turns them into a candidate mask, far visits taken
deepest level first with an exact re-test, an explicit stack whose entries are tested when pushed and re-tested
when popped, and a bucket scan that is a tournament on bit patterns.  DESIGN.md section 2 claims that all of this
visits the same buckets in the same order and makes the same comparisons as libnabo's recurseKnn, hence
bit-identical results.  This file restates that formulation step by step in Python so the claim can be checked
on a CPU, every round, against the plain recursion (tests/pyref.py PyNabo) — the GPU tests check the kernels
against the oracle, this checks the ALGORITHM the kernels implement.

Mirrors: kd_num_levels / locate_node (kdtree.cu:26-34), kd_node_kernel's split rule, kd_compact_buckets_kernel (padded
x[8] y[8] z[8] buckets, +inf padding, members in ascending original index), knn_root_visit, knn1_smem,
visit_subtree, knn_far_phase and scan_bucket of knn_smem.cuh.
"""
from __future__ import annotations

import struct

import numpy as np

INF = float("inf")


def _bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _float_rd(x: float) -> float:
    """__double2float_rd: the largest float <= x (as a Python float)."""
    f = np.float32(x)
    if float(f) > x or (np.isinf(f) and x != INF):
        f = np.nextafter(f, np.float32(-np.inf))
    return float(f)


class GpuKnnModel:
    def __init__(self, cloud, bucket=8):
        self.pts = np.asarray(cloud, dtype=np.float64)
        n = self.pts.shape[0]
        self.bucket = bucket
        # kd_num_levels: depth of the deepest leaf of the shape recursion (count <= bucket stops)
        levels, count = 0, n
        while count > bucket:
            count = count - (count >> 1)          # the LEFT child is the larger one
            levels += 1
        self.levels = levels
        self.cut = {}                              # heap index -> cut value (inner nodes)
        self.dim = {}                              # heap index -> 0..2, 3 = leaf
        self.pb = np.full(((1 << levels) * 8, 3), INF)          # padded buckets of the deepest level's slots
        self.pid = np.full((1 << levels) * 8, -1, dtype=np.int64)
        rows = [tuple(float(v) for v in p) for p in self.pts]
        mn = [float(v) for v in self.pts.min(axis=0)] if n else [0.0] * 3
        mx = [float(v) for v in self.pts.max(axis=0)] if n else [0.0] * 3
        self._build(rows, list(range(n)), 0, 0, mn, mx)

    def _build(self, rows, idx, h, level, mn, mx):
        if len(idx) <= self.bucket:
            self.dim[h] = 3
            slot = ((h + 1 - (1 << level)) << (self.levels - level)) * 8
            for k, i in enumerate(sorted(idx)):    # members in ascending original index
                self.pb[slot + k] = self.pts[i]
                self.pid[slot + k] = i
            return
        ext = [mx[d] - mn[d] for d in range(3)]
        dim, mv = 0, 0.0                           # argmax3: first strictly greater wins, from 0
        for d in range(3):
            if ext[d] > mv:
                mv, dim = ext[d], d
        order = sorted(idx, key=lambda i: (rows[i][dim], i))     # total order (coordinate, index)
        right = len(idx) >> 1
        left = len(idx) - right
        cut = rows[order[left]][dim]
        self.cut[h], self.dim[h] = cut, dim
        lmx = list(mx); lmx[dim] = cut
        rmn = list(mn); rmn[dim] = cut
        self._build(rows, order[:left], 2 * h + 1, level + 1, mn, lmx)
        self._build(rows, order[left:], 2 * h + 2, level + 1, rmn, mx)

    # ---- scan_bucket: two tournaments of four on the bit patterns, lower index keeps a tie, strict '<' vs head
    def _scan(self, bucket, q, state):
        base = bucket * 8
        for half in range(2):
            keys = []
            for k in range(4):
                p = self.pb[base + 4 * half + k]
                dx, dy, dz = q[0] - p[0], q[1] - p[1], q[2] - p[2]
                with np.errstate(invalid="ignore", over="ignore"):
                    d = (dx * dx + dy * dy) + dz * dz
                keys.append(_bits(float(d)))
            k0, a0, k2, a2 = keys[0], 0, keys[2], 2
            if keys[1] < k0:
                k0, a0 = keys[1], 1
            if keys[3] < k2:
                k2, a2 = keys[3], 3
            if k2 < k0:
                k0, a0 = k2, a2
            if k0 < _bits(state["head"]):
                state["head"] = struct.unpack("<d", struct.pack("<Q", k0))[0]
                state["best"] = base + 4 * half + a0
        state["visits"] += 1

    # ---- knn_root_visit: descent, first bucket, mask of path levels from FLOAT lower bounds
    def _root_visit(self, q, me2, state):
        state["head"], state["best"] = INF, -1
        lb = []
        h = level = 0
        while level < self.levels:
            cd = self.dim[h]
            if cd == 3:
                break
            off = q[cd] - self.cut[h]
            lb.append(_float_rd(off * off))
            h = 2 * h + 1 + (1 if off > 0.0 else 0)
            level += 1
        self._scan((h + 1 - (1 << level)) << (self.levels - level), q, state)
        mask = 0
        for a in range(level):
            if lb[a] * me2 < state["head"]:
                mask |= 1 << a
        return h + 1, level, mask

    # ---- visit_subtree: near child first, far child pushed if it passes NOW, re-tested when popped
    def _visit_subtree(self, q, me2, h, rd, off, state):
        stack = []
        while True:
            level = (h + 1).bit_length() - 1
            while level < self.levels:
                cd = self.dim[h]
                if cd == 3:
                    break
                cut = self.cut[h]
                old_off = off[cd]
                new_off = q[cd] - cut
                rd_new = rd + (-(old_off * old_off) + new_off * new_off)
                right = 1 if q[cd] > cut else 0
                if rd_new * me2 < state["head"]:
                    o = list(off); o[cd] = new_off
                    stack.append((rd_new, o, 2 * h + 2 - right))
                h = 2 * h + 1 + right
                level += 1
            self._scan((h + 1 - (1 << level)) << (self.levels - level), q, state)
            found = False
            while stack:
                rd_e, o_e, h_e = stack.pop()
                if rd_e * me2 < state["head"]:
                    h, rd, off = h_e, rd_e, o_e
                    found = True
                    break
            if not found:
                return

    def _far_levels(self, q, me2, hp1, ll, mask, state):
        """the levels of the mask deepest first, each re-tested exactly with the head of that moment"""
        while mask:
            a = mask.bit_length() - 1
            mask &= ~(1 << a)
            n = (hp1 >> (ll - a)) - 1
            off_v = q[self.dim[n]] - self.cut[n]
            rd_new = off_v * off_v
            if rd_new * me2 < state["head"]:
                off = [0.0, 0.0, 0.0]
                off[self.dim[n]] = off_v
                near_p1 = hp1 >> (ll - a - 1)
                self._visit_subtree(q, me2, (near_p1 ^ 1) - 1, rd_new, off, state)

    def knn1(self, query, epsilon=3.16, visits=None):
        """knn1_smem per query -> (original ids, squared distances)."""
        Q = np.asarray(query, dtype=np.float64)
        me2 = (1.0 + epsilon) * (1.0 + epsilon)
        ids = np.full(Q.shape[0], -1, dtype=np.int32)
        d2 = np.full(Q.shape[0], INF)
        for j in range(Q.shape[0]):
            q = (float(Q[j, 0]), float(Q[j, 1]), float(Q[j, 2]))
            st = {"head": INF, "best": -1, "visits": 0}
            hp1, ll, mask = self._root_visit(q, me2, st)
            self._far_levels(q, me2, hp1, ll, mask, st)
            ids[j] = self.pid[st["best"]] if st["best"] >= 0 else -1
            d2[j] = st["head"]
            if visits is not None:
                visits.append(st["visits"])
        return ids, d2

    def knn1_batched(self, query, epsilon=3.16, lanes=32):
        """knn_batch_cta / knn_far_phase: root visits first, queries with a non-empty mask are parked; then `lanes`
        lanes work through the list, ONE bucket visit per busy lane and pass (nested far children popped from the
        lane's stack first, else the next level of the mask), a finished lane takes the next item."""
        Q = np.asarray(query, dtype=np.float64)
        me2 = (1.0 + epsilon) * (1.0 + epsilon)
        ids = np.full(Q.shape[0], -1, dtype=np.int32)
        d2 = np.full(Q.shape[0], INF)
        items, states = [], {}
        for j in range(Q.shape[0]):
            q = (float(Q[j, 0]), float(Q[j, 1]), float(Q[j, 2]))
            st = {"head": INF, "best": -1, "visits": 0}
            hp1, ll, mask = self._root_visit(q, me2, st)
            if mask == 0:
                ids[j] = self.pid[st["best"]] if st["best"] >= 0 else -1
                d2[j] = st["head"]
            else:
                states[j] = st
                items.append((j, q, hp1, ll, mask))
        lane = [None] * lanes
        nxt = 0
        while True:
            for k in range(lanes):                       # idle lanes take the next items in order
                if lane[k] is None and nxt < len(items):
                    j, q, hp1, ll, mask = items[nxt]
                    nxt += 1
                    lane[k] = {"j": j, "q": q, "hp1": hp1, "ll": ll, "mask": mask, "stack": []}
            if all(x is None for x in lane):
                break
            for k in range(lanes):
                w = lane[k]
                if w is None:
                    continue
                st, q = states[w["j"]], w["q"]
                go = None
                while w["stack"]:                         # nested far children first
                    rd_e, o_e, h_e = w["stack"].pop()
                    if rd_e * me2 < st["head"]:
                        go = (h_e, rd_e, o_e)
                        break
                while go is None and w["mask"]:           # then the root path, deepest level first
                    a = w["mask"].bit_length() - 1
                    w["mask"] &= ~(1 << a)
                    n = (w["hp1"] >> (w["ll"] - a)) - 1
                    off_v = q[self.dim[n]] - self.cut[n]
                    rd_new = off_v * off_v
                    if rd_new * me2 < st["head"]:
                        off = [0.0, 0.0, 0.0]
                        off[self.dim[n]] = off_v
                        go = (((w["hp1"] >> (w["ll"] - a - 1)) ^ 1) - 1, rd_new, off)
                if go is None:
                    ids[w["j"]] = self.pid[st["best"]] if st["best"] >= 0 else -1
                    d2[w["j"]] = st["head"]
                    lane[k] = None
                    continue
                h, rd, off = go
                level = (h + 1).bit_length() - 1
                while level < self.levels:
                    cd = self.dim[h]
                    if cd == 3:
                        break
                    cut = self.cut[h]
                    old_off = off[cd]
                    new_off = q[cd] - cut
                    rd_new = rd + (-(old_off * old_off) + new_off * new_off)
                    right = 1 if q[cd] > cut else 0
                    if rd_new * me2 < st["head"]:
                        o = list(off); o[cd] = new_off
                        w["stack"].append((rd_new, o, 2 * h + 2 - right))
                    h = 2 * h + 1 + right
                    level += 1
                self._scan((h + 1 - (1 << level)) << (self.levels - level), q, st)
        return ids, d2
