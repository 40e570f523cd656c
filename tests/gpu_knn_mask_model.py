"""A CPU model of the k-NN kernels' search state as knn_smem.cuh runs it now: level masks instead of a stack.

TEST INFRASTRUCTURE ONLY.  tests/gpu_knn_model.py restates the tree, the bucket layout and the scan of the kernels,
and the earlier search bookkeeping (float lower-bound mask of the root path, an explicit stack of far children).
This file keeps its tree, layout and scan (GpuKnnMaskModel derives from GpuKnnModel) and restates the search the
kernels now make.  The root visit's candidate mask is an exact test of every path level after the first bucket.
There is no stack: a query's pending far sides are the siblings of its current path's nodes, at most one per level,
so the whole state is the leaf (hp1, ll: the path), a `pending` bit per level (set when a far child passes its test
during a descent) and a `turns` bit per level (where the path went to a far side).  A pop takes the deepest pending
level, replays rd and off[] of its far child exactly over the turns above it (the same dsub / dmul / dadd sequence
the recursion made), and re-tests it with the head of that moment.  tests/test_search_state_model.py checks it
against libnabo's plain recursion (tests/pyref.py PyNabo) and the oracle, and checks every replayed rd against the
value the old stack held.

Mirrors: knn_root_visit, knn_pop (with its replay), knn_descend, knn1_smem and knn_far_phase of knn_smem.cuh.
"""
from __future__ import annotations

import numpy as np

from gpu_knn_model import INF, GpuKnnModel


class GpuKnnMaskModel(GpuKnnModel):
    def __init__(self, cloud, bucket=8):
        super().__init__(cloud, bucket)
        self.replay_log = None      # a list: every pop appends (replayed rd, rd the old stack held, a turn above?)

    # ---- knn_root_visit: descent, first bucket, then the mask of the path levels whose far side passes an EXACT
    # test with the head that bucket left (path node of level a: (hp1 >> (ll - a)) - 1; rd = 0 and off = 0 along
    # the root path, so rd_new(a) = 0 + (-(0*0) + off^2) = off^2 exactly)
    def _root_visit(self, q, me2, state):
        state["head"], state["best"] = INF, -1
        h = level = 0
        while level < self.levels:
            cd = self.dim[h]
            if cd == 3:
                break
            h = 2 * h + 1 + (1 if q[cd] - self.cut[h] > 0.0 else 0)
            level += 1
        self._scan((h + 1 - (1 << level)) << (self.levels - level), q, state)
        hp1, mask = h + 1, 0
        for a in range(level):
            n = (hp1 >> (level - a)) - 1
            off = q[self.dim[n]] - self.cut[n]
            if (off * off) * me2 < state["head"]:
                mask |= 1 << a
        return hp1, level, mask

    # ---- knn_replay: rd and off[] of the far child of path level j, recomputed along the path.  rd and off change
    # only where the path went to a far side (the turns), in the order the recursion made those changes.
    def _replay(self, q, hp1, ll, turns, j):
        rd, off = 0.0, [0.0, 0.0, 0.0]
        for a in range(j + 1):
            if a == j or turns >> a & 1:
                n = (hp1 >> (ll - a)) - 1
                cd = self.dim[n]
                old_off, new_off = off[cd], q[cd] - self.cut[n]
                rd = rd + (-(old_off * old_off) + new_off * new_off)
                off[cd] = new_off
        return rd, off

    # ---- knn_pop: the deepest pending level, its far child's rd replayed and re-tested with the head of that moment.
    # The pending far sides of a query are the siblings of its path's nodes, at most one per level: a descent sets bits
    # only below the level it starts from, and every pending bit left is above it.  So the recursion's stack is the
    # level mask, its top the deepest bit.  w: the query's search state (hp1, ll, pending, turns), updated in place;
    # returns (h, rd, off) of the subtree to visit next, or None when nothing is left.
    def _pop(self, q, me2, w, state):
        while w["pending"]:
            j = w["pending"].bit_length() - 1
            w["pending"] &= ~(1 << j)
            rd, off = self._replay(q, w["hp1"], w["ll"], w["turns"], j)
            if self.replay_log is not None:
                self.replay_log.append((rd, w["pushed"][j], w["turns"] & ((1 << j) - 1) != 0))
            if rd * me2 < state["head"]:
                w["turns"] = (w["turns"] & ((1 << j) - 1)) | (1 << j)
                return ((w["hp1"] >> (w["ll"] - j - 1)) ^ 1) - 1, rd, off
        return None

    # ---- knn_descend: near child first down to a leaf; a far child that passes rd_new*(1+eps)^2 < head now gets
    # the pending bit of its parent's level (re-tested when popped, which is when the recursion tests it)
    def _descend(self, q, me2, h, rd, off, w, state):
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
                w["pending"] |= 1 << level
                w["pushed"][level] = rd_new            # what the old stack entry held: checked against the replay
            h = 2 * h + 1 + right
            level += 1
        w["hp1"], w["ll"] = h + 1, level
        self._scan((h + 1 - (1 << level)) << (self.levels - level), q, state)

    def _search_state(self, q, hp1, ll, mask):
        """a parked query: its leaf, the candidate mask as pending bits, no turns.  `pushed` keeps, per level, the rd
        the old explicit stack held for it (for the root path, the off^2 the old kernel computed when testing it)."""
        pushed = {}
        for a in range(ll):
            if mask >> a & 1:
                n = (hp1 >> (ll - a)) - 1
                off = q[self.dim[n]] - self.cut[n]
                pushed[a] = off * off
        return {"hp1": hp1, "ll": ll, "pending": mask, "turns": 0, "pushed": pushed}

    def _far_visits(self, q, me2, w, state):
        while True:
            go = self._pop(q, me2, w, state)
            if go is None:
                return
            self._descend(q, me2, *go, w, state)

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
            self._far_visits(q, me2, self._search_state(q, hp1, ll, mask), st)
            ids[j] = self.pid[st["best"]] if st["best"] >= 0 else -1
            d2[j] = st["head"]
            if visits is not None:
                visits.append(st["visits"])
        return ids, d2

    def knn1_batched(self, query, epsilon=3.16, lanes=32):
        """knn_batch_cta / knn_far_phase: root visits first, queries with a non-empty mask are parked; then `lanes`
        lanes work through the list, ONE bucket visit per busy lane and pass (the deepest pending level of the lane's
        query, popped as knn1 pops it), a finished lane takes the next item with no turns."""
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
                    lane[k] = (j, q, self._search_state(q, hp1, ll, mask))
            if all(x is None for x in lane):
                break
            for k in range(lanes):
                if lane[k] is None:
                    continue
                j, q, w = lane[k]
                st = states[j]
                go = self._pop(q, me2, w, st)             # the same pop as knn1: deepest pending level, replayed
                if go is None:
                    ids[j] = self.pid[st["best"]] if st["best"] >= 0 else -1
                    d2[j] = st["head"]
                    lane[k] = None
                    continue
                self._descend(q, me2, *go, w, st)
        return ids, d2
