"""A CPU model of the k-NN kernel of staticmapping_b200/csrc/knn.cu: the 1-NN kernels' search state (level masks, see
tests/gpu_knn_mask_model.py) with a sorted k-entry list for the head, maxRadius and self-match exclusion.

TEST INFRASTRUCTURE ONLY.  What it restates on top of GpuKnnMaskModel (tree, padded buckets, replay, descent):
  scan_bucket_k   the 8 entries of a padded bucket in order; an entry enters the list iff d2 <= r^2, d2 < head and
                  (ALLOW_SELF_MATCH or d2 > DBL_EPSILON), after every entry of equal distance; head = the k-th entry
  root mask       a path level is pending iff off^2 <= r^2 and off^2 * (1 + eps)^2 < head after the first bucket
  far visits      knn_pop as before (deepest pending level, rd replayed, re-tested against the head of the moment);
                  a popped far side with rd > r^2 is dropped before its descent
tests/test_knn_oracle.py checks it against the oracle and against the plain recursion of tests/pyref_knn.py.
"""
from __future__ import annotations

import sys

import numpy as np

from gpu_knn_mask_model import GpuKnnMaskModel
from gpu_knn_model import INF

DBL_EPSILON = sys.float_info.epsilon


class GpuKnnKModel(GpuKnnMaskModel):
    def _scan(self, bucket, q, state):
        base = bucket * 8
        lst, k = state["list"], state["k"]
        for c in range(8):
            p = self.pb[base + c]
            dx, dy, dz = q[0] - p[0], q[1] - p[1], q[2] - p[2]
            with np.errstate(invalid="ignore", over="ignore"):
                d = float((dx * dx + dy * dy) + dz * dz)
            if d <= state["r2"] and d < state["head"] and (state["self"] or d > DBL_EPSILON):
                j = k - 1
                while j > 0 and not (lst[j - 1][0] <= d):
                    lst[j] = lst[j - 1]
                    j -= 1
                lst[j] = (d, base + c)
                state["head"] = lst[k - 1][0]
        state["visits"] += 1

    def _root_visit(self, q, me2, state):
        state["head"] = INF
        h = level = 0
        while level < self.levels:
            cd = self.dim[h]
            if cd == 3:
                break
            h = 2 * h + 1 + (1 if q[cd] > self.cut[h] else 0)
            level += 1
        self._scan((h + 1 - (1 << level)) << (self.levels - level), q, state)
        hp1, mask = h + 1, 0
        for a in range(level):
            n = (hp1 >> (level - a)) - 1
            off = q[self.dim[n]] - self.cut[n]
            rd = off * off
            if rd <= state["r2"] and rd * me2 < state["head"]:
                mask |= 1 << a
        return hp1, level, mask

    def _far_visits(self, q, me2, w, state):
        while True:
            go = self._pop(q, me2, w, state)
            if go is None:
                return
            if not go[1] <= state["r2"]:
                continue
            self._descend(q, me2, *go, w, state)

    def knn(self, query, k, epsilon=0.0, max_radius=INF, flags=1):
        Q = np.asarray(query, dtype=np.float64).reshape(-1, 3)
        me2 = (1.0 + epsilon) * (1.0 + epsilon)
        ids = np.full((Q.shape[0], k), -1, dtype=np.int32)
        d2 = np.full((Q.shape[0], k), INF)
        for j in range(Q.shape[0]):
            q = (float(Q[j, 0]), float(Q[j, 1]), float(Q[j, 2]))
            st = {"head": INF, "visits": 0, "k": k, "list": [(INF, -1)] * k, "r2": max_radius * max_radius,
                  "self": bool(flags & 1)}
            hp1, ll, mask = self._root_visit(q, me2, st)
            self._far_visits(q, me2, self._search_state(q, hp1, ll, mask), st)
            for i, (d, e) in enumerate(st["list"]):
                ids[j, i] = self.pid[e] if e >= 0 else -1
                d2[j, i] = d
        return ids, d2
