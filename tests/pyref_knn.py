"""Second, independent restatement of libnabo's k-NN search (KDTREE_LINEAR_HEAP) in pure Python, on the tree of
tests/pyref.py's PyNabo.  TEST INFRASTRUCTURE ONLY: written from the published libnabo 1.0.7 algorithm, not from
tests/cpp/knn_oracle.cc, and compared with it in tests/test_knn_oracle.py.  Python floats are IEEE doubles without
contraction, so ids and squared distances are expected to agree bit for bit, order included.

  heap      IndexHeapBruteForceVector: k entries (-1, +inf), sorted ascending, the head is the last one; replaceHead
            moves every entry whose value is STRICTLY greater one place back, so a new entry lands after its equals
  leaf      dist <= maxRadius^2 and dist < head and (ALLOW_SELF_MATCH or dist > DBL_EPSILON)
  inner     near child, then the far child iff rd <= maxRadius^2 and rd * (1 + eps)^2 < head
"""
from __future__ import annotations

import sys

import numpy as np

from pyref import INF, PyNabo

DBL_EPSILON = sys.float_info.epsilon
ALLOW_SELF_MATCH = 1


class PyNaboK(PyNabo):
    def knn(self, query, k, epsilon=0.0, max_radius=INF, flags=ALLOW_SELF_MATCH):
        """-> (ids int32 (nq, k), -1 = none; squared distances f64 (nq, k), +inf = none)"""
        q_all = np.asarray(query, dtype=np.float64).reshape(-1, 3)
        ids = np.full((q_all.shape[0], k), -1, dtype=np.int32)
        d2 = np.full((q_all.shape[0], k), INF)
        if not self.nodes:
            return ids, d2
        me2 = (1.0 + epsilon) * (1.0 + epsilon)
        r2 = max_radius * max_radius
        allow_self = bool(flags & ALLOW_SELF_MATCH)
        for j in range(q_all.shape[0]):
            q = (float(q_all[j, 0]), float(q_all[j, 1]), float(q_all[j, 2]))
            heap = [[INF, -1] for _ in range(k)]
            self._recurse_k(q, 0, 0.0, [0.0, 0.0, 0.0], me2, r2, allow_self, heap)
            for i, (v, index) in enumerate(heap):
                ids[j, i], d2[j, i] = index, v
        return ids, d2

    def _recurse_k(self, q, n, rd, off, me2, r2, allow_self, heap):
        dim, a, right_child = self.nodes[n]
        if dim == 3:
            for index in a:
                p = self.pts[index]
                dist = 0.0
                for r in range(3):
                    diff = q[r] - p[r]
                    dist += diff * diff
                if dist <= r2 and dist < heap[-1][0] and (allow_self or dist > DBL_EPSILON):
                    i = len(heap) - 1
                    while i > 0 and heap[i - 1][0] > dist:
                        heap[i] = heap[i - 1]
                        i -= 1
                    heap[i] = [dist, index]
            return
        new_off = q[dim] - a
        old_off = off[dim]
        near, far = (right_child, n + 1) if new_off > 0.0 else (n + 1, right_child)
        self._recurse_k(q, near, rd, off, me2, r2, allow_self, heap)
        rd = rd + (-(old_off * old_off) + new_off * new_off)
        if rd <= r2 and rd * me2 < heap[-1][0]:
            off[dim] = new_off
            self._recurse_k(q, far, rd, off, me2, r2, allow_self, heap)
            off[dim] = old_off
