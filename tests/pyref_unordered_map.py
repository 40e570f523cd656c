"""An independent Python restatement of how libstdc++'s std::unordered_map (unique keys, insert only) orders its
nodes: one singly linked list in which every bucket's nodes are one contiguous run, each bucket remembering the node
before its run.  An insert into a non-empty bucket goes to the head of its run, one into an empty bucket to the front
of the list; a rehash walks the old list front to back and puts each node at the front of the new list if its new
bucket is still empty, else at the head of that bucket's run.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import numpy as np

FRONT = -1     # "before the first node": the list's own head pointer


def iteration_order(hashes, bucket_counts):
    """hashes (by insertion rank) and bucket_count() after each insert -> the ranks in iteration order"""
    h = [int(x) for x in np.asarray(hashes, np.uint64)]
    counts = [int(x) for x in np.asarray(bucket_counts, np.uint64)]
    m = len(h)
    nxt = [-1] * m
    head = -1
    n_buckets = 1
    before = {}                       # bucket -> the node before its run (FRONT for the list's head)

    def next_of(node):
        return head if node == FRONT else nxt[node]

    for t in range(m):
        if counts[t] != n_buckets:    # rehash, then insert
            n_buckets = counts[t]
            p, head, before = head, -1, {}
            front_bucket = None       # the bucket of the list's first node
            while p != -1:
                following = nxt[p]
                b = h[p] % n_buckets
                if b not in before:
                    nxt[p], head = head, p
                    before[b] = FRONT
                    if nxt[p] != -1:
                        before[front_bucket] = p
                    front_bucket = b
                else:
                    prev = before[b]
                    nxt[p] = next_of(prev)
                    if prev == FRONT:
                        head = p
                    else:
                        nxt[prev] = p
                p = following
        b = h[t] % n_buckets
        if b in before:
            prev = before[b]
            nxt[t] = next_of(prev)
            if prev == FRONT:
                head = t
            else:
                nxt[prev] = t
        else:
            nxt[t] = head
            head = t
            if nxt[t] != -1:
                before[h[nxt[t]] % n_buckets] = t
            before[b] = FRONT
    out = []
    p = head
    while p != -1:
        out.append(p)
        p = nxt[p]
    return np.asarray(out, np.int64)
