"""The sending end of Node.sync restated in index space, for tests: the requester's summary (swirld.py:125-126) and
ask_sync's reply (swirld.py:154-161, utils.py:24-34) as the BFS the reference runs, and the closed form the engine's
kernels select (swirld_sync.cuh).  Events are a view's arrival indices; a view is a Trace (p0, p1, creator) with its
can_see rows and heights.  The reference is not imported."""
from collections import deque

import numpy as np

from swirld_b200 import traces


class View:
    """One node-view's graph: columns, can_see rows and heights, over its first n events."""

    def __init__(self, tr, n=None):
        n = tr.N if n is None else n
        self.tr = tr.slice(0, n) if n < tr.N else tr
        self.M = tr.M
        self.p0, self.p1, self.creator = self.tr.p0, self.tr.p1, self.tr.creator
        self.row = traces.can_see_rows(self.tr)
        self.height = traces.heights(self.tr)


def summary(view, head):
    """{c: height[can_see[head][c]]} as M entries, -1 where head sees none of c's events."""
    r = view.row[head]
    return np.where(r >= 0, view.height[np.maximum(r, 0)], -1).astype(np.int32)


def bfs_reply(view, head, S):
    """ask_sync: bfs((head,), parents p with creator not in S or height[p] > S[creator p]), as a sorted index array."""
    keep = lambda p: S[view.creator[p]] < 0 or view.height[p] > S[view.creator[p]]
    seen, q = {head}, deque([head])
    while q:
        u = q.popleft()
        if view.p0[u] < 0:
            continue
        for p in (int(view.p0[u]), int(view.p1[u])):
            if p not in seen and keep(p):
                seen.add(p)
                q.append(p)
    return np.array(sorted(seen), np.int32)


def closed_reply(view, head, S):
    """{head} u {x < head : x <= row(head)[creator x] and (S[creator x] = -1 or height[x] > S[creator x])}."""
    x = np.arange(head, dtype=np.int64)
    c = view.creator[:head]
    s = np.asarray(S)[c]
    pick = (x <= view.row[head][c]) & ((s < 0) | (view.height[:head] > s))
    return np.append(np.flatnonzero(pick), head).astype(np.int32)
