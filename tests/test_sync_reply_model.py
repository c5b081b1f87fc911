"""The closed form of ask_sync's reply (swirld_sync.cuh) against the BFS the reference runs (tests/sync_model.py), on
the CPU: for node-views of G1, G2 (stale other-parents), a partition that splits and heals, and a late-joining member,
every responder view answers requester views at every turn.  A turn is a point of the gossip's source; each view is
then its prefix up to its last own event before that point, with that event as its head; every pair of views, the
empty summary too, at every turn (3 turns above 16 members, 6 below).  Also: an empty summary, a
requester that knows more of some member than the responder, and one summary no view of the gossip could send, where
the two differ -- the precondition the header states."""
import numpy as np
import pytest

import sync_model as sm
from swirld_b200 import traces

CASES = {
    "g1_m4": lambda: traces.gossip(4, 300, seed=11),
    "g1_m16": lambda: traces.gossip(16, 900, seed=12),
    "g2_m16": lambda: traces.adversarial(16, 900, seed=13, p_stale=0.6),
    "partition_m16": lambda: traces.partition(16, 1200, seed=14, start=200, end=800),
    "late_m16": lambda: traces.late_joiner(16, 1000, join_at=500, seed=15),
    "g1_m64": lambda: traces.gossip(64, 2000, seed=16),
    "g2_m64": lambda: traces.adversarial(64, 2000, seed=17, p_stale=0.5),
    "g1_m97": lambda: traces.gossip(97, 2500, seed=18),
}
TURNS = 6


def _views_at(base, turns):
    """Per turn, per member X: (View of X's prefix, its head), or None before X's first event."""
    out = [[None] * base.M for _ in turns]
    for X, (tr, sizes) in enumerate(traces.node_views(base)):
        chain = np.flatnonzero(base.creator == X)
        ends = np.cumsum(sizes)
        full = sm.View(tr)
        for k, T in enumerate(turns):
            j = int(np.searchsorted(chain, T))          # X's own events before T
            if j:
                out[k][X] = (full, int(ends[j - 1]) - 1)
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_closed_form_equals_bfs(name):
    base = CASES[name]()
    nt = TURNS if base.M <= 16 else 3
    turns = [int(base.N * (k + 1) / nt) for k in range(nt)]
    ahead = 0
    for per in _views_at(base, turns):
        live = [x for x in per if x is not None]
        for u, x in enumerate(per):
            if x is None:
                continue
            vu, hu = x
            summaries = [sm.summary(vw, hw) for vw, hw in live] + [np.full(base.M, -1, np.int32)]
            mine = sm.summary(vu, hu)
            for S in summaries:
                ahead += bool((S > mine).any())
                got, exp = sm.closed_reply(vu, hu, S), sm.bfs_reply(vu, hu, S)
                assert np.array_equal(got, exp), "%s: responder %d head %d" % (name, u, hu)
    assert ahead > 0, "no requester knew more of some member than its responder"


def test_empty_summary_is_every_ancestor():
    base = traces.gossip(8, 400, seed=3)
    v = sm.View(base)
    for head in (0, 7, 150, 399):
        got = sm.closed_reply(v, head, np.full(8, -1, np.int32))
        anc = np.flatnonzero(v.row[head][v.creator[:head + 1]] >= np.arange(head + 1))
        assert np.array_equal(got, anc)
        assert np.array_equal(got, sm.bfs_reply(v, head, np.full(8, -1, np.int32)))


def test_head_is_sent_even_when_the_requester_has_it():
    v = sm.View(traces.gossip(4, 200, seed=4))
    head = 150
    S = sm.summary(v, head)
    assert np.array_equal(sm.closed_reply(v, head, S), [head])
    assert np.array_equal(sm.bfs_reply(v, head, S), [head])


def test_inconsistent_summary_differs():
    """Members A, B, C: roots a0, b0, c0; b1 = (b0, a0); head c1 = (c0, b1).  A summary that holds b1 but not a0, which
    b1 sees, comes from no view of this gossip: the BFS stops at b1 and never reaches a0; the closed form sends a0."""
    tr = traces.Trace(3, np.array([-1, -1, -1, 1, 2], np.int32), np.array([-1, -1, -1, 0, 3], np.int32),
                      np.array([0, 1, 2, 1, 2], np.int32), np.arange(5, dtype=np.float64), np.zeros((5, 64), np.uint8), "abc")
    v = sm.View(tr)
    S = np.array([-1, int(v.height[3]), -1], np.int32)
    assert sm.bfs_reply(v, 4, S).tolist() == [2, 4]
    assert sm.closed_reply(v, 4, S).tolist() == [0, 2, 4]
