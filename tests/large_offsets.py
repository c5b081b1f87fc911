"""Helpers for the tests past 2^31 table elements (tests/test_gpu_large_offsets.py).

Every kernel and host copy of the engine computes its own offsets into the can_see table (`row`, N x M int32) and the
signature column (64 bytes per event).  A missing size_t cast in any of them corrupts results only beyond 2^31
elements, so these helpers check an engine that large without holding its table twice on the host: every comparison
walks the table in chunks, and the restatements below fetch only the rows they read.

Where no oracle can run (M = 1024), the reference is restated here from its own per-event rules, in exact integers:
- can_see (swirld.py:203-205, 220): per column the higher of the parents' entries by height (`higher`, swirld.py:183-184,
  on a fork-free graph), the event itself in its own column;
- round and witness flag (swirld.py:200-222): `hits` counted from pre(h) -- the parents' merged row before the event
  enters its own column -- the rows of the events pre(h) names and the rounds of earlier events, then the two
  `> min_s` tests; a witness is an event whose round exceeds its self-parent's.
tests/test_large_offsets_model.py checks both against the oracle on small traces, and that every check here fails on a
copy of the oracle's output with one element changed.

`get_rows(first, n)` is any source of can_see rows: Engine.can_see, Oracle.can_see, or a slice of an array in memory."""
from types import SimpleNamespace

import numpy as np

import order_meta
import sync_model as sm

GAP = 4096          # gather_rows fetches two wanted rows in one range when they are at most this many rows apart


def first_mismatch(name, exp, got, offset=0):
    """None if exp and got are equal (shape and every element), else a message naming the first differing element;
    the leading index is shifted by offset (the chunk's first event)."""
    exp, got = np.asarray(exp), np.asarray(got)
    if exp.shape != got.shape:
        return "%s: shape %s, expected %s" % (name, got.shape, exp.shape)
    if np.array_equal(exp, got):
        return None
    d = np.argwhere(exp != got)
    i = tuple(int(x) for x in d[0])
    at = (i[0] + offset,) + i[1:] if i else i
    return "%s: %d elements differ, the first at %s: expected %s, got %s" % (
        name, len(d), at, exp[i].item(), got[i].item())


def assert_equal(name, exp, got, offset=0):
    msg = first_mismatch(name, exp, got, offset)
    assert msg is None, msg


def compare_rows(name, get_exp, get_got, first, n, chunk=1 << 20):
    """Rows [first, first + n) of two row sources, element for element, chunk rows at a time."""
    for a in range(first, first + n, chunk):
        k = min(chunk, first + n - a)
        assert_equal(name, get_exp(a, k), get_got(a, k), offset=a)


def ranges(u, gap=GAP):
    """Sorted distinct indices as (first, n) ranges that cover them, split where two neighbours lie more than gap apart."""
    u = np.asarray(u, np.int64)
    if u.size == 0:
        return []
    cut = np.flatnonzero(np.diff(u) > gap) + 1
    starts, ends = u[np.r_[0, cut]], u[np.r_[cut - 1, u.size - 1]]
    return [(int(a), int(b - a + 1)) for a, b in zip(starts, ends)]


def gather_rows(get_rows, idx, M, gap=GAP):
    """The rows of events idx (any order, repeats allowed, every index >= 0), fetched range by range."""
    idx = np.asarray(idx, np.int64)
    u, inv = np.unique(idx, return_inverse=True)
    out = np.empty((u.size, M), np.int32)
    for first, n in ranges(u, gap):
        lo, hi = np.searchsorted(u, [first, first + n])
        out[lo:hi] = get_rows(first, n)[u[lo:hi] - first]
    return out[inv.reshape(-1)]


def merged_parents(get_rows, p0, p1, height, h, M):
    """pre(h) of non-root events h: per column the higher (by height) of the two parents' entries, -1 where neither
    parent sees that member (swirld.py:170-174, 203-205)."""
    a = gather_rows(get_rows, p0[h], M)
    b = gather_rows(get_rows, p1[h], M)
    ha = np.where(a >= 0, height[np.maximum(a, 0)], -1)
    hb = np.where(b >= 0, height[np.maximum(b, 0)], -1)
    return np.where((a >= 0) & ((b < 0) | (ha >= hb)), a, b)


def expected_rows(get_rows, p0, p1, creator, height, first, n, M):
    """can_see rows of events [first, first + n) by the recurrence, from the rows of their parents (get_rows)."""
    h = np.arange(first, first + n, dtype=np.int64)
    out = np.full((n, M), -1, np.int32)
    inner = p0[h] >= 0
    if inner.any():
        out[inner] = merged_parents(get_rows, p0, p1, height, h[inner], M)
    out[np.arange(n), creator[h]] = h
    return out


def check_can_see(get_rows, p0, p1, creator, height, first, n, M, chunk=1 << 15):
    """Every row of [first, first + n) equals the recurrence over the rows get_rows gives its parents."""
    for a in range(first, first + n, chunk):
        k = min(chunk, first + n - a)
        assert_equal("can_see", expected_rows(get_rows, p0, p1, creator, height, a, k, M), get_rows(a, k), offset=a)


def expected_rounds(get_rows, rnd, stake, p0, p1, height, first, n, M):
    """The round of each event of [first, first + n) (swirld.py:200-219), from pre(h), the rows of the events pre(h)
    names and rnd, the rounds of earlier events (for h it reads rnd of events below h only, so the rounds the same
    window checks come in as inputs of later events).  Exact integers: with tot the total stake, x > min_s = 2 tot / 3
    is 3 x > 2 tot."""
    stake = np.asarray(stake, np.int64)
    tot = int(stake.sum())
    h = np.arange(first, first + n, dtype=np.int64)
    out = np.zeros(n, np.int32)                          # roots: round 0 (swirld.py:195-198)
    inner = np.flatnonzero(p0[h] >= 0)
    if inner.size == 0:
        return out
    hi = h[inner]
    r = np.maximum(rnd[p0[hi]], rnd[p1[hi]])             # swirld.py:200
    pre = merged_parents(get_rows, p0, p1, height, hi, M)
    # an entry k of pre(h) counts iff round[k] == r; its row then counts at every c_ whose entry k_ has round[k_] ==
    # r == round[k]: B[k, c_] depends on k alone
    ks = np.unique(pre[pre >= 0])
    rows_k = gather_rows(get_rows, ks, M)
    B = (rows_k >= 0) & (rnd[np.maximum(rows_k, 0)] == rnd[ks][:, None])
    for j in range(hi.size):
        K = pre[j]
        cols = np.flatnonzero((K >= 0) & (rnd[np.maximum(K, 0)] == r[j]))
        hits = stake[cols] @ B[np.searchsorted(ks, K[cols])].astype(np.int64)     # swirld.py:207-214
        cnt = int(np.count_nonzero(3 * hits > 2 * tot))
        out[inner[j]] = r[j] + 1 if 3 * cnt > 2 * tot else r[j]                   # swirld.py:216-219
    return out


def expected_witness(rnd, p0, first, n):
    """Witness flags of [first, first + n): roots, and events whose round exceeds their self-parent's (swirld.py:221-222)."""
    h = np.arange(first, first + n, dtype=np.int64)
    p = p0[h]
    return np.where(p < 0, 1, rnd[h] > rnd[np.maximum(p, 0)]).astype(np.uint8)


def check_witness_table(wt, wit, rnd, creator, lo, windows):
    """Every witness-table entry w >= lo that lies in one of windows ([a, b) pairs) is a flagged witness of its own row
    and column, and every flagged witness in those windows is in the table at (round, creator)."""
    R, c = np.nonzero(wt >= lo)
    w = wt[R, c].astype(np.int64)
    inside = np.zeros(w.size, bool)
    for a, b in windows:
        inside |= (w >= a) & (w < b)
    R, c, w = R[inside], c[inside], w[inside]
    assert inside.any(), "no witness-table entry inside the checked windows"
    assert_equal("witness flag of the table's entries", np.ones(w.size, np.uint8), wit[w])
    assert_equal("round of the table's entries", R.astype(np.int32), rnd[w])
    assert_equal("creator of the table's entries", c.astype(np.int32), creator[w])
    for a, b in windows:
        x = a + np.flatnonzero(wit[a:b])
        assert_equal("witness table at (round, creator) of the flagged witnesses", x, wt[rnd[x], creator[x]], offset=a)


def consensus_times(get_rows, end, p0, creator, t, wt, famous, X, rr):
    """swirld.py:295-305 for ordered events X with rounds received rr, from the can_see rows of events below end: those
    from X.min() on, and the few older ones the walks of famous witnesses that do not see x end on."""
    out = np.empty(X.size, np.float64)
    cs = _Window(get_rows, int(X.min()), end)
    for r in np.unique(rr):
        sel = np.flatnonzero(rr == r)
        F = np.array([w for w in wt[r] if w >= 0 and famous[w] == 1], np.int64)
        a, b = order_meta.median_halves(cs, p0, creator, t, F, np.asarray(X[sel], np.int64))
        with np.errstate(over="ignore"):
            out[sel] = .5 * (a + b)
    return out


class _Window:
    """The can_see rows of events [lo, end) as cs[i, c], fetched once and extended downwards, GAP rows past the
    lowest event read, when an older row is read."""

    def __init__(self, get_rows, lo, end):
        self.get_rows, self.lo = get_rows, lo
        self.rows = get_rows(lo, end - lo)

    def __getitem__(self, ic):
        i, c = ic
        i = np.asarray(i)
        low = int(i.min())
        if low < self.lo:
            new = max(0, low - GAP)
            self.rows = np.concatenate([self.get_rows(new, self.lo - new), self.rows])
            self.lo = new
        return self.rows[i - self.lo, c]


def sync_expected(rows, height, creator, head, old):
    """(summary of head, summary of the earlier head old, head's reply to that summary) by sync_model's closed form,
    from rows = {head: its can_see row, old: its row}, the heights and the creators."""
    v = SimpleNamespace(row=rows, height=height, creator=creator)
    S_old = sm.summary(v, old)
    return sm.summary(v, head), S_old, sm.closed_reply(v, head, S_old)
