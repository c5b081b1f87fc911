"""Consensus timestamps and rounds received on the oracle, for the tests.

The oracle reports the order only.  Its find_order takes the new consensus rounds one after the other (swirld.py:283),
so ordering them one call per round gives the same order and tells which round ordered each event: its round received.
The consensus timestamp of each such event is then restated here from the oracle's can_see table and witness / fame
state, as swirld.py:295-305 computes it: for every famous witness of the round that sees x, the time of the last
self-ancestor that still sees x (or the chain's root, quirk Q10), and the lopsided median of those times (quirk Q11).
tests/golden/meta_*.npz pin both to the unmodified reference (tools/make_order_meta.py)."""
import numpy as np

import oracle as orc


class OrderMeta:
    """Rides along one oracle view: given the event columns it was fed, find_order(new_c) orders through the oracle and
    returns what that call appended to the order as (events, consensus times, rounds received)."""

    def __init__(self, o):
        self.o = o
        self.p0 = np.empty(0, np.int32)
        self.creator = np.empty(0, np.int32)
        self.t = np.empty(0, np.float64)
        self.cs = np.empty((0, o.M), np.int32)      # can_see rows fetched so far (they never change once divided)
        self.ts, self.rr = [], []                   # parallel to the oracle's transactions
        self.med = []                               # ... and the two times each median was taken from

    def add_columns(self, p0, creator, t):
        self.p0 = np.concatenate([self.p0, np.asarray(p0, np.int32)])
        self.creator = np.concatenate([self.creator, np.asarray(creator, np.int32)])
        self.t = np.concatenate([self.t, np.asarray(t, np.float64)])

    def _rows(self, n_divided):
        have = self.cs.shape[0]
        if have < n_divided:
            self.cs = np.concatenate([self.cs, self.o.can_see(have, n_divided - have)])

    def _times(self, r, X, wt, fam):
        F = np.array([w for w in wt[r] if w >= 0 and fam[w] == 1], np.int64)
        return median_halves(self.cs, self.p0, self.creator, self.t, F, X)

    def find_order(self, new_c, n_divided):
        L, h = orc.lib(), self.o._h
        start = L.or_n_transactions(h)
        self._rows(n_divided)
        res = None
        for r in sorted(new_c):
            before = L.or_n_transactions(h)
            self.o.find_order([r])
            after = L.or_n_transactions(h)
            if after == before:
                continue
            if res is None:                          # (find_order changes no witness or fame state)
                res = self.o.results()
            tx = np.empty(after, np.int32)
            L.or_get_transactions(h, tx)
            X = tx[before:].astype(np.int64)
            a, b = self._times(r, X, res["witness_table"], res["famous"])
            with np.errstate(over="ignore"):         # two times near DBL_MAX: the sum is +inf, as in the reference
                self.ts += (.5 * (a + b)).tolist()
            self.med += list(zip(a.tolist(), b.tolist()))
            self.rr += [r] * X.size
        end = L.or_n_transactions(h)
        tx = np.empty(end, np.int32)
        if end:
            L.or_get_transactions(h, tx)
        return (tx[start:].copy(), np.array(self.ts[start:end], np.float64), np.array(self.rr[start:end], np.int32))


def median_halves(cs, p0, creator, t, F, X):
    """The two times whose mean is the consensus timestamp of each ordered event X of a round whose famous witnesses
    are F: for every f in F that sees x, the time of the event where the walk down f's self-parents (swirld.py:298-302)
    stops, and the median of those (swirld.py:305).  cs[i, c] reads can_see rows (an array, or anything indexed the
    same way)."""
    if X.size == 0:
        return np.empty((2, 0), np.float64)
    C = creator[X]
    A = np.repeat(F[:, None], X.size, axis=1)
    sees = cs[A, C] >= X
    cur = A.copy()
    while True:                                  # swirld.py:298-302
        go = sees & (cs[cur, C] >= X) & (p0[cur] >= 0)
        if not go.any():
            break
        cur = np.where(go, p0[cur], cur)
    s = np.sort(np.where(sees, t[cur], np.inf), axis=0)
    n = sees.sum(axis=0)
    cols = np.arange(X.size)
    return s[n // 2, cols], s[(n + 1) // 2, cols]             # swirld.py:305 (n >= 2 for an ordered event)


def run_oracle_meta(tr, K, stake=None, coin_period=6, extra=False):
    """Feed a trace with the call schedule K (chunk size, or a list of chunk sizes); returns the oracle's transactions
    and their consensus times and rounds received.  extra=True adds the two times of each median ("median", [n, 2]),
    results() and coverage()."""
    from swirld_b200.traces import chunks
    o = orc.Oracle(tr.M, stake, coin_period)
    o.append(tr)
    m = OrderMeta(o)
    m.add_columns(tr.p0, tr.creator, tr.t)
    sched = chunks(tr.N, K) if not isinstance(K, (list, tuple)) else _sizes(K)
    for first, cnt in sched:
        o.divide_rounds(first, cnt)
        m.find_order(o.decide_fame(), first + cnt)
    tx = np.empty(o.n_transactions, np.int32)
    if tx.size:
        orc.lib().or_get_transactions(o._h, tx)
    out = {"transactions": tx, "consensus_time": np.array(m.ts, np.float64),
           "round_received": np.array(m.rr, np.int32)}
    if extra:
        out.update(median=np.array(m.med, np.float64).reshape(-1, 2), results=o.results(), coverage=o.coverage())
    o.close()
    return out


def _sizes(sizes):
    first = 0
    for s in sizes:
        yield first, s
        first += s
