"""sw_batch_ingest_verified: the sync replies of several node-views in one call, each distinct event verified once on
the GPU.  Every view is compared with a twin engine that ingested the same rows through its own sw_ingest_verified:
index_out, counts, n_events, heights, the lookup of every id seen and, after divide_rounds / decide_fame / find_order
of everything, rounds, witnesses, fame, consensus, order and can_see.  The replies are what a peer view (or the
gossip's source) holds beyond the receiving view's events, with tampered copies (signature, signed bytes, preimage),
resends of known events and duplicate rows mixed in.  Covered: shared keys at 1 to 64 views on both kernel families
and above 64 members; one id intact in one view and tampered in another; views of different member counts and key
sets in one call; events merged by their creator's key, not its member index; a view whose rows are not a DAG and one out of capacity; refusals; the launches per call; and the
reference's main loop over 16 views against the oracle."""
import ctypes as C
import random

import numpy as np
import pytest

import test_gpu_batch_consensus as tbc
import test_gpu_verify as tv
import verify_cases as vc
from oracle_engine import OracleEngine
from swirld_b200 import engine as E

pytestmark = pytest.mark.gpu

CAP = 4096


class Gossip:
    """A signed gossip graph of M members in creation order (test_gpu_verify's events), revealed step events per turn
    by its source."""

    def __init__(self, M, n, seed, step):
        self.M, self.step = M, step
        self.pks, bursts = tv._gossip(M, n, seed)
        self.evs = [x for b in bursts for x in b]            # (id, Event, msg, preimage, member)
        self.F = 0

    def advance(self):
        self.F = min(len(self.evs), self.F + self.step)


def _tamper(rng, x):
    h, ev, msg, pre, c = x
    kind = rng.randrange(3)
    if kind == 0:
        ev = ev._replace(s=vc.flip(ev.s, rng.randrange(512)))
    elif kind == 1:
        msg = vc.flip(msg, rng.randrange(8 * len(msg)))
    else:
        pre = vc.flip(pre, rng.randrange(8 * len(pre)))
    return (h, ev, msg, pre, c)


def _batch(items):
    if not items:
        z = np.zeros(0, np.uint8)
        return (z, z, z, np.zeros(0, np.int32), np.zeros(0), z, [], [])
    return tv._cols(items) + ([x[2] for x in items], [x[3] for x in items])


class Views:
    """Node-views of one or more gossip graphs: views[v] = (gossip, keys).  Each turn every view receives one reply:
    what a peer view of the same graph, or the graph's source, holds beyond the view's own events (in creation order,
    at most `burst` of them), shuffled, with tampered copies, resends and duplicates mixed in."""

    def __init__(self, views, seed, burst=None, tamper=0.05, extras=True, cap=CAP):
        self.g = [g for g, _ in views]
        self.keys = [k for _, k in views]
        self.rng = random.Random(seed)
        self.burst, self.tamper, self.extras = burst, tamper, extras
        self.engs = [self._engine(g.M, k, cap) for g, k in views]
        self.known = [dict() for _ in views]                 # id -> the original item, per view
        self.seen = [set() for _ in views]                   # every id a view's rows ever held

    @staticmethod
    def _engine(M, keys, cap):
        e = E.Engine(M, cap)
        e.set_member_keys(keys)
        return e

    def rows(self):
        for g in dict.fromkeys(self.g):
            g.advance()
        rows = []
        for v, g in enumerate(self.g):
            rng = self.rng
            peers = [u for u in range(len(self.g)) if u != v and self.g[u] is g]
            u = rng.choice([None] + peers)
            have = ({x[0] for x in g.evs[:g.F]} if u is None else self.known[u].keys())
            diff = [x for x in g.evs if x[0] in have and x[0] not in self.known[v]][:self.burst]
            items = [_tamper(rng, x) if rng.random() < self.tamper else x for x in diff]
            if self.extras:
                if self.known[v] and rng.random() < 0.5:              # a resend, intact or not
                    x = rng.choice(list(self.known[v].values()))
                    items.append(_tamper(rng, x) if rng.random() < 0.5 else x)
                if items and rng.random() < 0.5:                      # a duplicate row, intact or not
                    x = rng.choice(items)
                    items.append(_tamper(rng, x) if rng.random() < 0.5 else x)
            if self.burst is not None:
                items = items[:self.burst]
            rng.shuffle(items)
            rows.append(items)
        return rows

    def expected_verified(self, rows, views=None):
        """The distinct (creator key, id, sig, msg, preimage) among the events new to some view: the first row of an
        id the view does not know."""
        out = set()
        for v in (range(len(rows)) if views is None else views):
            first = set()
            for h, ev, msg, pre, c in rows[v]:
                if h in first:
                    continue
                first.add(h)
                if h not in self.known[v]:
                    out.add((bytes(self.keys[v][c]), h, ev.s, msg, pre))
        return len(out)

    def record(self, rows, results):
        for v, (items, (idx, _)) in enumerate(zip(rows, results)):
            g = self.g[v]
            orig = {x[0]: x for x in g.evs}
            for x, i in zip(items, idx):
                self.seen[v].add(x[0])
                if i >= 0:
                    self.known[v].setdefault(x[0], orig[x[0]])


def _twins(views):
    return [Views._engine(g.M, k, CAP) for g, k in zip(views.g, views.keys)]


def _twin_ingest(tw, items):
    """sw_ingest_verified of one view's rows; returns (index_out, appended, events verified)."""
    before = tw.stats()["d2h_bytes"]
    b = _batch(items)
    idx, m = tw.ingest(*b[:6], msgs=b[6], preimages=b[7])
    return idx, m, tw.stats()["d2h_bytes"] - before


def _turn(views, twins, rows):
    got, nv = E.batch_ingest(views.engs, [_batch(r) for r in rows])
    twin_sum = 0
    for v, (items, (idx, m)) in enumerate(zip(rows, got)):
        ti, tm, tn = _twin_ingest(twins[v], items)
        twin_sum += tn
        assert np.array_equal(idx, ti) and m == tm, v
        assert views.engs[v].n_events == twins[v].n_events
    assert nv == views.expected_verified(rows)
    views.record(rows, got)
    return nv, twin_sum


def _ids(ids):
    return np.frombuffer(b"".join(ids), np.uint8) if ids else np.zeros(0, np.uint8)


def _same_state(a, b, seen):
    assert a.n_events == b.n_events
    assert np.array_equal(a.heights(), b.heights())
    ids = _ids(sorted(seen))
    assert np.array_equal(a.lookup(ids), b.lookup(ids))


def _same_consensus(a, b):
    n = a.n_events
    if n == 0:                                               # (a view whose every event failed holds nothing)
        return
    for x in (a, b):
        if n > x.n_divided:
            x.divide_rounds(x.n_divided, n - x.n_divided)
            x.find_order(x.decide_fame())
    assert np.array_equal(a.can_see(), b.can_see())
    ra, rb = a.results(), b.results()
    for k in ("round", "witness", "witness_table", "famous", "consensus", "transactions"):
        assert np.array_equal(ra[k], rb[k]), k


def _close(*engs):
    for e in engs:
        e.close()


# ---------------------------------------------------------------- 1. shared keys
@pytest.mark.parametrize("M,wide", [(8, False), (8, True), (64, False), (64, True), (72, False)])
@pytest.mark.parametrize("B", [1, 4, 16, 64])
def test_shared_keys(B, M, wide, monkeypatch):
    if wide:
        monkeypatch.setenv("SW_FORCE_WIDE", "1")
    g = Gossip(M, 700 if M <= 8 else 1100, seed=M + B, step=60)
    views = Views([(g, g.pks)] * B, seed=B * 7 + M + wide)
    twins = _twins(views)
    saved = tot = turns = 0
    while any(len(k) < len(g.evs) for k in views.known) and turns < 300:
        turns += 1
        nv, ts = _turn(views, twins, views.rows())
        saved += ts - nv
        tot += ts
        if g.F >= len(g.evs):
            views.tamper, views.extras = 0.0, False              # let every view catch up
    assert all(len(k) == len(g.evs) for k in views.known)
    if B >= 4:
        assert saved > 0, (saved, tot)
    for v in range(B):
        _same_state(views.engs[v], twins[v], views.seen[v])
    for v in range(B):
        _same_consensus(views.engs[v], twins[v])
    assert views.engs[0].max_round >= (2 if M <= 8 else 1)
    _close(*views.engs, *twins)


# ---------------------------------------------------------------- 2. one id, different bytes
def test_same_id_different_bytes():
    g = Gossip(8, 300, seed=5, step=300)
    views = Views([(g, g.pks)] * 2, seed=1, tamper=0.0, extras=False)
    twins = _twins(views)
    g.advance()
    evs = g.evs[:200]
    pick = evs[40]                                           # an event with descendants among the rows
    below = {pick[0]}
    for h, ev, *_ in evs:
        if ev.p and set(ev.p) & below:
            below.add(h)
    assert len(below) > 5
    rows = [list(evs), [_tamper(random.Random(2), x) if x[0] == pick[0] else x for x in evs]]
    for r in rows:
        random.Random(3).shuffle(r)
    nv, ts = _turn(views, twins, rows)
    assert nv == len(evs) + 1 and ts == 2 * len(evs)
    l0, l1 = views.engs[0].lookup(_ids([pick[0]])), views.engs[1].lookup(_ids(sorted(below)))
    assert l0[0] >= 0 and (l1 == -1).all()
    assert views.engs[0].n_events == len(evs) and views.engs[1].n_events == len(evs) - len(below)
    for v in range(2):
        _same_state(views.engs[v], twins[v], views.seen[v])
        _same_consensus(views.engs[v], twins[v])
    _close(*views.engs, *twins)


# ---------------------------------------------------------------- 3. different key sets
def test_different_key_sets():
    g4, g8, g72 = Gossip(4, 400, 11, 50), Gossip(8, 500, 12, 50), Gossip(72, 900, 13, 120)
    rot = g8.pks[1:] + g8.pks[:1]                            # the same graph under other keys: every event fails there
    views = Views([(g4, g4.pks), (g8, g8.pks), (g8, g8.pks), (g72, g72.pks), (g8, rot)], seed=4)
    twins = _twins(views)
    shared = 0
    for _ in range(12):
        rows = views.rows()
        alone = sum(views.expected_verified(rows, [v]) for v in range(5))
        pair = views.expected_verified(rows, [1, 2])
        rest = sum(views.expected_verified(rows, [v]) for v in (0, 3, 4))
        nv, ts = _turn(views, twins, rows)
        assert ts == alone and nv == pair + rest, (nv, pair, rest)
        shared += ts - nv
    assert shared > 0
    assert views.engs[4].n_events == 0 and len(views.known[1]) > 0
    for v in range(5):
        _same_state(views.engs[v], twins[v], views.seen[v])
        _same_consensus(views.engs[v], twins[v])
    _close(*views.engs, *twins)


# ---------------------------------------------------------------- 3b. merging by key, not by member index
def test_merge_by_key_not_member_index():
    """One graph in three views.  View 1 numbers the members in another order (its keys permuted, every creator index
    renumbered to match), so a shared event has another creator index there than in view 0 under the same key: it
    is verified once.  View 2 holds member j's key at member i too, so member i's events have the same index as in
    view 0 under another key: they fail there alone, with everything below them, and are not merged with view 0's."""
    M, i, j = 8, 2, 5
    g = Gossip(M, 500, seed=41, step=60)
    perm = list(range(M))
    random.Random(4).shuffle(perm)                           # the source's member c is view 1's member perm[c]
    assert all(perm[c] != c for c in (i, j))
    keys1 = [None] * M
    for c in range(M):
        keys1[perm[c]] = g.pks[c]
    keys2 = list(g.pks)
    keys2[i] = g.pks[j]
    views = Views([(g, g.pks), (g, keys1), (g, keys2)], seed=6)
    twins = _twins(views)
    shared01 = 0
    for _ in range(12):
        rows = views.rows()
        rows[1] = [x[:4] + (perm[x[4]],) for x in rows[1]]
        alone = [views.expected_verified(rows, [v]) for v in range(3)]
        shared01 += alone[0] + alone[1] - views.expected_verified(rows, [0, 1])
        nv, ts = _turn(views, twins, rows)
        assert ts == sum(alone)
    assert shared01 > 0
    assert len(views.known[1]) > 100
    own2 = {x[4] for x in views.known[2].values()}
    assert i not in own2 and j in own2
    for v in range(3):
        _same_state(views.engs[v], twins[v], views.seen[v])
        _same_consensus(views.engs[v], twins[v])
    _close(*views.engs, *twins)


# ---------------------------------------------------------------- 4. per-view failures
def test_failures_stay_with_their_view():
    g = Gossip(8, 600, seed=21, step=40)
    views = Views([(g, g.pks)] * 4, seed=9, tamper=0.0, extras=False)
    small = Views._engine(8, g.pks, 120)                     # view 2 runs out of capacity
    views.engs[2].close()
    views.engs[2] = small
    twins = _twins(views)
    twins[2].close()
    twins[2] = Views._engine(8, g.pks, 120)
    for _ in range(2):
        _turn(views, twins, views.rows())
    rows = views.rows()
    # view 1: two new events that name each other as self-parent (a cycle; their ids are not their hashes either)
    rng = random.Random(5)
    a, b = rng.randbytes(32), rng.randbytes(32)
    ev_a = vc.Event(None, (b, g.evs[0][0]), 1.0, g.pks[1], rng.randbytes(64))
    ev_b = vc.Event(None, (a, g.evs[0][0]), 2.0, g.pks[1], rng.randbytes(64))
    rows[1] = rows[1] + [(a, ev_a, b"m", b"p", 1), (b, ev_b, b"m", b"p", 1)]
    # view 2: more new events than its capacity holds
    have = views.engs[2].n_events
    rows[2] = [x for x in g.evs[:300] if x[0] not in views.known[2]]
    assert have + len(rows[2]) > 120
    state = [(e.n_events, e.heights().copy()) for e in views.engs]
    with pytest.raises(ExceptionGroup) as ei:
        E.batch_ingest(views.engs, [_batch(r) for r in rows])
    grp = ei.value
    assert sorted(x.view for x in grp.exceptions) == [1, 2]
    res = grp.results
    for v in (1, 2):
        with pytest.raises(E.EngineError) as single:
            tb = _batch(rows[v])
            twins[v].ingest(*tb[:6], msgs=tb[6], preimages=tb[7])
        ex = [x for x in grp.exceptions if x.view == v][0]
        assert ex.code == single.value.code == (-1 if v == 1 else -5)
        assert str(ex) == str(single.value)
        assert views.engs[v].n_events == state[v][0] and np.array_equal(views.engs[v].heights(), state[v][1])
        assert res[v] is None
    for v in (0, 3):
        ti, tm, _ = _twin_ingest(twins[v], rows[v])
        assert np.array_equal(res[v][0], ti) and res[v][1] == tm
    views.record([rows[v] if v in (0, 3) else [] for v in range(4)],
                 [res[v] if v in (0, 3) else (np.zeros(0, np.int32), 0) for v in range(4)])
    for v in range(4):
        _same_state(views.engs[v], twins[v], views.seen[v])
        _same_consensus(views.engs[v], twins[v])
    _close(*views.engs, *twins)


# ---------------------------------------------------------------- 5. refusals
def _raw(engs, offsets, rows, moff=None, B=None):
    cols = [np.zeros(0, np.uint8)] * 3 + [np.zeros(0, np.int32), np.zeros(0), np.zeros(0, np.uint8)]
    msgs, pres = [], []
    if any(rows):
        flat = [x for r in rows for x in r]
        b = _batch(flat)
        cols, msgs, pres = [np.ascontiguousarray(a) for a in b[:6]], b[6], b[7]
    (msg, mo), (pre, po) = E._packed(msgs), E._packed(pres)
    if moff is not None:
        mo = np.ascontiguousarray(moff, np.int64)
    offs = np.ascontiguousarray(offsets, np.int32)
    n = max(1, int(sum(len(r) for r in rows)))
    out = np.full(n, -7, np.int32)
    cnt = np.full(max(1, len(engs)), 12345, np.int32)
    arr = (C.c_void_p * max(1, len(engs)))(*[e._h if e is not None else None for e in engs])
    rc = E.load_library().sw_batch_ingest_verified(C.cast(arr, C.c_void_p), len(engs) if B is None else B,
                                                   E._ptr(offs), *[E._ptr(a) for a in cols], E._ptr(msg), E._ptr(mo),
                                                   E._ptr(pre), E._ptr(po), E._ptr(out), E._ptr(cnt), None)
    return rc, cnt


def test_refusals_change_nothing():
    g = Gossip(8, 200, seed=31, step=50)
    views = Views([(g, g.pks)] * 3, seed=2, tamper=0.0, extras=False)
    twins = _twins(views)
    _turn(views, twins, [g.evs[:20]] * 3)
    rows = [g.evs[20:40], g.evs[20:50], g.evs[20:60]]
    offs = np.cumsum([0] + [len(r) for r in rows])
    assert offs[-1] > 3
    nokeys = E.Engine(8, CAP)
    e0, e1, e2 = views.engs
    n0 = [e.n_events for e in views.engs]
    cases = [
        ("B < 1", dict(engs=[e0], offsets=offs[:1], rows=[], B=0), -1),
        ("NULL view", dict(engs=[e0, None, e2], offsets=offs, rows=rows), -1),
        ("repeated view", dict(engs=[e0, e1, e0], offsets=offs, rows=rows), -1),
        ("no keys", dict(engs=[e0, nokeys, e2], offsets=offs, rows=rows), -1),
        ("rows not monotone", dict(engs=views.engs, offsets=[0, offs[2], offs[1], offs[3]], rows=rows), -1),
        ("negative first row", dict(engs=views.engs, offsets=[-1] + list(offs[1:]), rows=rows), -1),
    ]
    flat_m = [x[2] for r in rows for x in r]
    mo = np.zeros(len(flat_m) + 1, np.int64)
    mo[1:] = np.cumsum([len(m) for m in flat_m])
    bad = mo.copy(); bad[2], bad[3] = bad[3], bad[2]
    cases.append(("byte offsets not monotone", dict(engs=views.engs, offsets=offs, rows=rows, moff=bad), -1))
    cases.append(("byte offsets not from 0", dict(engs=views.engs, offsets=offs, rows=rows, moff=mo + 1), -1))
    for what, kw, code in cases:
        rc, cnt = _raw(**kw)
        assert rc == code, what
        assert (cnt == 12345).all(), what
        assert [e.n_events for e in views.engs] == n0, what
        if kw.get("B") != 0:
            assert E.load_library().sw_last_error(e0._h), what
    # and the same rows then go in normally
    _turn(views, twins, rows)
    for v in range(3):
        _same_state(views.engs[v], twins[v], views.seen[v])
    _close(nokeys, *views.engs, *twins)


# ---------------------------------------------------------------- 6. launches
def test_three_launches_per_call():
    for B in (1, 64, tbc._n_sm() + 3):
        g = Gossip(8, 400, seed=B, step=30)
        views = Views([(g, g.pks)] * B, seed=B, burst=64)
        e0 = views.engs[0]
        calls = 0
        while g.F < len(g.evs):
            rows = views.rows()
            if not views.expected_verified(rows):
                continue
            before = e0.stats()["kernel_launches"]
            got, nv = E.batch_ingest(views.engs, [_batch(r) for r in rows])
            assert max(len(r) for r in rows) <= 64
            assert e0.stats()["kernel_launches"] - before == 2 + any(m for _, m in got), B
            views.record(rows, got)
            calls += 1
        assert calls >= 5
        _close(*views.engs)


# ---------------------------------------------------------------- 7. the whole loop
def test_main_loop_matches_oracle():
    M, B = 16, 16
    g = Gossip(M, 1600, seed=77, step=40)
    views = Views([(g, g.pks)] * B, seed=77)
    sample = (0, 5, 10, 15)
    orcs = {v: OracleEngine(M, CAP) for v in sample}
    idmap = [dict() for _ in range(B)]                       # id -> index, per view
    ncs = {v: [] for v in sample}
    oncs = {v: [] for v in sample}
    turns = 0
    while any(len(k) < len(g.evs) for k in views.known) and turns < 200:
        turns += 1
        if g.F >= len(g.evs):
            views.tamper, views.extras = 0.0, False
        rows = views.rows()
        before = [e.n_events for e in views.engs]
        got, _ = E.batch_ingest(views.engs, [_batch(r) for r in rows])
        views.record(rows, got)
        newv = []
        for v, (items, (idx, m)) in enumerate(zip(rows, got)):
            added = sorted({int(i): x for x, i in zip(items, idx) if i >= before[v]}.items())
            assert [i for i, _ in added] == list(range(before[v], before[v] + m))
            for i, x in added:
                idmap[v][x[0]] = i
            if m:
                newv.append(v)
            if v in orcs and m:
                evs = [views.known[v][x[0]] for _, x in added]
                p0 = [idmap[v][ev.p[0]] if ev.p else -1 for _, ev, *_ in evs]
                p1 = [idmap[v][ev.p[1]] if ev.p else -1 for _, ev, *_ in evs]
                orcs[v].append(p0, p1, [x[4] for x in evs], [x[1].t for x in evs],
                               np.frombuffer(b"".join(x[1].s for x in evs), np.uint8))
                orcs[v].divide_rounds(before[v], m)
        if newv:
            E.batch_divide_rounds([views.engs[v] for v in newv], [before[v] for v in newv],
                                  [views.engs[v].n_events - before[v] for v in newv])
        live = [v for v in range(B) if views.engs[v].n_divided > 0]
        if live:
            new_c = E.batch_decide_fame([views.engs[v] for v in live])
            E.batch_find_order([views.engs[v] for v in live], new_c)
            for v, nc in zip(live, new_c):
                if v in orcs:
                    ncs[v].append(sorted(nc))
                    onc = orcs[v].decide_fame()
                    oncs[v].append(sorted(onc))
                    orcs[v].find_order(onc)
    assert all(len(k) == len(g.evs) for k in views.known)
    for v in sample:
        e, o = views.engs[v], orcs[v]
        assert ncs[v] == oncs[v], v
        ro, re_ = o.results(), e.results()
        for k in ("round", "witness_table", "famous", "consensus", "transactions"):
            assert np.array_equal(np.asarray(ro[k]), np.asarray(re_[k])), (v, k)
        assert np.array_equal(o.can_see(), e.can_see()), v
    orders = []
    for v in range(B):
        rev = {i: h for h, i in idmap[v].items()}
        orders.append([rev[int(i)] for i in views.engs[v].transactions()])
    assert min(len(o) for o in orders) > 100
    for o in orders:
        k = min(len(o), len(orders[0]))
        assert o[:k] == orders[0][:k]
    _close(*views.engs, *orcs.values())
