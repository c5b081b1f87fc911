"""The whole gossip turn of many node-views on the engine's batched calls only, turn by turn against the reference's
Node as tests/gossip_model.py restates it.

Each turn a driver makes these calls, in this order, over the views in groups of B (one batched call per group):
  1. batch_sync_summary of every view's head;
  2. batch_sync_reply: each view's peer answers it.  A batched call takes an engine once, so when a responder answers
     several views in one turn, its second answer goes in a second batched call (and its third in a third);
  3. batch_ingest (the verified path) of the reply's rows, with the schedule's tampered rows in place of the originals;
  4. batch_new_events with ingest: one template for a view whose remote head was valid, none for the others;
  5. batch_divide_rounds of the views that entered events (on the any-M kernels, which batch calls of at most 16
     events a view, a view that entered more goes through its own Engine.divide_rounds);
  6. batch_decide_fame and 7. batch_find_order_out of every view.
After every turn every view's new ids and heights, its summary, its reply, its new event's signature and id (libsodium,
BLAKE2b of the pickle), the lookup of that id and the count each call returned equal the model's, exactly.  At two
intermediate turns and at the end, every view's results(), consensus_times(), rounds_received(), the new consensus rounds
of each call and what find_order_out returned equal the oracle's replay of that view's trace and call schedule, bit for
bit.  A failing view's trace and schedule are kept in the temporary directory (failing_gossip_view_*.npz).

Also: Engine.new_events at 4 096 and 4 097 templates (either side of the switch from 8 lanes per event to 1), and
batch_new_events with views of zero templates beside views of several."""
import math
import os
import pickle
import tempfile
from collections import Counter

import numpy as np
import pytest

nacl = pytest.importorskip("nacl.bindings")

import gossip_model as gm
from swirld_b200 import engine as E
from swirld_b200.events import event_template

pytestmark = pytest.mark.gpu
ZERO = bytes(32)
RESULT_KEYS = ("round", "witness", "witness_table", "famous", "consensus", "transactions")


def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rows(rows, net):
    """(id, Event) rows as batch_ingest takes them: ids, p0_ids, p1_ids, creator, t, sig, msgs, preimages."""
    ids = np.frombuffer(b"".join(h for h, _ in rows), np.uint8).reshape(-1, 32)
    p0 = np.frombuffer(b"".join(ev.p[0] if ev.p else ZERO for _, ev in rows), np.uint8).reshape(-1, 32)
    p1 = np.frombuffer(b"".join(ev.p[1] if ev.p else ZERO for _, ev in rows), np.uint8).reshape(-1, 32)
    cr = np.array([net.member[ev.c] for _, ev in rows], np.int32)
    t = np.array([ev.t for _, ev in rows], np.float64)
    sig = np.frombuffer(b"".join(ev.s for _, ev in rows), np.uint8).reshape(-1, 64)
    return (ids, p0, p1, cr, t, sig, [pickle.dumps(ev[:-1]) for _, ev in rows], [pickle.dumps(ev) for _, ev in rows])


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


class EngineSet:
    """One engine per model view, driven through the batched calls.  rotate: every call's groups start at another
    view each turn, so each batched call follows one with a different first engine; sync: Engine.sync() on every view
    of a group before each batched call (the twin of a rotated set, with no work of any view left in flight)."""

    def __init__(self, loop, rotate=False, sync=False):
        self.loop, self.rotate, self.sync = loop, rotate, sync
        m = loop.m
        self.E = []
        for v, x in enumerate(m.views):
            e = E.Engine(m.M, loop.cap)
            e.set_member_keys(x.g.pks)
            e.set_signing_key(x.member, x.sk)
            self.E.append(e)
        self.head = [-1] * len(m.views)
        self.ncs = [[] for _ in m.views]                       # decide_fame's new rounds, per call
        self.out = [[[], [], []] for _ in m.views]             # find_order_out's (events, times, rounds received)
        self.firsts = []

    def groups(self, k, call):
        V, B = len(self.E), self.loop.B
        order = list(range(V))
        if self.rotate:
            r = (7 * k + 3 * call + 1) % V
            order = order[r:] + order[:r]
        gs = [order[i:i + B] for i in range(0, V, B)]
        self.firsts.append(gs[0][0])
        return gs

    def enter(self, views):
        if self.sync:
            for v in views:
                self.E[v].sync()
        return [self.E[v] for v in views]

    def close(self):
        for e in self.E:
            e.close()


class Loop:
    def __init__(self, schedule, B, cap=None, sets=((False, False),)):
        self.m = gm.Gossip(schedule)
        self.M, self.B = schedule.M, B
        self.cap = cap or schedule.M * (schedule.turns + 1) + 64
        self.wide = schedule.M > 64 or os.environ.get("SW_FORCE_WIDE") == "1"
        self.sets = [EngineSet(self, r, s) for r, s in sets]
        self.cov = Counter()
        self.k = 0

    def new_events(self, S, k, made):
        """Step 4 (and the roots): made[v] = (id, Event) of view v's new event or None."""
        m = self.m
        for grp in S.groups(k, 3):
            tms = [[event_template(gm.Event, made[v][1].d, made[v][1].p, made[v][1].t, m.views[v].pk)] if made[v] else []
                   for v in grp]
            p0 = [[made[v][1].p[0] if made[v][1].p else ZERO] if made[v] else [] for v in grp]
            p1 = [[made[v][1].p[1] if made[v][1].p else ZERO] if made[v] else [] for v in grp]
            p0 = [np.frombuffer(b"".join(x), np.uint8) for x in p0]
            p1 = [np.frombuffer(b"".join(x), np.uint8) for x in p1]
            ts = [[made[v][1].t] if made[v] else [] for v in grp]
            self.cov["zero_template_views"] += sum(1 for v in grp if not made[v])
            if any(made[v] for v in grp) and not all(made[v] for v in grp):
                self.cov["mixed_new_event_calls"] += 1
            res = E.batch_new_events(S.enter(grp), tms, p0, p1, ts)
            for v, (sig, ids, idx, n) in zip(grp, res):
                x = m.views[v]
                if not made[v]:
                    assert n == 0 and len(sig) == 0 and len(ids) == 0, (k, v)
                    continue
                h, ev = made[v]
                assert bytes(sig[0]) == ev.s, ("signature", k, v)
                assert bytes(ids[0]) == h, ("id", k, v)
                assert n == 1 and list(idx) == [x.index[h]], (k, v, n, list(idx))
                S.head[v] = x.index[h]
        for v in range(len(made)):
            if made[v]:
                assert list(S.E[v].lookup(np.frombuffer(made[v][0], np.uint8))) == [m.views[v].index[made[v][0]]]

    def consensus(self, S, k, sizes, firsts):
        """Steps 5 to 7."""
        for grp in S.groups(k, 4):
            live = [v for v in grp if sizes[v] > 0]
            # the any-M kernels batch calls of at most 16 events a view; a larger one goes through its own single call
            alone = [v for v in live if self.wide and sizes[v] > 16]
            live = [v for v in live if v not in alone]
            if live:
                E.batch_divide_rounds(S.enter(live), [firsts[v] for v in live], [sizes[v] for v in live])
                self.cov["batched_divides"] += len(live)
            for v in alone:
                S.enter([v])[0].divide_rounds(firsts[v], sizes[v])
                self.cov["single_divides"] += 1
        for grp in S.groups(k, 5):
            ncs = E.batch_decide_fame(S.enter(grp))
            for v, nc in zip(grp, ncs):
                S.ncs[v].append(sorted(nc))
            outs = E.batch_find_order_out(S.enter(grp), ncs)
            for v, nc, (ev, ts, rr) in zip(grp, ncs, outs):
                assert len(ev) == len(ts) == len(rr) and (nc or not len(ev))
                for a, b in zip(S.out[v], (ev, ts, rr)):
                    a.append(np.array(b))

    def start(self):
        m = self.m
        m.start()
        made = [(x.arrival[0], x.hg[x.arrival[0]]) for x in m.views]
        for S in self.sets:
            self.new_events(S, -1, made)
            self.consensus(S, -1, [1] * len(made), [0] * len(made))
            for v, (h, _) in enumerate(made):
                assert S.E[v].ids().tobytes() == h and S.E[v].heights().tolist() == [0], ("root", v)

    def turn(self):
        m, k = self.m, self.k
        vt = m.turn()
        V = len(vt)
        self.cov["repeated_responder_turns"] += len(set(t.peer for t in vt)) < V
        for S in self.sets:
            E_ = S.E
            # 1. summaries
            sums = [None] * V
            for grp in S.groups(k, 0):
                for v, s in zip(grp, E.batch_sync_summary(S.enter(grp), [S.head[v] for v in grp])):
                    assert np.array_equal(s, vt[v].request), ("summary", k, v, s, vt[v].request)
                    sums[v] = s
            # 2. replies: a responder answers once per batched call; its further answers go in further calls
            for grp in S.groups(k, 1):
                rounds = []
                for v in grp:
                    p = vt[v].peer
                    for r in rounds:
                        if p not in r:
                            r[p] = v
                            break
                    else:
                        rounds.append({p: v})
                if len(rounds) > 1:
                    self.cov["second_reply_calls"] += len(rounds) - 1
                for r in rounds:
                    ps = list(r)
                    idx, cols = E.batch_sync_reply(S.enter(ps), [S.head[p] for p in ps], [sums[r[p]] for p in ps])
                    for p, ix, c in zip(ps, idx, cols):
                        v = r[p]
                        rep = vt[v].reply
                        net = m.views[p].g
                        want = _rows(rep, net)
                        assert list(ix) == [m.views[p].index[h] for h, _ in rep], ("reply", k, v, p)
                        for a, b in zip(c, want[:6]):
                            assert np.array_equal(np.asarray(a).reshape(np.shape(b)), b), ("reply columns", k, v, p)
            # 3. ingest, verified
            for grp in S.groups(k, 2):
                batches = [_rows(vt[v].delivered, m.views[v].g) for v in grp]
                got, nv = E.batch_ingest(S.enter(grp), batches)
                distinct = set()
                for v in grp:
                    t, x = vt[v], m.views[v]
                    for i in t.new_rows:
                        h, ev = t.delivered[i]
                        distinct.add((ev.c, h, ev.s, pickle.dumps(ev[:-1]), pickle.dumps(ev)))
                assert nv == len(distinct), ("verified", k, nv, len(distinct))
                for v, (ix, n) in zip(grp, got):
                    t, x = vt[v], m.views[v]
                    assert n == len(t.added), ("appended", k, v, n, len(t.added))
                    want = [x.index[h] if h in x.hg and x.index[h] < t.first + len(t.added) else -1
                            for h, _ in t.delivered]
                    assert list(ix) == want, ("index_out", k, v)
            # 4. new events
            made = [t.new for t in vt]
            self.new_events(S, k, made)
            # 5 - 7.
            sizes = [len(t.added) + (t.new is not None) for t in vt]
            self.consensus(S, k, sizes, [t.first for t in vt])
            for v, t in enumerate(vt):
                x = m.views[v]
                n = t.first + sizes[v]
                assert E_[v].n_events == n == len(x.arrival), ("n_events", k, v)
                if sizes[v]:
                    got = E_[v].ids(t.first)
                    assert got.tobytes() == b"".join(x.arrival[t.first:]), ("ids", k, v)
                    assert E_[v].heights(t.first).tolist() == [x.height[h] for h in x.arrival[t.first:]], ("heights", k, v)
        self.k += 1
        return vt

    def check(self, tag):
        """Every view of every set against the oracle's replay of its trace and call schedule."""
        m = self.m
        ordered = 0
        for v, x in enumerate(m.views):
            tr = x.trace()
            r = gm.replay(tr, x.sizes)
            gm.check_replay(r)
            ordered += r["transactions"].size
            for S in self.sets:
                e = S.E[v]
                try:
                    assert e.ids().tobytes() == b"".join(x.arrival)
                    got = e.results()
                    for key in RESULT_KEYS:
                        assert np.array_equal(np.asarray(got[key]), np.asarray(r[key])), (tag, v, key)
                    assert np.array_equal(_bits(e.consensus_times()), _bits(r["consensus_time"])), (tag, v, "times")
                    assert np.array_equal(e.rounds_received(), r["round_received"]), (tag, v, "rounds received")
                    assert S.ncs[v] == r["new_c"], (tag, v, "new_c")
                    ev, ts, rr = (np.concatenate(a) if a else np.zeros(0) for a in S.out[v])
                    assert np.array_equal(ev, r["transactions"]) and np.array_equal(rr, r["round_received"])
                    assert np.array_equal(_bits(ts), _bits(r["consensus_time"]))
                except AssertionError:
                    _dump("%s_v%d" % (tag, v), tr, x.sizes, m.schedule)
                    raise
        return ordered

    def close(self):
        for S in self.sets:
            S.close()


def _dump(tag, tr, sizes, schedule):
    """Keeps a failing view's trace and call schedule, and the gossip's schedule, for a replay outside the test."""
    out = tempfile.gettempdir()
    np.savez(os.path.join(out, "failing_gossip_view_%s.npz" % tag), M=tr.M, p0=tr.p0, p1=tr.p1, creator=tr.creator,
             t=tr.t, sig=tr.sig, sizes=np.array(sizes, np.int32),
             schedule=np.frombuffer(pickle.dumps(schedule), np.uint8))


def _run(loop, turns, checks=None, each=None):
    checks = set(checks or (turns // 3, 2 * turns // 3))
    loop.start()
    ordered = 0
    for k in range(turns):
        loop.turn()
        if each:
            each(loop, k)
        if k + 1 in checks:
            loop.check("turn%d" % (k + 1))
    ordered = loop.check("end")
    return ordered


CASES = {
    # the reference's own cadence: one to a few events per call, the streaming kernel
    "m4_b4": dict(M=4, G=1, B=4, turns=300),
    # drops, dependants of drops, tampered remote heads, zero-event views in batch_new_events
    "m16_b16_tampered": dict(M=16, G=1, B=16, turns=80, tamper=0.1),
    # the any-M kernel family under the same loop
    "m16_wide": dict(M=16, G=1, B=16, turns=50, wide=True),
    "m97": dict(M=97, G=1, B=97, turns=80),
}


@pytest.mark.parametrize("name", list(CASES))
def test_gossip_loop(name, monkeypatch):
    c = dict(CASES[name])
    if c.pop("wide", False):
        monkeypatch.setenv("SW_FORCE_WIDE", "1")
    turns, B = c.pop("turns"), c.pop("B")
    s = gm.make_schedule(c["M"], c["G"], turns, seed=len(name), tamper=c.get("tamper", 0.0))
    loop = Loop(s, B)
    ordered = _run(loop, turns)
    cov = loop.m.cov + loop.cov
    print(name, dict(cov), "ordered", ordered)
    assert ordered > 0 and cov["repeated_responder_turns"] > 0 and cov["second_reply_calls"] > 0
    if loop.wide:
        assert cov["batched_divides"] > 0 and (cov["single_divides"] > 0 or c["M"] <= 64)
    if name == "m16_b16_tampered":
        for what in ("tampered_sig", "tampered_msg", "tampered_id", "tampered_head", "dropped_dependants",
                     "zero_template_views", "mixed_new_event_calls"):
            assert cov[what] > 0, what
    loop.close()


def test_gossip_loop_more_views_than_sms():
    """Gossips of 16 members, n_sm + 3 views or more in one group: every batched call takes more views than the GPU has
    SMs.  Each gossip's peers are a derangement, so the replies too go in one call."""
    n_sm = _n_sm()
    G = math.ceil((n_sm + 3) / 16)
    s = gm.make_schedule(16, G, 50, seed=5, derange=True)
    loop = Loop(s, 16 * G)
    assert 16 * G >= n_sm + 3
    assert _run(loop, 50) > 0
    loop.close()


def test_gossip_loop_apart_then_healed():
    """M = 64, 8 views per batched call.  Views 0-7 (one group) gossip only among themselves for 60 turns, then each
    asks one of the others: catch-up replies of well over 2048 events, which the group divides in one batched call on
    the cluster round kernel (it takes a batch whose views all bring 2048 events or more).  Not reached here: the
    hand-over to k_rounds_batch, which needs chains more than 32 rounds apart, some 450 turns of this gossip at
    M = 64 (14 turns a round); tests/test_gpu_partition.py reaches it on traces."""
    apart, heal = list(range(8)), 60
    s = gm.make_schedule(64, 1, heal + 10, seed=64, apart=(apart, heal))
    loop = Loop(s, 8)
    seen = {}

    def each(lp, k):
        engs = lp.sets[0].E
        if k == heal - 1:
            for e in engs:
                e.debug_counters()                          # (cleared)
        if k == heal:
            seen["catch_up"] = [lp.m.views[v].sizes[-1] for v in apart]
            seen["cluster_launches"] = sum(int(e.debug_counters()[7]) for e in engs)
    assert _run(loop, heal + 10, checks=(heal, heal + 1), each=each) > 0
    assert min(seen["catch_up"]) > 2048, seen
    assert seen["cluster_launches"] > 0, seen
    loop.close()


def test_gossip_loop_rotated_first_engine():
    """Every batched call starts at another view each turn, so it follows a call with another first engine while
    views have appends or a round-stream piece of the previous call pending; a twin set that syncs every view before
    each batched call ends byte-identical (and both equal the model and the oracle)."""
    s = gm.make_schedule(16, 1, 60, seed=16, tamper=0.05)
    loop = Loop(s, 16, sets=((True, False), (True, True)))
    _run(loop, 60)
    a, b = loop.sets
    assert len(set(a.firsts)) > 8
    changed = sum(1 for x, y in zip(a.firsts, a.firsts[1:]) if x != y)
    assert changed > len(a.firsts) // 2
    for ea, eb in zip(a.E, b.E):
        assert ea.ids().tobytes() == eb.ids().tobytes()
        assert np.array_equal(ea.can_see(), eb.can_see())
        ra, rb = ea.results(), eb.results()
        for key in RESULT_KEYS:
            assert np.array_equal(ra[key], rb[key]), key
        assert np.array_equal(_bits(ea.consensus_times()), _bits(eb.consensus_times()))
    loop.close()


def test_gossip_loop_reload(tmp_path):
    """View 3 is saved at turn 40 and reloaded with Engine.load; member keys and its signing key are set again and the
    loop goes on.  Its own events from before the save are still served by sync_reply (sw_load rebuilds the index ->
    id table), and every later turn equals the model."""
    s = gm.make_schedule(16, 1, 60, seed=40, tamper=0.05)
    loop = Loop(s, 8)
    done = []

    def each(lp, k):
        if k != 39:
            return
        S, v = lp.sets[0], 3
        x = lp.m.views[v]
        path = str(tmp_path / "view3.bin")
        S.E[v].save(path)
        S.E[v].close()
        e = E.Engine.load(path, capacity=lp.cap)
        e.set_member_keys(x.g.pks)
        e.set_signing_key(x.member, x.sk)
        S.E[v] = e
        assert e.ids().tobytes() == b"".join(x.arrival)
        idx, cols = e.sync_reply(S.head[v], np.full(lp.M, -1, np.int32))
        own = [i for i, h in enumerate(x.arrival) if x.hg[h].c == x.pk]
        assert set(own) <= set(idx.tolist()) and len(own) > 30
        assert cols[0].tobytes() == b"".join(x.arrival[i] for i in idx)
        done.append(k)
    assert _run(loop, 60, each=each) > 0
    assert done == [39]
    loop.close()


# ---------------------------------------------------------------- new events either side of the lane switch
@pytest.mark.parametrize("n", [4096, 4097])
def test_new_events_lane_switch(n):
    keys = gm.member_keys(4, 7)
    e = E.Engine(4, 64)
    e.set_member_keys([pk for pk, _ in keys])
    e.set_signing_key(2, keys[2][1])
    pk = keys[2][0]
    tm = [event_template(gm.Event, b"x" * (i % 300) if i % 3 else None, (), 1.7e9 + i / 7, pk) for i in range(n)]
    sig, ids = e.new_events(tm, ingest=False)
    for i, (msg, pre, at) in enumerate(tm):
        want = nacl.crypto_sign(msg, keys[2][1])[:64]
        assert bytes(sig[i]) == want, i
        ev = gm.Event(*pickle.loads(msg), want)
        assert bytes(ids[i]) == gm.event_id(ev), i
    e.close()


def test_batch_new_events_zero_template_views():
    """Views of zero templates beside views of several, the first view among the empty ones: each view equals its own
    single call, byte for byte, and the batch is one launch.  With ingest, empty views enter nothing."""
    keys = gm.member_keys(8, 8)
    counts = [0, 3, 0, 0, 5, 1, 0, 2]

    def view(m):
        e = E.Engine(8, 64)
        e.set_member_keys([pk for pk, _ in keys])
        e.set_signing_key(m, keys[m][1])
        return e
    A = [view(m) for m in range(8)]
    S = [view(m) for m in range(8)]
    tms = [[event_template(gm.Event, b"v%d.%d" % (m, i), (), 1.5 + i * 0.25, keys[m][0]) for i in range(c)]
           for m, c in enumerate(counts)]
    before = A[0].stats()["kernel_launches"]
    got = E.batch_new_events(A, tms, ingest=False)
    assert A[0].stats()["kernel_launches"] - before == 1
    for m, (sig, ids) in enumerate(got):
        s1, i1 = S[m].new_events(tms[m], ingest=False)
        assert sig.tobytes() == s1.tobytes() and ids.tobytes() == i1.tobytes() and len(sig) == counts[m]
        for (msg, pre, at), s in zip(tms[m], sig):
            assert bytes(s) == nacl.crypto_sign(msg, keys[m][1])[:64]
    # with ingest: one root for some views, none for the others
    roots = [[t[0]] if t and m % 2 else [] for m, t in enumerate(tms)]
    zeros = [np.zeros((len(r), 32), np.uint8) for r in roots]
    ts = [[1.5] * len(r) for r in roots]
    got = E.batch_new_events(A, roots, zeros, zeros, ts)
    for m, (sig, ids, idx, n) in enumerate(got):
        s1, i1, x1, n1 = S[m].new_events(roots[m], zeros[m], zeros[m], ts[m])
        assert sig.tobytes() == s1.tobytes() and ids.tobytes() == i1.tobytes()
        assert list(idx) == list(x1) and n == n1 == len(roots[m])
        assert A[m].n_events == S[m].n_events == len(roots[m])
        assert A[m].ids().tobytes() == S[m].ids().tobytes()
        if roots[m]:
            assert list(A[m].lookup(ids)) == [0]
    for e in A + S:
        e.close()
