"""A pure-Python model of the reference's Node (swirld.py:34-160) for many node-views at once: one gossip turn of the
main loop (swirld.py:319-328) for every view, with real Ed25519 signatures (libsodium through PyNaCl) and BLAKE2b ids.

Each ModelView keeps what `sync` and `ask_sync` need: hg (id -> Event), the arrival list, `height`, and `can_see` of the
heads as {pk: id} dicts (swirld.py:196-207).  Consensus is left to the oracle: a view's trace (its events in arrival
order) and call schedule (events entered per turn) replay through it (`replay`).

A turn, for every view v with peer p = schedule.peers[turn][v]:
  1. v's request is {c: height[h] for c, h in can_see[head].items()} (swirld.py:125-126);
  2. p answers from its state before the turn with ask_sync's BFS (swirld.py:154-161), listed in p's arrival order;
  3. the reply reaches v with the schedule's tampered rows in place of the originals (a flipped signature bit; a
     changed payload under the kept id; an id that does not hash the preimage; a tampered remote head);
  4. v enters the rows it lacks that pass is_valid_event (swirld.py:97-110), parents first, and drops the others and
     whatever depends on them;
  5. if the remote head is valid (swirld.py:139), v makes new_event(payload, (head, remote_head)) at the time the
     schedule gives, and enters it.

One substitution: the reference enters the rows in toposort(remote_hg.keys() - hg.keys()) order (swirld.py:131), which
iterates a set of bytes, so its order follows the hash seed and cannot serve as an expected value.  The model enters
them in the engine's documented ingest order instead (include/swirld_b200.h, sw_ingest): a depth-first walk over the
rows in the order the reply lists them, parents first.  Any parents-first order gives the same graph; the arrival
indices, and with them the call schedule the oracle replays, are those of this order."""
from __future__ import annotations

import hashlib
import pickle
import random
from collections import Counter, namedtuple
from dataclasses import dataclass, field

import numpy as np

from swirld_b200.traces import Trace

Event = namedtuple("Event", "d p t c s")           # swirld.py:29

TAMPER_KINDS = ("sig", "msg", "id", "head")


def _nacl():
    from nacl import bindings
    return bindings


def event_id(ev):
    return hashlib.blake2b(pickle.dumps(ev), digest_size=32).digest()


def flip(b, bit):
    a = bytearray(b)
    a[bit // 8] ^= 1 << (bit % 8)
    return bytes(a)


def member_keys(M, seed):
    rng = random.Random(seed)
    return [_nacl().crypto_sign_seed_keypair(rng.randbytes(32)) for _ in range(M)]


def tamper(h, ev, kind, rng):
    """A copy of row (h, ev) as a faulty link delivers it: 'sig' flips a signature bit, 'msg' changes the payload and
    keeps the id, 'id' names the event by an id that is not the hash of its preimage."""
    if kind == "sig":
        return h, ev._replace(s=flip(ev.s, rng.randrange(512)))
    if kind == "msg":
        return h, ev._replace(d=(ev.d, "tampered"))
    assert kind == "id"
    return flip(h, rng.randrange(256)), ev


@dataclass
class Schedule:
    """What a driver picks: peers[k][v] answers view v in turn k (k = 0 .. turns-1, the same gossip, may repeat);
    times[k][v] is the time of v's event made in turn k (times[turns] are the roots'); tamper[k] lists (v, kind, u):
    view v's reply in turn k arrives with a row tampered as `kind`, u in [0, 1) picking which of the rows new to v."""
    M: int
    G: int                          # gossips; view v is member v % M of gossip v // M
    peers: list
    times: list
    tamper: list
    seed: int = 0

    @property
    def turns(self):
        return len(self.peers)

    @property
    def n_views(self):
        return self.M * self.G


def make_schedule(M, G, turns, seed, tamper=0.0, apart=None, derange=False):
    """A schedule for G gossips of M members each.  Times are non-integral and grow by turn; in each turn one of three
    patterns: every view of a gossip at one time, each view at its own time, or views one ulp apart (times that differ
    only in the last bits of a double).  tamper = the chance that a view's reply has a tampered row, each kind in turn.
    apart = (views, until): before turn `until` those views ask only each other and the rest only the rest; turn
    `until` has every view of the first set ask one of the rest (the catch-up).  derange: each gossip's peers are a
    permutation without fixed points, so no view answers twice in a turn."""
    rng = random.Random(seed)
    V = M * G
    peers, times, tam = [], [], []
    side = set(apart[0]) if apart else set()
    for k in range(turns + 1):
        base = 1.7e9 + 0.731 * k + rng.random() * 0.1
        row = []
        for g in range(G):
            mode = rng.randrange(3)
            t = base
            for _ in range(M):
                if mode == 1:
                    t = base + rng.randrange(1000) / 997
                elif mode == 2:
                    t = float(np.nextafter(t, np.inf))
                row.append(float(t))
        times.append(row)
    for k in range(turns):
        row = []
        for v in range(V):
            g = v // M
            if derange:
                if v % M == 0:
                    perm = list(range(M))
                    while any(p == i for i, p in enumerate(perm)):
                        rng.shuffle(perm)
                row.append(g * M + perm[v % M])
                continue
            pool = [u for u in range(g * M, (g + 1) * M) if u != v]
            if apart and k < apart[1]:
                pool = [u for u in pool if (u in side) == (v in side)] or pool
            elif apart and k == apart[1] and v in side:
                pool = [u for u in pool if u not in side]
            row.append(rng.choice(pool))
        peers.append(row)
        tam.append([(v, TAMPER_KINDS[(k * V + v) % 4], rng.random()) for v in range(V)
                    if tamper and rng.random() < tamper])
    times = times[1:] + times[:1]                  # times[turns] = the roots' times
    return Schedule(M, G, peers, times, tam, seed)


class ModelView:
    """One node-view (swirld.py:34-80): the member's keys, hg, arrival list, heights and its head."""

    def __init__(self, gossip, member, kp):
        self.g = gossip
        self.member = member
        self.pk, self.sk = kp
        self.hg, self.arrival, self.index, self.height = {}, [], {}, {}
        self.head = None
        self.sizes = []                             # events entered per turn: the divide_rounds call schedule

    @property
    def can_see(self):
        """can_see of the heads: an event's can_see depends only on its ancestors, so one dict serves the gossip."""
        return self.g.can_see

    def is_valid_event(self, h, ev):                # swirld.py:97-110
        try:
            _nacl().crypto_sign_open(ev.s + pickle.dumps(ev[:-1]), ev.c)
        except Exception:
            return False
        return (event_id(ev) == h
                and (ev.p == ()
                     or (len(ev.p) == 2 and ev.p[0] in self.hg and ev.p[1] in self.hg
                         and self.hg[ev.p[0]].c == ev.c and self.hg[ev.p[1]].c != ev.c)))

    def add_event(self, h, ev):                     # swirld.py:112-118
        self.hg[h] = ev
        self.index[h] = len(self.arrival)
        self.arrival.append(h)
        self.height[h] = 0 if ev.p == () else max(self.height[p] for p in ev.p) + 1

    def new_event(self, d, p, t):                   # swirld.py:82-95, at the driver's time t
        s = _nacl().crypto_sign(pickle.dumps((d, p, t, self.pk)), self.sk)[:64]
        ev = Event(d, p, t, self.pk, s)
        return event_id(ev), ev

    def own_event(self, d, p, t):
        """new_event, entered as this view's head, with its can_see (swirld.py:196-207)."""
        h, ev = self.new_event(d, p, t)
        assert self.is_valid_event(h, ev)
        self.add_event(h, ev)
        if p == ():
            cs = {ev.c: h}
        else:
            a, b = self.can_see[p[0]], self.can_see[p[1]]
            hi = lambda x, y: x is not None and (y is None or self.height[x] >= self.height[y])
            cs = {c: (a.get(c) if hi(a.get(c), b.get(c)) else b.get(c)) for c in a.keys() | b.keys()}
            cs[ev.c] = h
        self.can_see[h] = cs
        self.head = h
        return h, ev

    def request(self):                              # swirld.py:125-126
        return {c: self.height[h] for c, h in self.can_see[self.head].items()}

    def summary(self):
        """The request as M heights by member index, -1 for a member the head sees none of (sw_sync_summary)."""
        r = self.request()
        return np.array([r.get(pk, -1) for pk in self.g.pks], np.int32)

    def answer(self, cs):                           # swirld.py:154-161, utils.py:24-34
        """ask_sync's subset, as (id, Event) rows in this view's arrival order."""
        keep = lambda p: self.hg[p].c not in cs or self.height[p] > cs[self.hg[p].c]
        seen = {self.head}
        q = [self.head]
        while q:
            u = q.pop(0)
            for p in self.hg[u].p:
                if p not in seen and keep(p):
                    seen.add(p)
                    q.append(p)
        return [(h, self.hg[h]) for h in sorted(seen, key=self.index.__getitem__)]

    def trace(self, n=None):
        """This view's events [0, n) in arrival order, in index space."""
        ids = self.arrival[:n]
        ev = [self.hg[h] for h in ids]
        at = self.index
        p0 = np.array([at[e.p[0]] if e.p else -1 for e in ev], np.int32)
        p1 = np.array([at[e.p[1]] if e.p else -1 for e in ev], np.int32)
        cr = np.array([self.g.member[e.c] for e in ev], np.int32)
        t = np.array([e.t for e in ev], np.float64)
        sig = np.frombuffer(b"".join(e.s for e in ev), np.uint8).reshape(-1, 64).copy()
        return Trace(self.g.M, p0, p1, cr, t, sig, "gossip view")


def _parents_first(rows):
    """The order sw_ingest enters a batch in: a depth-first walk over the rows in their order, each row after the rows
    of its parents (p0, then p1) that are in the batch (utils.py:8-21 over a list instead of a set)."""
    at = {}
    for i, (h, _) in enumerate(rows):
        at.setdefault(h, i)
    done, out = set(), []

    def visit(i):
        stack = [(i, False)]
        while stack:
            j, expanded = stack.pop()
            if j in done:
                continue
            if expanded:
                done.add(j)
                out.append(rows[j])
                continue
            stack.append((j, True))
            for p in reversed(rows[j][1].p):
                k = at.get(p)
                if k is not None and k not in done:
                    stack.append((k, False))

    for i in range(len(rows)):
        if rows[i][0] in at and at[rows[i][0]] == i:
            visit(i)
    return out


@dataclass
class ViewTurn:
    """What one view saw and did in one turn."""
    peer: int
    request: np.ndarray             # the summary it sent
    reply: list                     # (id, Event) rows as the peer sent them
    delivered: list                 # ... as they reached the view (tampered rows in place)
    new_rows: list                  # positions in delivered of the ids the view lacked
    added: list                     # ids entered, in arrival order
    head_ok: bool
    new: tuple | None               # (id, Event) of the view's own new event
    first: int                      # the view's event count before the turn


@dataclass
class Gossip:
    """G gossips of M members, one ModelView per member, run turn by turn on one schedule."""
    schedule: Schedule
    views: list = field(default_factory=list)
    cov: Counter = field(default_factory=Counter)

    def __post_init__(self):
        s = self.schedule
        self.M = s.M
        self.keys = [member_keys(s.M, 1000 * s.seed + g) for g in range(s.G)]
        self.nets = []
        for g in range(s.G):
            net = _Net(self, g)
            self.nets.append(net)
            for m in range(s.M):
                self.views.append(ModelView(net, m, self.keys[g][m]))
        self.turn_no = 0
        self.rng = random.Random(s.seed ^ 0x5eed)

    def start(self):
        """Every view's root (swirld.py:75-80), at schedule.times[turns]."""
        t = self.schedule.times[-1]
        for v, x in enumerate(self.views):
            x.own_event(None, (), t[v])
            x.sizes.append(1)

    def payload(self, k, v):
        return None if (k + v) % 5 == 0 else b"tx %d.%d" % (k, v)

    def turn(self):
        """One turn of every view; returns [ViewTurn per view]."""
        s, k = self.schedule, self.turn_no
        peers = s.peers[k]
        reqs = [x.request() for x in self.views]
        sums = [x.summary() for x in self.views]
        replies = [self.views[p].answer(reqs[v]) for v, p in enumerate(peers)]     # all from the state before the turn
        reps = Counter(peers)
        self.cov["repeated_responders"] += sum(1 for n in reps.values() if n > 1)
        tam = {}
        for v, kind, u in s.tamper[k]:
            tam.setdefault(v, []).append((kind, u))
        out = []
        for v, x in enumerate(self.views):
            rows = list(replies[v])
            remote_head = rows[-1][0]
            fresh = [i for i, (h, _) in enumerate(rows) if h not in x.hg]
            self.cov["known_rows"] += len(rows) - len(fresh)
            for kind, u in tam.get(v, []):
                if kind == "head":
                    if fresh and fresh[-1] == len(rows) - 1:
                        rows[-1] = tamper(*rows[-1], "sig" if u < 0.5 else "msg", self.rng)
                        self.cov["tampered_head"] += 1
                    continue
                cand = [i for i in fresh if i != len(rows) - 1 and rows[i] == replies[v][i]]
                if cand:
                    i = cand[int(u * len(cand))]
                    rows[i] = tamper(*rows[i], kind, self.rng)
                    self.cov["tampered_" + kind] += 1
            first = len(x.arrival)
            added = []
            for h, ev in _parents_first([rows[i] for i in fresh]):
                if h not in x.hg and x.is_valid_event(h, ev):
                    x.add_event(h, ev)
                    added.append(h)
            dropped = len(fresh) - len(added)
            tampered = sum(1 for i in fresh if rows[i] != replies[v][i])
            self.cov["dropped"] += dropped
            self.cov["dropped_dependants"] += dropped - tampered
            delivered = dict(rows)
            head_ok = remote_head in delivered and x.is_valid_event(remote_head, delivered[remote_head])
            new = None
            if head_ok:
                new = x.own_event(self.payload(k, v), (x.head, remote_head), s.times[k][v])
            else:
                self.cov["zero_event_views"] += 1
            x.sizes.append(len(added) + (new is not None))
            self.cov["max_reply"] = max(self.cov["max_reply"], len(rows))
            out.append(ViewTurn(peers[v], sums[v], replies[v], rows, fresh, added, head_ok, new, first))
        self.turn_no += 1
        return out


class _Net:
    """One gossip's shared state: its members' keys and the can_see of every event made in it."""

    def __init__(self, gossip, g):
        self.M = gossip.M
        self.pks = [pk for pk, _ in gossip.keys[g]]
        self.member = {pk: m for m, pk in enumerate(self.pks)}
        self.can_see = {}


def time_cases(schedule):
    """How many turns of a gossip put several views at one time, and how many put views one ulp apart."""
    c = Counter()
    for row in schedule.times:
        for g in range(schedule.G):
            t = row[g * schedule.M:(g + 1) * schedule.M]
            c["non_integral"] += sum(1 for x in t if x != int(x))
            if len(set(t)) < len(t):
                c["equal_times"] += 1
            if any(b == float(np.nextafter(a, np.inf)) for a, b in zip(t, t[1:])):
                c["last_bit_times"] += 1
    return c


def replay(tr, sizes):
    """The oracle on one view's trace and call schedule (one divide_rounds, decide_fame, find_order per turn, as
    node_sim.replay_oracle), with tests/order_meta.py's consensus times and rounds received.  Returns results() plus
    'new_c' (per call), 'consensus_time' and 'round_received'."""
    import oracle as orc
    from order_meta import OrderMeta
    o = orc.Oracle(tr.M)
    o.append(tr)
    m = OrderMeta(o)
    m.add_columns(tr.p0, tr.creator, tr.t)
    ncs, first = [], 0
    for s in sizes:
        o.divide_rounds(first, s)
        nc = o.decide_fame()
        ncs.append(sorted(nc))
        m.find_order(nc, first + s)
        first += s
    assert first == tr.N
    r = o.results()
    r.update(new_c=ncs, consensus_time=np.array(m.ts, np.float64), round_received=np.array(m.rr, np.int32))
    o.close()
    return r


def check_replay(r):
    """The internal consistency a view's consensus must have: each event ordered once, rounds received non-decreasing,
    and within one round received consensus times non-decreasing (find_order sorts by (time, white ^ sig),
    swirld.py:306)."""
    tx, ts, rr = r["transactions"], r["consensus_time"], r["round_received"]
    assert len(set(tx.tolist())) == tx.size == ts.size == rr.size
    assert (np.diff(rr) >= 0).all()
    same = rr[1:] == rr[:-1]
    assert (ts[1:][same] >= ts[:-1][same]).all()
    assert set(np.flatnonzero(r["round"] >= 0).tolist()) >= set(tx.tolist())
