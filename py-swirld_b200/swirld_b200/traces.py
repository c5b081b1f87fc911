"""Deterministic synthetic hashgraph traces (SURVEY.md section 8d).

A trace is the *global* view of a gossip run in index space: event ``i`` has a
self-parent ``p0[i]``, an other-parent ``p1[i]`` (both ``-1`` for a member's
root event), a creator ``creator[i]`` (member id ``0..M-1``), a float64
timestamp ``t[i]`` and a 64-byte signature ``sig[i]``.  Events are listed in a
topological (arrival) order, so ``p0[i] < i`` and ``p1[i] < i``.

The generators reproduce the shape of what the reference simulation produces
(``swirld.py:315-345``: a random member syncs with a random
*other* member and creates one event whose parents are the two heads), without
crypto:

* G1 ``gossip``       -- the reference sim's process (swirld.py:323, 341-344).
* G2 ``adversarial``  -- G1 restricted to two cliques with a small cross-clique
  probability (delayed fame, coin rounds) plus stale other-parents ("near
  forks": an other-parent that is 1..7 events behind the peer's head; still a
  valid event per swirld.py:103-108, never a true fork).
* G3 ``tick``         -- tick-synchronous: every tick each member creates one
  event on a random peer's previous-tick head (frontier width == M).
* G5 ``partition``    -- G1 with the network split in two sides for a window of
  events, then healed (stalled rounds, chains far behind, huge heal rounds).

Everything is pure ``random.Random(seed)`` + ``hashlib.blake2b`` so that the
same trace is rebuilt bit-for-bit here, in the golden-fixture script and on
any machine.
"""
from __future__ import annotations

import hashlib
import random
from dataclasses import dataclass

import numpy as np


@dataclass
class Trace:
    """SoA view of a hashgraph; the layout the engine keeps in HBM."""
    M: int
    p0: np.ndarray        # int32[N]  self-parent index, -1 for roots
    p1: np.ndarray        # int32[N]  other-parent index, -1 for roots
    creator: np.ndarray   # int32[N]  member id
    t: np.ndarray         # float64[N] creation time (swirld.py:91)
    sig: np.ndarray       # uint8[N,64] signature bytes (swirld.py:92)
    name: str = ""

    @property
    def N(self) -> int:
        return int(self.p0.shape[0])

    def slice(self, a: int, b: int) -> "Trace":
        return Trace(self.M, self.p0[a:b], self.p1[a:b], self.creator[a:b],
                     self.t[a:b], self.sig[a:b], self.name)


def make_sigs(seed: int, n: int) -> np.ndarray:
    """sig[i] = blake2b(b'sig<seed>:<i>', 64 bytes) -- stands in for the
    Ed25519 signature whose bytes the hot path consumes (swirld.py:272, 281)."""
    out = np.empty((n, 64), dtype=np.uint8)
    for i in range(n):
        out[i] = np.frombuffer(
            hashlib.blake2b(b"sig%d:%d" % (seed, i), digest_size=64).digest(),
            dtype=np.uint8)
    return out


def _finish(M, p0, p1, cr, seed, name, tied=0) -> Trace:
    n = len(p0)
    if tied:
        t = (np.arange(n, dtype=np.int64) // tied).astype(np.float64)
    else:
        t = np.arange(n, dtype=np.float64)
    return Trace(M, np.asarray(p0, dtype=np.int32), np.asarray(p1, dtype=np.int32),
                 np.asarray(cr, dtype=np.int32), t, make_sigs(seed, n), name)


def gossip(M: int, N: int, seed: int = 1, tied: int = 0) -> Trace:
    """G1: events 0..M-1 are the roots (creator == index); afterwards a random
    member ``a`` syncs with a random other member ``b`` and creates an event
    with parents (head[a], head[b])."""
    assert M >= 2 and N >= M
    rng = random.Random(seed)
    p0 = [-1] * M
    p1 = [-1] * M
    cr = list(range(M))
    head = list(range(M))
    for i in range(M, N):
        a = rng.randrange(M)
        b = rng.randrange(M - 1)
        b += (b >= a)
        p0.append(head[a])
        p1.append(head[b])
        cr.append(a)
        head[a] = i
    return _finish(M, p0, p1, cr, seed, "G1(M=%d,N=%d,seed=%d)" % (M, N, seed), tied)


def adversarial(M: int, N: int, seed: int = 1, p_cross: float = 0.02,
                p_stale: float = 0.3, tied: int = 0) -> Trace:
    """G2: two cliques (members < M/2 and >= M/2).  The peer is drawn from the
    creator's own clique unless a ``p_cross`` coin says otherwise; with
    probability ``p_stale`` the other-parent is not the peer's head but an
    event 1..7 steps back on the peer's self-parent chain (clamped at the
    peer's root)."""
    assert M >= 4 and N >= M
    rng = random.Random(seed)
    half = M // 2
    p0 = [-1] * M
    p1 = [-1] * M
    cr = list(range(M))
    head = list(range(M))
    for i in range(M, N):
        a = rng.randrange(M)
        lo, hi = (0, half) if a < half else (half, M)
        if rng.random() < p_cross:
            lo, hi = (half, M) if a < half else (0, half)
            b = lo + rng.randrange(hi - lo)
        else:
            b = lo + rng.randrange(hi - lo - 1)
            b += (b >= a)
        other = head[b]
        if rng.random() < p_stale:
            back = 1 + rng.randrange(7)
            while back > 0 and p0[other] >= 0:
                other = p0[other]
                back -= 1
        p0.append(head[a])
        p1.append(other)
        cr.append(a)
        head[a] = i
    return _finish(M, p0, p1, cr, seed,
                   "G2(M=%d,N=%d,seed=%d,pc=%g,ps=%g)" % (M, N, seed, p_cross, p_stale), tied)


def partition(M: int, N: int, seed: int = 1, split: int | None = None, start: int = 0, end: int | None = None,
              tied: int = 0) -> Trace:
    """G5: a network partition that heals.  G1, except that for events ``start <= i < end`` the peer ``b`` is drawn
    from the creator's own side, ``[0, split)`` or ``[split, M)`` (``split`` defaults to M // 2, ``end`` to N).

    With an even split neither side holds more than 2/3 of the members, so no witness of either side can strongly see
    a supermajority: every member stalls in one round for the whole partition, hundreds of events per chain.  With
    a split above 2/3 the majority side keeps advancing rounds while the minority stalls, and on heal the minority's
    chains are dozens to hundreds of rounds behind.  The heal round orders a whole partition's events at once.  These
    are the sizes the kernels are built around (DESIGN.md section 2): runs of one member's events in one round longer
    than the 256-event rings of the round kernels (RB_RING, RW_RING) and the 128-row window of the cluster round
    kernel (RC_WN), chains more than the 32 rounds of its Wf mirror (RB_WR) apart, and consensus rounds of more than
    the 1024 events k_order_sort's block sorts in one pass."""
    split = M // 2 if split is None else split
    end = N if end is None else end
    assert 2 <= split <= M - 2 and N >= M and 0 <= start <= end
    rng = random.Random(seed)
    p0 = [-1] * M
    p1 = [-1] * M
    cr = list(range(M))
    head = list(range(M))
    for i in range(M, N):
        a = rng.randrange(M)
        if start <= i < end:
            lo, hi = (0, split) if a < split else (split, M)
            b = lo + rng.randrange(hi - lo - 1)
        else:
            b = rng.randrange(M - 1)
        b += (b >= a)
        p0.append(head[a])
        p1.append(head[b])
        cr.append(a)
        head[a] = i
    return _finish(M, p0, p1, cr, seed, "G5(M=%d,N=%d,seed=%d,split=%d,[%d,%d))" % (M, N, seed, split, start, end), tied)


def tick(M: int, N: int, seed: int = 1) -> Trace:
    """G3: tick-synchronous gossip; in tick k every member (in a random order)
    creates one event whose other-parent is a random peer's tick k-1 event."""
    assert M >= 2 and N >= M
    rng = random.Random(seed)
    p0 = [-1] * M
    p1 = [-1] * M
    cr = list(range(M))
    prev = list(range(M))
    i = M
    while i < N:
        cur = list(prev)
        order = list(range(M))
        rng.shuffle(order)
        for a in order:
            if i >= N:
                break
            b = rng.randrange(M - 1)
            b += (b >= a)
            p0.append(prev[a])
            p1.append(prev[b])
            cr.append(a)
            cur[a] = i
            i += 1
        prev = cur
    return _finish(M, p0, p1, cr, seed, "G3(M=%d,N=%d,seed=%d)" % (M, N, seed))


def late_joiner(M: int, N: int, join_at: int, seed: int = 1) -> Trace:
    """G4: gossip among members 0..M-2; member M-1 creates its root only after ``join_at`` events (dozens of rounds
    in) and gossips like the others from then on: its chain starts far more rounds behind than the round kernels mirror
    in shared memory (swirld_rcluster.cuh hands such a chunk to the grid-wide kernel)."""
    assert M >= 3 and M - 1 <= join_at < N
    rng = np.random.default_rng(seed)
    p0, p1, cr, head = [], [], [], {}
    for c in range(M - 1):
        head[c] = len(cr); p0.append(-1); p1.append(-1); cr.append(c)
    while len(cr) < N:
        if len(cr) == join_at:
            c = M - 1
            head[c] = len(cr); p0.append(-1); p1.append(-1); cr.append(c)
            continue
        act = sorted(head)
        c = int(act[rng.integers(len(act))])
        o = int(act[rng.integers(len(act))])
        if o == c:
            continue
        p0.append(head[c]); p1.append(head[o]); cr.append(c)
        head[c] = len(cr) - 1
    return _finish(M, np.array(p0, np.int32), np.array(p1, np.int32), np.array(cr, np.int32), seed, "late-joiner")


TIME_KINDS = ("wall", "shuffle", "neg", "const", "huge", "tiny")
PREFIXES = (8, 16, 32, 56, 60)
SIG_KINDS = tuple("prefix%d" % p for p in PREFIXES) + tuple("prefix%d_coin" % p for p in PREFIXES) + ("coin0", "coin1")


def _restamp_times(kind, tr, rng):
    N = tr.N
    i = np.arange(N, dtype=np.float64)
    if kind == "wall":           # a wall clock in seconds, each member's off by up to 5 s, with sub-microsecond jitter
        skew = rng.uniform(-5.0, 5.0, tr.M)
        return 1.7e9 + i * 1e-3 + skew[tr.creator] + rng.uniform(0.0, 1e-6, N)
    if kind == "shuffle":
        return rng.permutation(N) + 1.0
    if kind == "neg":
        return rng.uniform(-1e6, 1e6, N)
    if kind == "const":
        return np.full(N, 1234.5)
    if kind == "huge":           # medians of two 1e308 overflow to +inf
        t = rng.uniform(-1.0, 1.0, N)
        t[rng.random(N) < 0.5] = 1e308
        return t
    if kind == "tiny":           # odd multiples of the least subnormal: .5 * (a + b) rounds half to even
        return rng.integers(1, 1 << 12, N).astype(np.float64) * 5e-324
    raise ValueError(kind)


def _restamp_sigs(kind, tr, rng):
    N = tr.N
    sig = tr.sig.copy()
    if kind in ("coin0", "coin1"):
        sig[:, 0] = (sig[:, 0] & 0x7F) | (0x80 if kind == "coin1" else 0)
        return sig
    P = int(kind[len("prefix"):].split("_")[0])
    assert P in PREFIXES, kind
    sig[:, :P] = rng.integers(0, 256, P, dtype=np.uint8)
    sig[:, 60:] = rng.permutation(N).astype(">u4").view(np.uint8).reshape(N, 4)
    if kind.endswith("_coin"):
        sig[:, 0] = (sig[:, 0] & 0x7F) | (tr.sig[:, 0] & 0x80)
    return sig


def restamped(base: str, times: str, sigs: str, seed: int = 1, **base_kwargs) -> Trace:
    """The graph of generator ``base`` (called with ``seed`` and ``base_kwargs``) with other value columns: the
    timestamps and signatures that only find_order and the coin read.

    times: ``wall`` (fractional seconds near 1.7e9, out of arrival order across members), ``shuffle`` (a permutation of
    1..N, not monotone along chains), ``neg`` (mixed signs), ``const`` (one value: every order is decided by the
    signature key), ``huge`` (half 1e308, the rest in (-1, 1): medians overflow to +inf), ``tiny`` (subnormals).
    sigs: ``prefixP`` (bytes [0, P) one constant for the trace, bytes [60, 64) a permutation of the events, so ties are
    decided at byte P or later), ``prefixP_coin`` (the same with bit 7 of byte 0, the coin, left as it was), ``coin0`` /
    ``coin1`` (the coin bit forced).

    No time is NaN, +-0.0 or -inf and signatures stay pairwise distinct: on such columns the reference's order depends
    on how Python iterates a set."""
    tr = globals()[base](seed=seed, **base_kwargs)
    rng = np.random.default_rng([seed, 0x7E57])
    t = _restamp_times(times, tr, rng)
    sig = _restamp_sigs(sigs, tr, rng)
    assert not np.isnan(t).any() and not (t == 0).any() and not (t == -np.inf).any()
    assert np.unique(sig, axis=0).shape[0] == tr.N, "signatures must stay distinct"
    return Trace(tr.M, tr.p0, tr.p1, tr.creator, t, sig, "%s[t=%s,sig=%s]" % (tr.name, times, sigs))


def chunks(n: int, k: int):
    """The call schedule: consecutive [first, first+count) slices of K events,
    one (divide_rounds, decide_fame, find_order) triple per slice
    (swirld.py:324-328).  The final order depends on it (SURVEY.md section 0.5)."""
    first = 0
    while first < n:
        cnt = min(k, n - first)
        yield first, cnt
        first += cnt


def can_see_rows(tr: Trace) -> np.ndarray:
    """int32[N, M]: row[i][m] = the latest event of member m that event i sees (itself in its own column), -1 none --
    the max-plus recurrence over the parents (swirld.py:203-205), one pass in index order."""
    row = np.full((tr.N, tr.M), -1, np.int32)
    p0, p1, cr = tr.p0.tolist(), tr.p1.tolist(), tr.creator.tolist()
    for i in range(tr.N):
        if p0[i] >= 0:
            np.maximum(row[p0[i]], row[p1[i]], out=row[i])
        row[i, cr[i]] = i
    return row


def node_view(base: Trace, X: int, rows: np.ndarray | None = None):
    """Node X's own view of the gossip that ``base`` records: (view trace, call sizes).

    In ``base`` event i is its creator syncing with a peer and creating i (the process gossip() draws), so X holds an
    event once one of X's own events sees it.  With x_1 < x_2 < ... X's events and row() the can_see rows of ``base``,
    an event e of member m is in the view iff e <= row(x_last)[m], and arrives with X's sync j: the first j with
    row(x_j)[m] >= e.  The view lists its events by (sync, base index): what each sync brought, parents first, then
    X's new event last.  Parents are remapped, ``t`` and ``sig`` travel with their event.  sizes[j] is the number of
    events of sync j: one divide_rounds call per sync, as the reference's Node.main makes them (swirld.py:324-328).
    ``rows``: can_see_rows(base), to share one pass among the views of every member (node_views)."""
    rows = can_see_rows(base) if rows is None else rows
    chain = np.flatnonzero(base.creator == X)
    assert chain.size, "member %d has no event" % X
    R = rows[chain]                                   # [J, M], every column non-decreasing along X's chain
    ev = np.arange(base.N)
    m = base.creator.astype(np.int64)
    inside = ev <= R[-1][m]
    key = np.full(base.N, -1, np.int64)
    for c in range(base.M):                           # one searchsorted per member, over X's chain
        mine = np.flatnonzero(inside & (m == c))
        key[mine] = np.searchsorted(R[:, c], mine, side="left")
    keep = np.flatnonzero(inside)
    order = keep[np.lexsort((keep, key[keep]))]
    new = np.full(base.N, -1, np.int64)
    new[order] = np.arange(order.size)
    remap = lambda p: np.where(p >= 0, new[np.maximum(p, 0)], -1).astype(np.int32)
    view = Trace(base.M, remap(base.p0[order]), remap(base.p1[order]), base.creator[order].copy(), base.t[order].copy(),
                 base.sig[order].copy(), "view%d[%s]" % (X, base.name))
    sizes = np.bincount(key[order], minlength=chain.size)
    return view, [int(s) for s in sizes]


def node_views(base: Trace):
    """node_view(base, X) of every member X, from one can_see pass over ``base``."""
    rows = can_see_rows(base)
    return [node_view(base, X, rows) for X in range(base.M)]


def heights(tr: Trace) -> np.ndarray:
    """Topological level of each event (swirld.py:114-120)."""
    h = np.zeros(tr.N, dtype=np.int32)
    p0, p1 = tr.p0.tolist(), tr.p1.tolist()
    hl = [0] * tr.N
    for i in range(tr.N):
        if p0[i] >= 0:
            hl[i] = max(hl[p0[i]], hl[p1[i]]) + 1
    h[:] = hl
    return h


# ---------------------------------------------------------------------------------------------------------
# Vectorised generators for the large configurations (BASELINE.json configs 4 and 5: 4 M and 16 M events).
# Same processes as G1 / G2 above, drawn from numpy's PCG64 instead of `random.Random` (so the traces differ
# from gossip()/adversarial() with the same seed, but are just as reproducible), built without a Python loop
# over the events: the head of member b "at time i" is the last event j < i with creator[j] == b, found by a
# searchsorted over b's own event list.
def _fast_sigs(seed: int, n: int) -> np.ndarray:
    """64 signature bytes per event from a counter-based generator (blake2b per event is ~1 us: too slow at 16 M)."""
    rng = np.random.Generator(np.random.Philox(key=seed ^ 0x5157))
    return rng.integers(0, 256, size=(n, 64), dtype=np.uint8)


def _finish_np(M, p0, p1, cr, seed, name):
    n = len(p0)
    return Trace(M, p0.astype(np.int32), p1.astype(np.int32), cr.astype(np.int32),
                 np.arange(n, dtype=np.float64), _fast_sigs(seed, n), name)


def _chain_lists(M, a):
    """events of every member in index order: (order, starts) with order[starts[c]:starts[c+1]] = c's events."""
    order = np.argsort(a, kind="stable")
    starts = np.searchsorted(a[order], np.arange(M + 1))
    return order, starts


def gossip_np(M: int, N: int, seed: int = 1) -> Trace:
    """G1 at scale: roots 0..M-1, then creator a ~ U(M), peer b ~ U(M) \\ {a}, parents (head[a], head[b])."""
    assert M >= 2 and N >= M
    rng = np.random.Generator(np.random.PCG64(seed))
    a = np.concatenate([np.arange(M), rng.integers(0, M, N - M)])
    b = rng.integers(0, M - 1, N)
    b += b >= a
    order, starts = _chain_lists(M, a)
    pos = np.empty(N, np.int64)                      # position of event i in its creator's list
    pos[order] = np.arange(N) - np.repeat(starts[:-1], np.diff(starts))
    p0 = np.where(pos > 0, order[np.maximum(starts[a] + pos - 1, 0)], -1)
    # head of b below i: number of b's events with index < i, minus one
    p1 = np.empty(N, np.int64)
    border, bstarts = _chain_lists(M, b)             # the events that chose peer c, in index order
    for c in range(M):
        idx = border[bstarts[c]:bstarts[c + 1]]
        ev = order[starts[c]:starts[c + 1]]
        k = np.searchsorted(ev, idx)                 # events of c strictly below idx (idx itself is not c's: b != a)
        p1[idx] = ev[np.maximum(k - 1, 0)]
    p0[:M] = -1
    p1[:M] = -1
    return _finish_np(M, p0, p1, a, seed, "G1np(M=%d,N=%d,seed=%d)" % (M, N, seed))


def adversarial_np(M: int, N: int, seed: int = 1, p_cross: float = 0.02, p_stale: float = 0.3) -> Trace:
    """G2 at scale: two cliques, cross-clique peer with probability p_cross, other-parent 1..7 events behind the
    peer's head with probability p_stale (clamped at the peer's root): delayed fame and near-forks, no true forks."""
    assert M >= 4 and N >= M
    rng = np.random.Generator(np.random.PCG64(seed))
    half = M // 2
    a = np.concatenate([np.arange(M), rng.integers(0, M, N - M)])
    low = a < half
    cross = rng.random(N) < p_cross
    lo_own = np.where(low, 0, half)
    n_own = np.where(low, half, M - half)
    lo_oth = np.where(low, half, 0)
    n_oth = np.where(low, M - half, half)
    u = rng.random(N)
    b_cross = lo_oth + np.minimum((u * n_oth).astype(np.int64), n_oth - 1)
    b_own = lo_own + np.minimum((u * (n_own - 1)).astype(np.int64), n_own - 2)
    b_own += b_own >= a
    b = np.where(cross, b_cross, b_own)
    back = np.where(rng.random(N) < p_stale, 1 + rng.integers(0, 7, N), 0)
    order, starts = _chain_lists(M, a)
    pos = np.empty(N, np.int64)
    pos[order] = np.arange(N) - np.repeat(starts[:-1], np.diff(starts))
    p0 = np.where(pos > 0, order[np.maximum(starts[a] + pos - 1, 0)], -1)
    p1 = np.empty(N, np.int64)
    border, bstarts = _chain_lists(M, b)
    for c in range(M):
        idx = border[bstarts[c]:bstarts[c + 1]]
        ev = order[starts[c]:starts[c + 1]]
        k = np.searchsorted(ev, idx) - 1             # the peer's head below idx
        p1[idx] = ev[np.maximum(k - back[idx], 0)]
    p0[:M] = -1
    p1[:M] = -1
    return _finish_np(M, p0, p1, a, seed, "G2np(M=%d,N=%d,seed=%d,pc=%g,ps=%g)" % (M, N, seed, p_cross, p_stale))
