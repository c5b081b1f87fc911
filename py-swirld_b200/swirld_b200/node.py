"""GpuNode -- the reference's `Node` with its consensus hot path on the H100 engine.

    import swirld, swirld_b200.node
    swirld.Node = swirld_b200.node.bind(swirld.Node)   # before swirld.test(...) / importing viz

`bind(host_cls)` returns a subclass of the reference's own class: gossip, crypto and the wire
format (`sync`, `ask_sync`, `new_event`, `is_valid_event`'s checks, `main`: swirld.py:82-161,
315-328) are INHERITED from the reference at run time -- nothing of them lives in this package --
while the consensus state and the three hot-path methods (`divide_rounds`, `decide_fame`,
`find_order`: swirld.py:187-311) run on the GPU through the C ABI.  The attributes `viz.py` and the
drivers read (`round`, `famous`, `idx`, `can_see`, `witnesses`, `tbd`) become lazy mapping views that
pull from the device only what is asked for; `hg`, `height`, `head`, `transactions`, `consensus`
stay plain Python objects.  Beyond the reference's surface, `consensus_time` and `round_received` map
each ordered event to its consensus timestamp (swirld.py:305) and the round that ordered it
(swirld.py:283); find_order brings them back with the order itself.  Hashes (bytes) are mapped to arrival indices and public keys to member
ids at this boundary.

No CPU fallback: constructing a bound node without the CUDA library / a GPU raises.

Divergence from the reference, on purpose: the engine's index-space math is exact on fork-free
graphs only (the reference itself has no fork handling, swirld.py:110-112), so an event that forks
its creator's chain (a second root, or a self-parent that is not the creator's latest known event)
is treated as INVALID here and dropped by `sync` like any other invalid event, instead of being
accepted and silently corrupting the state.
"""
from __future__ import annotations

from collections.abc import Mapping

import numpy as np

COIN_PERIOD = 6                            # swirld.py:17


class _View(Mapping):
    """Read-only dict-like view keyed by event hash over a per-event device column."""

    def __init__(self, node, getter, present, count=None):
        self._n, self._get, self._present, self._count = node, getter, present, count

    def __getitem__(self, h):
        i = self._n._h2i[h]
        if not self._present(i):
            raise KeyError(h)
        return self._get(i)

    def __contains__(self, h):
        i = self._n._h2i.get(h)
        return i is not None and self._present(i)

    def __iter__(self):
        return (h for i, h in enumerate(self._n._i2h) if self._present(i))

    def __len__(self):
        return self._count() if self._count is not None else sum(1 for _ in self)


class _OrderView(Mapping):
    """Read-only dict-like view keyed by event hash over a host list parallel to `transactions` (ordered events only)."""

    def __init__(self, node, values):
        self._n, self._v = node, values

    def __getitem__(self, h):
        i = self._n._order_pos.get(h)
        if i is None or i >= len(self._v):
            raise KeyError(h)
        return self._v[i]

    def __contains__(self, h):
        i = self._n._order_pos.get(h)
        return i is not None and i < len(self._v)

    def __iter__(self):
        return iter(self._n.transactions[:len(self._v)])

    def __len__(self):
        return len(self._v)


class _Witnesses(Mapping):
    """witnesses[r] -> {member pk: event hash}  (swirld.py:61)."""

    def __init__(self, node):
        self._n = node

    def __getitem__(self, r):
        n = self._n
        if r < 0 or r > n._eng.max_round:
            raise KeyError(r)
        row = n._eng.witness_table(r, 1)[0]
        return {n._m2pk[c]: n._i2h[int(w)] for c, w in enumerate(row) if w >= 0}

    def __iter__(self):
        return iter(range(self._n._eng.max_round + 1))

    def __len__(self):
        return self._n._eng.max_round + 1


class GpuConsensus:
    """Mixed in front of the host class by bind(): owns the engine, the hash<->index maps, the views and the
    three hot-path methods.  Everything else resolves to the host class."""

    _engine_cls = None                     # tests substitute the oracle here by subclassing; the product never does

    # ------------------------------------------------------------------ construction (Node.__init__, swirld.py:38-80)
    def __init__(self, kp, network, n_nodes, stake, capacity=1 << 15, device=0):
        self.pk, self.sk = kp
        self.network = network
        self.n = n_nodes
        self.stake = stake
        self.tot_stake = sum(stake.values())
        self.min_s = 2 * self.tot_stake / 3
        self._m2pk = list(stake)           # member ids: the order of the stake dict (the same on every node)
        self._pk2m = {pk: m for m, pk in enumerate(self._m2pk)}
        self._stake_list = []
        for pk in self._m2pk:
            s = stake[pk]
            if int(s) != s or s < 0:
                raise ValueError("stake of %r is %r: the engine takes non-negative integer stakes" % (pk, s))
            self._stake_list.append(int(s))
        self._device, self._capacity = device, int(capacity)
        self._eng = self._make_engine(self._capacity)
        self.hg, self.height = {}, {}
        self._h2i, self._i2h = {}, []
        self._heads = {}                   # member pk -> its latest known event (fork check)
        self._pending = []                 # added to hg, not yet on the device
        self._n_on_device = 0
        self._ops = []                     # the call schedule, replayed if the engine has to grow
        self.head = None
        self.transactions, self.consensus, self.votes = [], set(), {}
        self._order_pos = {}               # event hash -> its position in transactions
        self._tx_ts, self._tx_rr = [], []  # parallel to transactions (empty when the engine cannot report them)
        self._round_cache = np.empty(0, np.int32)
        self._famous_cache = self._idx_cache = None
        self._views = {
            "round": _View(self, self._round_of, lambda i: i < self._eng.n_divided, lambda: self._eng.n_divided),
            "famous": _View(self, lambda i: bool(self._famous()[i]), lambda i: i < self._eng.n_events and self._famous()[i] >= 0,
                            lambda: int((self._famous() >= 0).sum())),
            "idx": _View(self, lambda i: int(self._idx()[i]), lambda i: i < self._eng.n_events and self._idx()[i] >= 0,
                         lambda: len(self.transactions)),
            "can_see": _View(self, self._can_see_of, lambda i: i < self._eng.n_divided, lambda: self._eng.n_divided),
            "witnesses": _Witnesses(self),
            "consensus_time": _OrderView(self, self._tx_ts),
            "round_received": _OrderView(self, self._tx_rr),
        }
        h, ev = self.new_event(None, ())   # the node's own root (the host class signs and hashes it)
        self.add_event(h, ev)
        self.divide_rounds((h,))
        self.head = h

    round = property(lambda self: self._views["round"])
    famous = property(lambda self: self._views["famous"])
    idx = property(lambda self: self._views["idx"])
    can_see = property(lambda self: self._views["can_see"])
    witnesses = property(lambda self: self._views["witnesses"])
    consensus_time = property(lambda self: self._views["consensus_time"])
    round_received = property(lambda self: self._views["round_received"])

    @property
    def tbd(self):
        """Events whose final order is still to be determined (swirld.py:52)."""
        return set(self._i2h) - set(self.transactions)

    # ------------------------------------------------------------------ engine plumbing
    def _make_engine(self, capacity):
        cls = self._engine_cls
        if cls is None:
            from .engine import Engine as cls
        return cls(len(self._m2pk), capacity, self._stake_list, COIN_PERIOD, self._device)

    def _columns(self, idxs):
        n = len(idxs)
        p0 = np.full(n, -1, np.int32); p1 = np.full(n, -1, np.int32); cr = np.empty(n, np.int32)
        t = np.empty(n, np.float64); sig = np.empty((n, 64), np.uint8)
        for j, i in enumerate(idxs):
            ev = self.hg[self._i2h[i]]
            if ev.p:
                p0[j], p1[j] = self._h2i[ev.p[0]], self._h2i[ev.p[1]]
            cr[j] = self._pk2m[ev.c]
            t[j] = ev.t
            sig[j] = np.frombuffer(ev.s, np.uint8)
        return p0, p1, cr, t, sig

    def _flush(self):
        """Events added since the last call go to the device in one sw_append."""
        if not self._pending:
            return
        need = self._n_on_device + len(self._pending)
        if need > self._capacity:
            self._grow(need)
        self._eng.append(*self._columns(self._pending))
        self._n_on_device = need
        self._pending = []

    def _grow(self, need):
        """A bigger engine that continues where this one stands: through a checkpoint (sw_save / sw_load with a larger
        capacity) where the engine has one, else by feeding the same events and the same call schedule again (the
        final order depends on the schedule)."""
        while self._capacity < need:
            self._capacity *= 2
        old = self._eng
        if hasattr(old, "save"):
            import os
            import tempfile
            fd, path = tempfile.mkstemp(suffix=".swb")
            os.close(fd)
            try:
                old.save(path)
                self._eng = type(old).load(path, device=self._device, capacity=self._capacity)
            finally:
                os.unlink(path)
            old.close()
            return
        self._eng = self._make_engine(self._capacity)
        if self._n_on_device:
            self._eng.append(*self._columns(range(self._n_on_device)))
        for op in self._ops:
            if op[0] == "d":
                self._eng.divide_rounds(op[1], op[2])
            elif op[0] == "f":
                self._eng.decide_fame()
            else:
                self._eng.find_order(list(op[1]))
        old.close()

    def _round_of(self, i):
        nd = self._eng.n_divided
        have = self._round_cache.shape[0]
        if have < nd:                       # rounds never change once assigned
            self._round_cache = np.concatenate([self._round_cache, self._eng.rounds(have, nd - have)])
        return int(self._round_cache[i])

    def _famous(self):
        if self._famous_cache is None:
            self._famous_cache = self._eng.famous()
        return self._famous_cache

    def _idx(self):
        if self._idx_cache is None:
            self._idx_cache = self._eng.idx()
        return self._idx_cache

    def _can_see_of(self, i):
        row = self._eng.can_see(i, 1)[0]
        return {self._m2pk[c]: self._i2h[int(k)] for c, k in enumerate(row) if k >= 0}

    # ------------------------------------------------------------------ events
    def is_valid_event(self, h, ev):
        """The host class's checks (signature, id, parent shape: swirld.py:97-108) AND the fork-free contract."""
        if not super().is_valid_event(h, ev):
            return False
        if h in self.hg:                    # already accepted (sync re-checks the remote head after adding it, swirld.py:138)
            return True
        known = self._heads.get(ev.c)
        return known is None if not ev.p else known == ev.p[0]

    def add_event(self, h, ev):
        """hg[h] = ev and its height (swirld.py:114-120); the device copy is batched into the next hot-path call."""
        self.hg[h] = ev
        self.height[h] = 1 + max(self.height[p] for p in ev.p) if ev.p else 0
        self._h2i[h] = len(self._i2h)
        self._i2h.append(h)
        self._heads[ev.c] = h
        self._pending.append(self._h2i[h])
        self._idx_cache = self._famous_cache = None

    # ------------------------------------------------------------------ the hot path (GPU)
    def divide_rounds(self, events):
        """can_see / round / witnesses of the topologically sorted new events (swirld.py:187-222): one sw_divide_rounds."""
        events = tuple(events)
        if not events:
            return
        self._flush()
        first = self._eng.n_divided
        for j, h in enumerate(events):
            if self._h2i[h] != first + j:        # (KeyError for an unknown id, like swirld.py:194)
                raise ValueError("divide_rounds: events must be the new events in arrival order")
        self._eng.divide_rounds(first, len(events))
        self._ops.append(("d", first, len(events)))

    def decide_fame(self):
        """Virtual voting (swirld.py:224-277); returns the set of new consensus rounds."""
        self._flush()
        new_c = set(self._eng.decide_fame())
        self._ops.append(("f",))
        self.consensus |= new_c
        self._famous_cache = None
        return new_c

    def find_order(self, new_c):
        """Consensus order of the events received in the new rounds (swirld.py:280-311)."""
        new_c = sorted(new_c)
        if new_c:
            have = len(self.transactions)
            if hasattr(self._eng, "find_order_out"):     # the order, times and rounds received in one copy
                ev, ts, rr = self._eng.find_order_out(new_c)
                self._tx_ts += ts.tolist()
                self._tx_rr += rr.tolist()
            else:
                added = self._eng.find_order(new_c)
                ev = self._eng.transactions(have, added) if added else ()
            self._ops.append(("o", tuple(new_c)))
            if len(ev):
                new = [self._i2h[int(i)] for i in ev]
                self._order_pos.update((h, have + j) for j, h in enumerate(new))
                self.transactions += new
                self._idx_cache = None
        if self.consensus:
            print(self.consensus)                  # swirld.py:310-311


_bound = {}


def bind(host_cls):
    """The GPU-backed node class over `host_cls` (the reference's `swirld.Node`, or any class with its
    `new_event` / `is_valid_event` / `sync` / `ask_sync` / `main`)."""
    if host_cls not in _bound:
        _bound[host_cls] = type("GpuNode", (GpuConsensus, host_cls), {"__doc__": GpuConsensus.__doc__})
    return _bound[host_cls]


def install(swirld_module):
    """`swirld.Node = bind(swirld.Node)`: the reference's drivers (`swirld.test`, `viz.py`) then run unchanged."""
    if not issubclass(swirld_module.Node, GpuConsensus):
        swirld_module.Node = bind(swirld_module.Node)
    return swirld_module.Node
