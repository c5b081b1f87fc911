"""The reference's main loop (swirld.py:319-328) for several node-views at its own cadence, a handful of events per
call: every turn is one sw_batch_append, one sw_batch_divide_rounds, one sw_batch_decide_fame and one
sw_batch_find_order over the views.  Every view must end exactly where single calls would have left it: views are
checked against the oracle (per-call new_c and can_see included) and against a twin engine that made the same calls one
at a time (every result array byte for byte).  Covered: member counts across the mask widths, views of different stakes
and coin periods in one batch, small and large calls in one batch, append errors that belong to one view, the launch
count per turn, single appends between batched ones, and a checkpoint after batched turns."""
import ctypes as C

import numpy as np
import pytest

import fame_cases as fc
import test_gpu_batch_consensus as tbc
from util import assert_same

pytestmark = pytest.mark.gpu


def _cols(tr, first, cnt):
    s = slice(first, first + cnt)
    return (tr.p0[s], tr.p1[s], tr.creator[s], tr.t[s], tr.sig[s])


class Cadence:
    """The views' calls, turn by turn.  A view whose find_order fails leaves the batch."""

    def __init__(self, cases, engs=None):
        from swirld_b200 import engine
        self.cases = cases
        self.trs = [c.trace() for c in cases]
        self.scheds = [c.schedule(tr.N) for c, tr in zip(cases, self.trs)]
        self.engs = engs or [engine.Engine(tr.M, tr.N, c.stakes(), c.C) for c, tr in zip(cases, self.trs)]
        self.ncs, self.failed = [[] for _ in cases], {}
        self.i = 0

    def live(self):
        return [v for v in range(len(self.cases)) if self.i < len(self.scheds[v]) and v not in self.failed]

    def append(self, views):
        from swirld_b200 import engine
        got = engine.batch_append([self.engs[v] for v in views],
                                  [_cols(self.trs[v], *self.scheds[v][self.i]) for v in views])
        assert got == [self.scheds[v][self.i][1] for v in views]

    def divide(self, views):
        from swirld_b200 import engine
        engine.batch_divide_rounds([self.engs[v] for v in views], [self.scheds[v][self.i][0] for v in views],
                                   [self.scheds[v][self.i][1] for v in views])

    def consensus(self, live):
        from swirld_b200 import engine
        got = engine.batch_decide_fame([self.engs[v] for v in live])
        for v, nc in zip(live, got):
            self.ncs[v].append(sorted(nc))
        try:
            engine.batch_find_order([self.engs[v] for v in live], got)
        except ExceptionGroup as g:
            for ex in g.exceptions:
                self.failed[live[ex.view]] = (self.i, ex)

    def turn(self):
        live = self.live()
        self.append(live)
        self.divide(live)
        self.consensus(live)
        self.i += 1

    def run(self, turns=None):
        while self.live() and (turns is None or turns > 0):
            self.turn()
            turns = None if turns is None else turns - 1
        return self


def _single_rest(cad, v):
    """View v's remaining calls, one at a time."""
    e, tr = cad.engs[v], cad.trs[v]
    for first, cnt in cad.scheds[v][cad.i:]:
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        cad.ncs[v].append(sorted(nc))


def _launches(engs):
    return sum(e.stats()["kernel_launches"] for e in engs)


# ---------------------------------------------------------------- 1: parity at every mask width
RAGGED = (1, 16, 3, 7, 2, 12, 5, 9, 16, 1, 4)
SIZES = [(4, 600, "default"), (16, 800, "default"), (33, 1500, "default"), (64, 2000, "default"),
         (4, 600, "wide"), (16, 800, "wide"), (33, 1500, "wide"), (64, 2000, "wide"),
         (97, 2500, "default"), (129, 3000, "default"), (300, 3000, "default"), (513, 4000, "default")]


@pytest.mark.parametrize("K", [1, 3, RAGGED], ids=["k1", "k3", "ragged"])
@pytest.mark.parametrize("M,N,family", SIZES, ids=["m%d_%s" % (m, f) for m, _, f in SIZES])
def test_cadence_matches_oracle_and_single_calls(M, N, family, K, monkeypatch):
    """Three views of one member count, every turn through the four batched calls ("wide": SW_FORCE_WIDE=1)."""
    monkeypatch.setenv("SW_FORCE_WIDE", "1" if family == "wide" else "0")
    cases = [tbc._gossip(M, N - 7 * v, 100 + v, K) for v in range(3)]
    cad = Cadence(cases).run()
    assert not cad.failed
    tbc._check(cases, cad.engs, cad.ncs, oracle_views={0, 2})


# ---------------------------------------------------------------- 2: stakes and coin periods differ within a batch
def test_mixed_views_m4():
    """A single seer at K = 3 (IndexError at the oracle's call, for that view only), a zero stake at C = 3, one event
    per call at C = 2 and mixed stakes on a ragged schedule, in one batch."""
    seer = fc.Case("gossip", dict(M=4, N=1000, seed=1), 3, [1, 0, 0, 0], 6, ("single_seer",))
    o = tbc._oracle(seer)
    assert o["coverage"]["single_seer"] == 1 and o["raised_at"] >= 0
    cases = [tbc._gossip(4, 900, 11, 3, [2, 1, 1, 0], 3), seer, tbc._gossip(4, 500, 12, 1, None, 2),
             tbc._gossip(4, 700, 13, RAGGED, "mixed", 6)]
    assert tbc._oracle(cases[0])["coverage"]["coin_votes"] > 0
    cad = Cadence(cases).run()
    assert list(cad.failed) == [1]
    call, ex = cad.failed[1]
    assert call == o["raised_at"] and isinstance(ex, IndexError)
    assert cad.ncs[1] == o["new_c_per_call"]
    others = [0, 2, 3]
    tbc._check([cases[v] for v in others], [cad.engs[v] for v in others], [cad.ncs[v] for v in others])


def test_mixed_views_m96():
    """Above 64 members: coin rounds at C = 2, a zero stake at C = 3 and mixed stakes at C = 6, calls of 1-16 events."""
    coin = fc.Case("adversarial", dict(M=96, N=6000, seed=68), RAGGED, None, 2, fc.COIN)
    zero = fc.Case("adversarial", dict(M=96, N=5000, seed=69), 3, "zero", 3)
    mixed = tbc._gossip(96, 4000, 70, RAGGED, "mixed", 6)
    assert not fc.missing(coin, tbc._oracle(coin)["coverage"])
    cases = [coin, zero, mixed]
    cad = Cadence(cases).run()
    assert not cad.failed
    tbc._check(cases, cad.engs, cad.ncs)


# ---------------------------------------------------------------- 3: small and large calls in one batch
def test_small_and_large_calls_m64():
    """A view that brings 2048 events and more in some calls (the cluster round kernel) beside views of 3 events per
    call, one of them with mixed stakes (only the chunk-path views must share a stake shape)."""
    big = tbc._gossip(64, 9000, 21, (3, 2100, 5, 2600, 1, 16, 2048))
    cases = [big, tbc._gossip(64, 1200, 22, 3), tbc._gossip(64, 1000, 23, 3, "mixed")]
    cad = Cadence(cases)
    rc0 = sum(e.stats()["rounds_cluster_launches"] for e in cad.engs)
    cad.run()
    assert not cad.failed
    assert sum(e.stats()["rounds_cluster_launches"] for e in cad.engs) > rc0
    tbc._check(cases, cad.engs, cad.ncs)


def test_large_call_above_64_members_is_refused():
    """At M = 97 a batch with a call of 17 events is refused as a whole; every view then continues with single calls."""
    from swirld_b200.engine import EngineError
    cases = [tbc._gossip(97, 600, 31, 3), tbc._gossip(97, 600, 32, (3,) * 5 + (17,)), tbc._gossip(97, 500, 33, 3)]
    cad = Cadence(cases).run(turns=5)
    live = cad.live()
    cad.append(live)
    before = [cad.engs[v].n_divided for v in live]
    with pytest.raises(EngineError) as ei:
        cad.divide(live)
    assert ei.value.code == -8
    assert [cad.engs[v].n_divided for v in live] == before
    for v in live:
        first, cnt = cad.scheds[v][cad.i]
        e = cad.engs[v]
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        cad.ncs[v].append(sorted(nc))
    cad.i += 1
    for v in live:
        _single_rest(cad, v)
    tbc._check(cases, cad.engs, cad.ncs)


# ---------------------------------------------------------------- 4: append errors belong to their view
def _raw_append(engs, offsets, cols, B=None):
    from swirld_b200 import engine
    arr = (C.c_void_p * max(1, len(engs)))(*[e._h for e in engs])
    rcs = np.full(max(1, len(engs)), 12345, np.int32)
    rc = engs[0]._lib.sw_batch_append(C.cast(arr, C.c_void_p), len(engs) if B is None else B,
                                      engine._ptr(np.ascontiguousarray(offsets, np.int32)),
                                      *[engine._ptr(c) for c in cols], engine._ptr(rcs))
    return rc, rcs


def test_append_errors_stay_with_their_view():
    """A fork (a second root), a bad parent and an exhausted capacity in three views of a batch: those views append
    nothing and raise what sw_append raises, the other two append; argument refusals change nothing."""
    from swirld_b200 import engine
    from swirld_b200.engine import EngineError
    cases = [tbc._gossip(8, 400, 40 + v, 3) for v in range(5)]
    cases[3] = fc.Case("gossip", dict(M=8, N=400, seed=43), 3, slice_to=30)
    engs = [engine.Engine(8, 30 if v == 3 else 400) for v in range(5)]
    cad = Cadence(cases, engs).run(turns=10)
    trs = [c.trace() for c in cases]
    full3 = tbc._gossip(8, 400, 43, 3).trace()
    cols = [list(_cols(trs[v] if v != 3 else full3, *cad.scheds[v][cad.i] if v != 3 else (30, 3))) for v in range(5)]
    n0 = cad.engs[0].n_events
    fork = [c.copy() for c in cols[1]]
    fork[0][0], fork[1][0] = -1, -1                           # a second root of a member that has events
    bad = [c.copy() for c in cols[2]]
    bad[0][1] = cad.engs[2].n_events + 5                      # a self-parent that does not exist yet
    cols[1], cols[2] = fork, bad
    # what sw_append says to the same events on twins in the same state
    twins = []
    for v in (1, 2, 3):
        t = engine.Engine(8, engs[v].capacity)
        for first, cnt in cad.scheds[v][:cad.i]:
            t.append_trace(trs[v], first, cnt)
            t.divide_rounds(first, cnt)
            t.find_order(t.decide_fame())
        twins.append(t)
    want = []
    for t, c in zip(twins, cols[1:4]):
        with pytest.raises(EngineError) as ei:
            t.append(*c)
        want.append((ei.value.code, str(ei.value)))
    # argument refusals: a repeated engine, offsets that go down, no view, a NULL engine
    flat = [np.ascontiguousarray(np.concatenate([c[k].reshape(-1) for c in cols]), dt)
            for k, dt in enumerate((np.int32, np.int32, np.int32, np.float64, np.uint8))]
    offs = np.concatenate([[0], np.cumsum([len(c[0]) for c in cols])])
    counts = [e.n_events for e in cad.engs]
    for views, o, B in [(cad.engs[:4] + [cad.engs[0]], offs, None), (cad.engs, offs[[0, 2, 1, 3, 4, 5]], None),
                        (cad.engs, offs, 0)]:
        rc, rcs = _raw_append(views, o, flat, B)
        assert rc == -1 and (rcs == 12345).all()
    arr = (C.c_void_p * 2)(cad.engs[0]._h, None)
    rcs = np.full(2, 12345, np.int32)
    assert cad.engs[0]._lib.sw_batch_append(C.cast(arr, C.c_void_p), 2, engine._ptr(offs[:3].astype(np.int32)),
                                            *[engine._ptr(c) for c in flat], engine._ptr(rcs)) == -1
    assert (rcs == 12345).all() and [e.n_events for e in cad.engs] == counts
    # the batch with three bad views
    with pytest.raises(ExceptionGroup) as gi:
        engine.batch_append(cad.engs, cols)
    g = gi.value
    assert [ex.view for ex in g.exceptions] == [1, 2, 3]
    assert [(ex.code, str(ex)) for ex in g.exceptions] == want
    assert [x.code for x in g.exceptions] == [-7, -6, -5]
    assert g.results == [3, None, None, None, 3]
    assert cad.engs[0].n_events == n0 + 3 and [cad.engs[v].n_events for v in (1, 2, 3)] == counts[1:4]
    # the good views divide what they appended; views 1 and 2 append their real events in the next batch
    cad.divide([0, 4])
    cad.consensus([0, 4])
    engine.batch_append([cad.engs[1], cad.engs[2]], [_cols(trs[v], *cad.scheds[v][cad.i]) for v in (1, 2)])
    cad.divide([1, 2])
    cad.consensus([1, 2])
    cad.i += 1
    cad.run()
    assert not cad.failed
    tbc._check(cases, cad.engs, cad.ncs)


def test_small_views_leave_the_callers_arrays_free():
    """Packed views are staged before sw_batch_append returns: overwriting the caller's (page-locked) arrays right
    after each call changes no result."""
    import torch
    from swirld_b200 import engine
    cases = [tbc._gossip(16, 600, 50 + v, (3, 16, 1)) for v in range(3)]
    cad = Cadence(cases)
    bufs = [torch.empty(64 * 16 * 3, dtype=dt, pin_memory=True).numpy() for dt in
            (torch.int32, torch.int32, torch.int32, torch.float64, torch.uint8)]
    while cad.live():
        live = cad.live()
        cols = [_cols(cad.trs[v], *cad.scheds[v][cad.i]) for v in live]
        offs = np.concatenate([[0], np.cumsum([len(c[0]) for c in cols])]).astype(np.int32)
        for k in range(5):
            flat = np.concatenate([c[k].reshape(-1) for c in cols])
            bufs[k][:flat.size] = flat
        rc, rcs = _raw_append([cad.engs[v] for v in live], offs, [b for b in bufs])
        assert rc == 0 and (rcs[:len(live)] == 0).all()
        for b in bufs:
            b[:] = 7                                        # (a creator out of range, parents that do not exist)
        cad.divide(live)
        cad.consensus(live)
        cad.i += 1
    assert not cad.failed
    tbc._check(cases, cad.engs, cad.ncs)


# ---------------------------------------------------------------- 5: launches per turn
@pytest.mark.parametrize("M", [33, 129])
def test_launches_per_turn_do_not_grow_with_views(M):
    """A turn's append and divide cost 2 launches summed over all engines, for 1, 64 and n_sm + 3 views."""
    for B in (1, 64, tbc._n_sm() + 3):
        cases = [tbc._gossip(M, 150 - (v % 7), 200 + v, 3) for v in range(B)]
        cad = Cadence(cases).run(turns=4)
        live = cad.live()
        assert len(live) == B
        l0 = _launches(cad.engs)
        cad.append(live)
        cad.divide(live)
        assert _launches(cad.engs) - l0 == 2, (M, B)
        cad.consensus(live)
        cad.i += 1
        cad.run()
        assert not cad.failed
        sample = sorted({0, B // 2, B - 1})
        tbc._check([cases[v] for v in sample], [cad.engs[v] for v in sample], [cad.ncs[v] for v in sample])
        for e in cad.engs:
            e.close()


# ---------------------------------------------------------------- 6: single appends in between, checkpoints
def test_single_appends_between_batched_ones():
    """Turn by turn: every view appends alone; all views in one batch; view 0 alone and the others in a batch."""
    cases = [tbc._gossip(16, 700 - 5 * v, 60 + v, (3, 1, 16, 5)) for v in range(4)]
    cad = Cadence(cases)
    while cad.live():
        live = cad.live()
        mode = cad.i % 3
        single = live if mode == 0 else [v for v in live if v == 0] if mode == 2 else []
        for v in single:
            cad.engs[v].append_trace(cad.trs[v], *cad.scheds[v][cad.i])
        batched = [v for v in live if v not in single]
        if batched:
            cad.append(batched)
        cad.divide(live)
        cad.consensus(live)
        cad.i += 1
    assert not cad.failed
    tbc._check(cases, cad.engs, cad.ncs)


@pytest.mark.parametrize("M,N", [(33, 900), (129, 1200)])
def test_checkpoint_after_batched_turns(M, N, tmp_path):
    """sw_save a view after half its calls went through batched turns, sw_load it and finish with single calls: equal
    to the oracle."""
    from swirld_b200 import engine
    cases = [tbc._gossip(M, N - 7 * v, 300 + v, (3, 1, 16)) for v in range(2)]
    cad = Cadence(cases).run(turns=len(cases[1].schedule(cases[1].trace().N)) // 2)
    path = str(tmp_path / "view1.swb")
    cad.engs[1].save(path)
    cad.engs[1].close()
    cad.engs[1] = engine.Engine.load(path, capacity=cad.trs[1].N)
    _single_rest(cad, 1)
    r = cad.engs[1].results()
    r["new_c_per_call"] = cad.ncs[1]
    o = tbc._oracle(cases[1])
    assert_same(o, r, what="view 1 resumed")
    assert np.array_equal(o["oracle"].can_see(), cad.engs[1].can_see())
