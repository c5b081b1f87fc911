"""find_order and the coin on other value columns (tests/column_cases.py, swirld_b200.traces.restamped), on the engine,
against the oracle bit for bit: the order, the consensus times (their bytes), the rounds received, the rounds, the
witness table and fame.

1. every column case under every implementation;
2. one restamped trace through every path that carries t and sig to the device: sw_append from pageable memory (packed
   and per-column copies) and from pinned memory appended ahead, sw_batch_append (packed and large), sw_ingest by id,
   and sw_save / sw_load mid-trace into a larger engine (how GpuNode grows), then on;
3. batch_find_order_out over views of different column kinds, against twins that made the single calls;
4. stake totals: sw_create refuses a total whose triple does not fit in int64, and runs the largest one that does."""
import hashlib

import numpy as np
import pytest

import column_cases as cc
import golden_specs as gs
import test_gpu_order_meta as tom
from fame_cases import RAGGED, Case
from test_gpu_parity import impl  # noqa: F401  (the fixture: default, grid, cluster, wide)
from util import KEYS, assert_same, load_golden

pytestmark = pytest.mark.gpu

_ORACLE = {}


def _oracle(case):
    if repr(case) not in _ORACLE:
        _ORACLE[repr(case)] = cc.run_oracle(case)
    return _ORACLE[repr(case)]


def _check(want, e, got=None, what=""):
    """The engine e (and the output of its find_order_out calls, got) against an oracle run of column_cases.run_oracle."""
    r = e.results()
    assert_same(want["results"], r, KEYS, what)
    assert np.array_equal(r["witness"], want["results"]["witness"]), what + ": witness flags"
    tom._same(want, tom._getters(e), what + " (getters)")
    if got is not None:
        tom._same(want, got, what + " (find_order_out)")


# ---------------------------------------------------------------- 1: the cases
@pytest.mark.parametrize("name", list(cc.CASES))
def test_column_case(name, impl):  # noqa: F811
    case = cc.CASES[name]
    if impl == "wide" and case.M > 64:
        pytest.skip("M > 64 always runs the wide kernels")
    tr = case.trace()
    e, got, _ = tom._run_out(tr, case.schedule(tr.N), case.stakes(), case.C, what=name)
    _check(_oracle(case), e, got, name)
    e.close()


# ---------------------------------------------------------------- 2: the paths that carry t and sig
PATH_CASE = Case("restamped", cc.rs("gossip", "wall", "prefix56_coin", 41, M=16, N=4000), RAGGED)


def _finish(e, sched, start=0):
    for first, cnt in sched[start:]:
        e.divide_rounds(first, cnt)
        e.find_order(e.decide_fame())


def test_append_pageable_packed_and_copied():
    """Calls of at most 64 events go over packed in one block (append_pack, k_unpack), larger ones column by column."""
    from swirld_b200 import engine
    tr = PATH_CASE.trace()
    sched = PATH_CASE.schedule(tr.N)
    assert any(c <= 64 for _, c in sched) and any(c > 64 for _, c in sched)
    e = engine.Engine(tr.M, tr.N)
    for first, cnt in sched:
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        e.find_order(e.decide_fame())
    _check(_oracle(PATH_CASE), e, what="sw_append")


def test_append_ahead_from_pinned_memory():
    import torch
    from swirld_b200 import engine
    tr = PATH_CASE.trace()
    sched = PATH_CASE.schedule(tr.N)
    pin = {k: torch.from_numpy(np.ascontiguousarray(getattr(tr, k))).pin_memory().numpy()
           for k in ("p0", "p1", "creator", "t", "sig")}
    e = engine.Engine(tr.M, tr.N)

    def feed(i):
        s = slice(sched[i][0], sched[i][0] + sched[i][1])
        e.append(pin["p0"][s], pin["p1"][s], pin["creator"][s], pin["t"][s], pin["sig"][s])
    feed(0)
    feed(1)
    for i, (first, cnt) in enumerate(sched):
        e.divide_rounds(first, cnt)
        if i + 2 < len(sched):
            feed(i + 2)
        e.find_order(e.decide_fame())
    _check(_oracle(PATH_CASE), e, what="pinned append-ahead")


@pytest.mark.parametrize("K", [(1, 16, 3, 7, 2, 12, 5, 9, 16, 1, 4), 700], ids=["packed", "large"])
def test_batch_append(K):
    """sw_batch_append of views with different columns: at most 64 events per view go over in one packed block."""
    from swirld_b200 import engine
    cases = [Case("restamped", cc.rs("gossip", t, s, 50 + v, M=16, N=3000 - 100 * v), K)
             for v, (t, s) in enumerate([("wall", "prefix56"), ("const", "prefix16_coin"), ("neg", "prefix60")])]
    trs = [c.trace() for c in cases]
    scheds = [c.schedule(tr.N) for c, tr in zip(cases, trs)]
    engs = [engine.Engine(tr.M, tr.N) for tr in trs]
    for i in range(max(len(s) for s in scheds)):
        live = [v for v in range(len(cases)) if i < len(scheds[v])]
        cols = []
        for v in live:
            s = slice(scheds[v][i][0], sum(scheds[v][i]))
            cols.append((trs[v].p0[s], trs[v].p1[s], trs[v].creator[s], trs[v].t[s], trs[v].sig[s]))
        assert engine.batch_append([engs[v] for v in live], cols) == [scheds[v][i][1] for v in live]
        for v in live:
            engs[v].divide_rounds(*scheds[v][i])
            engs[v].find_order(engs[v].decide_fame())
    for v, c in enumerate(cases):
        _check(_oracle(c), engs[v], what="batch_append view %d" % v)
        engs[v].close()


def test_ingest_by_id():
    """sw_ingest reorders each shuffled batch parents first: t and sig must travel with their event."""
    from swirld_b200 import engine, traces
    base = PATH_CASE.trace()
    N = base.N
    ids = np.stack([np.frombuffer(hashlib.blake2b(b"col%d" % i, digest_size=32).digest(), np.uint8) for i in range(N)])
    zero = np.zeros(32, np.uint8)
    pid = lambda a: np.stack([ids[x] if x >= 0 else zero for x in a])
    e = engine.Engine(base.M, N)
    rng = np.random.default_rng(9)
    arrival = np.full(N, -1, np.int64)
    first = 0
    for cnt in [16, 1, 7, 500, 3, 1473, 2000]:
        batch = rng.permutation(np.arange(first, first + cnt))
        out, m = e.ingest(ids[batch], pid(base.p0[batch]), pid(base.p1[batch]), base.creator[batch], base.t[batch],
                          base.sig[batch])
        assert m == cnt and np.all(out >= 0)
        arrival[batch] = out
        first += cnt
    assert first == N
    order = np.argsort(arrival)
    remap = lambda p: np.where(p >= 0, arrival[np.maximum(p, 0)], -1).astype(np.int32)
    tr = traces.Trace(base.M, remap(base.p0[order]), remap(base.p1[order]), base.creator[order], base.t[order],
                      base.sig[order], "ingested")
    sched = Case("gossip", dict(M=tr.M), 250).schedule(N)
    _finish(e, sched)
    want = order_meta_run(tr, sched)
    _check(want, e, what="sw_ingest")


def order_meta_run(tr, sched, stake=None, C=6):
    import order_meta
    return order_meta.run_oracle_meta(tr, [c for _, c in sched], stake, C, extra=True)


def test_checkpoint_mid_trace_into_a_larger_engine(impl, tmp_path):  # noqa: F811
    """sw_save half way, sw_load with more room, then on: the events appended before the save are ordered after it."""
    from swirld_b200 import engine
    tr = PATH_CASE.trace()
    sched = Case("gossip", dict(M=tr.M), 250).schedule(tr.N)
    half = len(sched) // 2
    e = engine.Engine(tr.M, sched[half][0] + 64)
    e.append_trace(tr, 0, sched[half][0])
    _finish(e, sched[:half])
    p = str(tmp_path / "cols.swb")
    e.save(p)
    e.close()
    e2 = engine.Engine.load(p, capacity=tr.N)
    for first, cnt in sched[half:]:
        e2.append_trace(tr, first, cnt)
        e2.divide_rounds(first, cnt)
        e2.find_order(e2.decide_fame())
    _check(order_meta_run(tr, sched), e2, what="resumed from the checkpoint")


# ---------------------------------------------------------------- 3: batched views of different columns
def test_batch_find_order_out_mixed_columns():
    cases = [Case("restamped", cc.rs("gossip", t, s, 60 + v, M=8, N=1500 - 50 * v), (1, 16, 3, 7, 2, 12, 5, 9, 16, 1, 4))
             for v, (t, s) in enumerate([("wall", "prefix56"), ("huge", "prefix8"), ("tiny", "prefix60_coin"),
                                         ("shuffle", "coin1")])]
    cad, _ = tom._cadence_out(cases)
    for v, c in enumerate(cases):
        _check(_oracle(c), cad.engs[v], what="view %d" % v)


# ---------------------------------------------------------------- 4: stake totals
B = (2 ** 63 - 1) // 3


@pytest.mark.parametrize("stake", [[2 ** 61] * 3 + [1], [B, 1, 0, 0], [2 ** 62, 2 ** 62, 2 ** 62, 2 ** 62]])
def test_create_refuses_a_total_whose_triple_overflows(stake):
    from swirld_b200 import engine
    with pytest.raises(engine.EngineError) as ei:
        engine.Engine(4, 64, stake)
    assert ei.value.code == -1


def test_largest_stake_total_matches_the_reference():
    from swirld_b200 import engine
    name = "g1_m4_n600_s31_k7_bigstake"
    tr, K, stake = gs.make_trace(name)
    assert sum(stake) == B
    r = engine.run_engine(tr, K, stake)
    assert_same(load_golden(name), r, what=name)
    assert (r["round"] == 0).all() and len(r["transactions"]) == 0
