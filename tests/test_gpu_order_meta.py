"""What find_order ordered, with each event's consensus timestamp (swirld.py:305) and round received (swirld.py:283),
from the engine: find_order_out / batch_find_order_out and the getters consensus_times / rounds_received.

Pinned to the unmodified reference (tests/golden/meta_*, every M <= 64 implementation and the any-M kernels) and to the
oracle (tests/order_meta.py) on coin rounds, tied times, partitions that heal (calls that order more than the 1024
events that come back with the scalars) and wide member counts.  Every call's output equals the getters' slices, and
every batched view equals a twin engine that made the plain calls.  The output calls make the launches of the plain
calls and one copy back (one more round trip past 1024 events per view); refused calls change nothing; checkpoints
carry the columns (version 2) or report -1 / NaN for what a version-1 file had ordered; GpuNode's views over the engine
equal the oracle's replay of each node, through engine growth."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

import fame_cases as fc
import golden_specs as gs
import node_sim
import order_meta
import shape_cases as sc
import test_gpu_batch_consensus as tbc
from test_gpu_parity import impl  # noqa: F401  (the fixture: default, grid, cluster, wide)

pytestmark = pytest.mark.gpu

ORDER_SPEC = 1024                  # swirld_b200.cu: the events a find_order call brings back with its scalars
SC_COUNT = 8                       # swirld_kernels.cuh: the scalars, in ints
KEYS = ("transactions", "consensus_time", "round_received")
META = sorted(os.path.basename(p)[len("meta_"):-len(".npz")]
              for p in glob.glob(os.path.join(gs.GOLDEN_DIR, "meta_*.npz")))


def _same(a, b, what):
    for k in KEYS:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), "%s: %s differs" % (what, k)


def _getters(e, first=0, n=None):
    return {"transactions": e.transactions(first, n), "consensus_time": e.consensus_times(first, n),
            "round_received": e.rounds_received(first, n)}


def _check_out(e, before, out, what):
    """One call's output is exactly what the getters give for the positions it added."""
    ev, ts, rr = out
    assert e.n_transactions - before == len(ev), what
    assert ev.dtype == np.int32 and ts.dtype == np.float64 and rr.dtype == np.int32
    _same(_getters(e, before, len(ev)), {"transactions": ev, "consensus_time": ts, "round_received": rr}, what)


def _run_out(tr, sched, stake=None, coin=6, what=""):
    """One engine through the schedule with find_order_out at every call; returns it, what the calls output
    (concatenated) and the largest count one call ordered."""
    from swirld_b200 import engine
    e = engine.Engine(tr.M, tr.N, stake, coin)
    outs, most = [], 0
    for i, (first, cnt) in enumerate(sched):
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        before = e.n_transactions
        out = e.find_order_out(nc)
        _check_out(e, before, out, "%s call %d" % (what, i))
        outs.append(out)
        most = max(most, len(out[0]))
    got = {k: np.concatenate([o[j] for o in outs]) if outs else np.empty(0) for j, k in enumerate(KEYS)}
    _same(_getters(e), got, what + ": the outputs vs the whole columns")
    return e, got, most


def _sched(tr, K):
    return fc.Case("gossip", dict(M=tr.M, N=tr.N, seed=0), K).schedule(tr.N)


# ---------------------------------------------------------------- 1: the reference's fixtures
@pytest.mark.parametrize("name", META)
def test_reference_fixture(name, impl):  # noqa: F811
    tr, K, stake = gs.make_trace(name)
    if impl == "wide" and tr.M > 64:
        pytest.skip("M > 64 always runs the wide kernels")
    z = np.load(os.path.join(gs.GOLDEN_DIR, "meta_%s.npz" % name))
    e, got, _ = _run_out(tr, _sched(tr, K), stake, what=name)
    _same({k: z[k] for k in KEYS}, got, name)
    e.close()


# ---------------------------------------------------------------- 2: the oracle
_ORACLE = {}


def _oracle(what, case):
    """The oracle's order, consensus times and rounds received over the case's schedule, once per case."""
    if repr(case) not in _ORACLE:
        tr = case.trace()
        _ORACLE[repr(case)] = order_meta.run_oracle_meta(tr, [c for _, c in case.schedule(tr.N)], case.stakes(), case.C)
    return _ORACLE[repr(case)]


def _vs_oracle(name, case):
    tr = case.trace()
    e, got, most = _run_out(tr, case.schedule(tr.N), case.stakes(), case.C, what=name)
    _same(_oracle(name, case), got, name + " vs the oracle")
    e.close()
    return most


# (coin_nj32_m513_gossip_np_c2 orders nothing in 60 000 events and its oracle is the slowest: left to its fame tests)
FAME = [n for n in fc.CASES if n.startswith(("coin", "tied")) and n != "coin_nj32_m513_gossip_np_c2"]


@pytest.mark.parametrize("name", FAME)
def test_coin_and_tied_cases(name):
    _vs_oracle(name, fc.CASES[name])


HEAL = ["part_m8_even", "part_m8_even_ragged", "part_m8_stake", "part_m97_even"]


@pytest.mark.parametrize("name", HEAL)
def test_partition_heals(name):
    """The rounds the partition held back reach consensus together: one call orders far more than ORDER_SPEC events,
    and the rest comes from the columns."""
    assert _vs_oracle(name, sc.CASES[name]) > ORDER_SPEC


@pytest.mark.parametrize("M,N,K", [(97, 6000, 1500), (129, 8000, 2000), (257, 40000, 8192)])
def test_wide_member_counts(M, N, K):
    """(300 members: tied_m300_gossip above)"""
    _vs_oracle("m%d" % M, tbc._gossip(M, N, 70 + M, K))


# ---------------------------------------------------------------- 3: batched output, views vs getters and twins
def _cadence_out(cases, check_twins=True):
    """The views turn by turn through batch_append, batch_divide_rounds, batch_decide_fame and batch_find_order_out;
    every view's output equals its getters, and a twin per view that made the plain single calls ends identical."""
    from swirld_b200 import engine
    import test_gpu_batch_cadence as tcad
    cad = tcad.Cadence(cases)
    twins = [engine.Engine(tr.M, tr.N, c.stakes(), c.C) for c, tr in zip(cases, cad.trs)]
    outs = [[] for _ in cases]
    while cad.live():
        live = cad.live()
        cad.append(live)
        cad.divide(live)
        ncs = engine.batch_decide_fame([cad.engs[v] for v in live])
        before = [cad.engs[v].n_transactions for v in live]
        got = engine.batch_find_order_out([cad.engs[v] for v in live], ncs)
        for k, v in enumerate(live):
            _check_out(cad.engs[v], before[k], got[k], "view %d turn %d" % (v, cad.i))
            outs[v].append(got[k])
            if check_twins:
                first, cnt = cad.scheds[v][cad.i]
                t = twins[v]
                t.append_trace(cad.trs[v], first, cnt)
                t.divide_rounds(first, cnt)
                assert sorted(t.decide_fame()) == sorted(ncs[k])
                t.find_order(ncs[k])
        cad.i += 1
    for v in range(len(cases)):
        if check_twins:
            _same(_getters(twins[v]), _getters(cad.engs[v]), "view %d vs its twin" % v)
        twins[v].close()
    return cad, outs


@pytest.mark.parametrize("M,N,family", [(4, 600, "default"), (33, 1500, "default"), (64, 2000, "wide"),
                                        (97, 2500, "default")])
@pytest.mark.parametrize("K", [1, 3, (1, 16, 3, 7, 2, 12, 5, 9, 16, 1, 4)], ids=["k1", "k3", "ragged"])
def test_batch_cadence(M, N, family, K, monkeypatch):
    monkeypatch.setenv("SW_FORCE_WIDE", "1" if family == "wide" else "0")
    cases = [tbc._gossip(M, N - 7 * v, 100 + v, K) for v in range(3)]
    cad, _ = _cadence_out(cases)
    _same(_oracle("cad", cases[0]), _getters(cad.engs[0]), "view 0 vs the oracle")


def test_batch_more_views_than_sms():
    n = tbc._n_sm() + 3
    cases = [tbc._gossip(4, 600, 300 + v, 3) for v in range(n)]
    cad, _ = _cadence_out(cases)
    assert any(e.n_transactions > 0 for e in cad.engs)


def test_batch_views_past_the_window():
    """Views that order more than ORDER_SPEC events in one batched call, beside views that order few."""
    cases = [sc.CASES["part_m8_even_ragged"], tbc._gossip(8, 12000, 5, (1, 16, 3, 7, 2, 12, 5, 9, 16, 1, 4))]
    cad, outs = _cadence_out(cases)
    assert max(len(o[0]) for o in outs[0]) > ORDER_SPEC
    for v, c in enumerate(cases):
        _same(_oracle("heal_cad%d" % v, c), _getters(cad.engs[v]), "view %d vs the oracle" % v)


# ---------------------------------------------------------------- 4: launches and copies
def _stats(engs):
    s = [e.stats() for e in engs]
    return sum(x["kernel_launches"] for x in s), sum(x["d2h_bytes"] for x in s)


@pytest.mark.parametrize("wide", ["0", "1"])
def test_counters_single(wide, monkeypatch):
    """Per call: the launches of the plain call; one copy of the scalars and the window (the events the call may order,
    at most ORDER_SPEC); a call that orders more adds exactly the rest."""
    from swirld_b200 import engine
    monkeypatch.setenv("SW_FORCE_WIDE", wide)
    tr = tbc._gossip(8, 8000, 9, 0).trace()
    sched = [(0, 3), (3, 500), (503, 3), (506, 6000), (6506, 1494)]
    a, b = engine.Engine(8, tr.N), engine.Engine(8, tr.N)
    big = False
    for first, cnt in sched:
        for e in (a, b):
            e.append_trace(tr, first, cnt)
            e.divide_rounds(first, cnt)
        nc = a.decide_fame()
        assert sorted(b.decide_fame()) == sorted(nc)
        win = min(ORDER_SPEC, a.n_divided - a.n_transactions)
        la, da = _stats([a])
        lb, db = _stats([b])
        ev, _, _ = a.find_order_out(nc)
        assert b.find_order(nc) == len(ev)
        la2, da2 = _stats([a])
        lb2, db2 = _stats([b])
        assert la2 - la == lb2 - lb
        want = 4 * (SC_COUNT + 4 * win) if nc else 0
        if len(ev) > win:
            want += 16 * (len(ev) - win)
            big = True
        assert da2 - da == want, (first, cnt, len(ev), win)
        assert db2 - db == (4 * SC_COUNT if nc else 0)
    assert big


def test_counters_batch():
    """The batched call: the launches of the plain batched call, one copy of every active view's scalars and window,
    and the rest of the views past the window in one more round trip."""
    from swirld_b200 import engine
    cases = [sc.CASES["part_m8_even_ragged"], tbc._gossip(8, 12000, 5, 700)]
    trs = [c.trace() for c in cases]
    scheds = [c.schedule(tr.N) for c, tr in zip(cases, trs)]
    A = [engine.Engine(8, tr.N) for tr in trs]
    Bp = [engine.Engine(8, tr.N) for tr in trs]
    big = False
    for i in range(max(len(s) for s in scheds)):
        live = [v for v in range(2) if i < len(scheds[v])]
        ncs = {}
        for v in live:
            for e in (A[v], Bp[v]):
                e.append_trace(trs[v], *scheds[v][i])
                e.divide_rounds(*scheds[v][i])
            ncs[v] = A[v].decide_fame()
            assert sorted(Bp[v].decide_fame()) == sorted(ncs[v])
        act = [v for v in live if ncs[v]]
        win = max([min(ORDER_SPEC, A[v].n_divided - A[v].n_transactions) for v in act], default=0)
        la, da = _stats(A)
        lb, db = _stats(Bp)
        got = engine.batch_find_order_out([A[v] for v in live], [ncs[v] for v in live])
        assert engine.batch_find_order([Bp[v] for v in live], [ncs[v] for v in live]) == [len(g[0]) for g in got]
        la2, da2 = _stats(A)
        lb2, db2 = _stats(Bp)
        assert la2 - la == lb2 - lb
        want = 4 * len(act) * (SC_COUNT + 4 * win)
        rest = sum(max(0, len(g[0]) - win) for g in got)
        big |= rest > 0
        assert da2 - da == want + 16 * rest
        assert db2 - db == 4 * len(act) * SC_COUNT
    assert big
    for v in range(2):
        _same(_getters(Bp[v]), _getters(A[v]), "view %d" % v)


# ---------------------------------------------------------------- 5: refusals
def _raw_out(engs, new_c, offsets, cap, B=None):
    from swirld_b200 import engine
    lib = engs[0]._lib
    B = len(engs) if B is None else B
    arr = (C.c_void_p * len(engs))(*[e._h for e in engs])
    flat = np.ascontiguousarray(new_c, np.int32)
    offs = np.ascontiguousarray(offsets, np.int32)
    cnt = np.full(len(engs), 12345, np.int32)
    n = max(1, cap)
    ev, ts, rr = np.zeros(n, np.int32), np.zeros(n, np.float64), np.zeros(n, np.int32)
    oo = np.full(len(engs) + 1, 777, np.int32)
    rc = lib.sw_batch_find_order_out(C.cast(arr, C.c_void_p), B, engine._ptr(flat), engine._ptr(offs), engine._ptr(cnt),
                                     engine._ptr(ev), engine._ptr(ts), engine._ptr(rr), engine._ptr(oo), cap)
    return rc, cnt, oo


def test_refusals_change_nothing():
    from swirld_b200 import engine
    cases = [tbc._gossip(8, 3000, 41, 500), tbc._gossip(8, 2500, 42, 500)]
    trs = [c.trace() for c in cases]
    scheds = [c.schedule(tr.N) for c, tr in zip(cases, trs)]
    engs = [engine.Engine(8, tr.N) for tr in trs]
    for e, tr, s in zip(engs, trs, scheds):
        e.append_trace(tr)
        e.divide_rounds(*s[0])
    ncs = [e.decide_fame() for e in engs]
    need = sum(e.n_divided - e.n_transactions for e in engs)
    flat = sorted(ncs[0]) + sorted(ncs[1])
    offs = [0, len(ncs[0]), len(flat)]
    # cap too small
    rc, cnt, oo = _raw_out(engs, flat, offs, need - 1)
    assert rc == -1 and (cnt == 12345).all() and (oo == 777).all()
    e = engs[0]
    a = np.ascontiguousarray(sorted(ncs[0]), np.int32)
    buf = np.zeros(max(1, need), np.int32), np.zeros(max(1, need), np.float64), np.zeros(max(1, need), np.int32)
    small = e.n_divided - e.n_transactions - 1
    assert e._lib.sw_find_order_out(e._h, engine._ptr(a), a.size, *[engine._ptr(x) for x in buf], small) == -1
    # offsets going down, an unknown round
    rc, cnt, oo = _raw_out(engs, flat, [0, len(flat), len(ncs[0])], need)
    assert rc == -1 and (cnt == 12345).all() and (oo == 777).all()
    rc, cnt, oo = _raw_out(engs, [10 ** 7], [0, 1, 1], need)
    assert rc == -3 and (cnt == 12345).all() and (oo == 777).all()
    bad = np.array([10 ** 7], np.int32)
    assert e._lib.sw_find_order_out(e._h, engine._ptr(bad), 1, *[engine._ptr(x) for x in buf], need) == -3
    assert all(x.n_transactions == 0 for x in engs)
    # nothing ran: each view continues (batched) from where it stood and equals the oracle
    got = engine.batch_find_order_out(engs, ncs)
    for i in range(1, max(len(s) for s in scheds)):
        live = [v for v in range(2) if i < len(scheds[v])]
        for v in live:
            engs[v].divide_rounds(*scheds[v][i])
        got = engine.batch_find_order_out([engs[v] for v in live], engine.batch_decide_fame([engs[v] for v in live]))
    for v, c in enumerate(cases):
        _same(_oracle("refuse%d" % v, c), _getters(engs[v]), "view %d after the refusals" % v)


# ---------------------------------------------------------------- 6: checkpoints
def _continue(e, tr, sched, what):
    outs = []
    for i, (first, cnt) in enumerate(sched):
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        before = e.n_transactions
        out = e.find_order_out(e.decide_fame())
        _check_out(e, before, out, "%s call %d" % (what, i))
        outs.append(out)
    return outs


def test_checkpoint_v2_continues(impl, tmp_path):  # noqa: F811
    from swirld_b200 import engine
    case = tbc._gossip(16, 8000, 12, 700)
    tr = case.trace()
    s = case.schedule(tr.N)
    full, ref, _ = _run_out(tr, s, what="uninterrupted")
    e = engine.Engine(16, tr.N)
    _continue(e, tr, s[:6], "first half")
    p = str(tmp_path / "v2.swb")
    e.save(p)
    e2 = engine.Engine.load(p)
    _same(_getters(e), _getters(e2), "loaded vs saved")
    _continue(e2, tr, s[6:], "after the load")
    _same(ref, _getters(e2), "resumed vs uninterrupted")
    for x in (full, e, e2):
        x.close()


def test_checkpoint_v1_loads(tmp_path):
    from swirld_b200 import engine
    case = tbc._gossip(16, 8000, 12, 700)
    tr = case.trace()
    s = case.schedule(tr.N)
    full, ref, _ = _run_out(tr, s, what="uninterrupted")
    e = engine.Engine(16, tr.N)
    _continue(e, tr, s[:6], "first half")
    n_tx = e.n_transactions
    assert n_tx > 0
    p2, p1 = str(tmp_path / "v2.swb"), str(tmp_path / "v1.swb")
    e.save(p2)
    raw = bytearray(open(p2, "rb").read())
    assert int.from_bytes(raw[8:12], "little") == 2
    tail = (8 + 8 * n_tx) + (8 + 4 * n_tx)           # the two version-2 sections: [u64 bytes][data]
    assert int.from_bytes(raw[len(raw) - tail:len(raw) - tail + 8], "little") == 8 * n_tx
    v1 = raw[:len(raw) - tail]
    v1[8:12] = (1).to_bytes(4, "little")
    open(p1, "wb").write(bytes(v1))
    e1 = engine.Engine.load(p1)
    assert e1.n_transactions == n_tx
    assert np.array_equal(e1.transactions(), e.transactions())
    assert np.isnan(e1.consensus_times()).all() and (e1.rounds_received() == -1).all()
    _continue(e1, tr, s[6:], "after the version-1 load")
    assert np.array_equal(e1.transactions(), ref["transactions"])
    g = _getters(e1, n_tx)
    _same({k: ref[k][n_tx:] for k in KEYS}, g, "positions ordered after the version-1 load")
    for x in (full, e, e1):
        x.close()


# ---------------------------------------------------------------- 7: GpuNode over the engine
def test_node_views_through_growth():
    """A gossip simulation over the real engine, with a small capacity so that every node grows through a checkpoint:
    each node's consensus_time / round_received equal the oracle's replay of its own trace and call schedule."""
    import host_sim
    from swirld_b200 import engine
    nodes = node_sim.run_sim(4, 400, host_cls=host_sim.HostNode, capacity=64, seed=5)
    for nd in nodes:
        assert isinstance(nd._eng, engine.Engine) and nd._capacity > 64
        tr, sizes = node_sim.node_trace(nd)
        want = order_meta.run_oracle_meta(tr, sizes)
        got = {"transactions": np.array([nd._h2i[h] for h in nd.transactions], np.int32),
               "consensus_time": np.array([nd.consensus_time[h] for h in nd.transactions], np.float64),
               "round_received": np.array([nd.round_received[h] for h in nd.transactions], np.int32)}
        assert len(got["transactions"]) > 20
        _same(want, got, "node vs oracle replay")
        _same(want, _getters(nd._eng), "node's engine vs oracle replay")
