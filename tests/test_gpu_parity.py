"""Parity tests proper: the CUDA engine, called through the C ABI
(libswirld_b200.so via ctypes), against the oracle on the same seeded traces and
call schedules, and against the committed reference fixtures.  Integer / index
work: bit-exact, no tolerance."""
import hashlib

import numpy as np
import pytest

import golden_specs as gs
import oracle as orc
from util import assert_same, load_golden, witness_flags_from_table

pytestmark = pytest.mark.gpu

ALL = list(gs.SPECS)


@pytest.fixture(params=["default", "grid", "cluster", "wide"])
def impl(request, monkeypatch):
    """The implementations of the path (all read by sw_create): "default" = the M <= 64 kernels with the cluster
    round kernel (swirld_rcluster.cuh) for chunks of >= 2048 events and the grid-wide one (swirld_rounds.cuh) below;
    "grid" = the grid-wide round kernel only; "cluster" = the cluster round kernel for every batch call; "wide" = the
    any-M kernels of swirld_wide.cuh, which SW_FORCE_WIDE=1 selects for M <= 64 too."""
    monkeypatch.setenv("SW_FORCE_WIDE", "1" if request.param == "wide" else "0")
    monkeypatch.setenv("SW_ROUNDS_CLUSTER", "0" if request.param == "grid" else "1")
    if request.param == "cluster":
        monkeypatch.setenv("SW_RC_MIN_N", "1")
    else:
        monkeypatch.delenv("SW_RC_MIN_N", raising=False)
    return request.param


def _run(tr, K, stake=None):
    from swirld_b200 import engine
    return engine.run_engine(tr, K, stake)


def _check_round_kernel(impl, tr, K, r):
    """The round kernel the fixture selected is the one that ran: "cluster" launches k_rounds_cluster for every
    divide_rounds call above the one-launch size (16 events) at M <= 64; "grid" and "wide" never do."""
    n = r["stats"]["rounds_cluster_launches"]
    if impl == "cluster" and tr.M <= 64 and K > 16:
        assert n > 0, "the cluster round kernel did not run (the device could not hold its 16-CTA cluster)"
    if impl in ("grid", "wide"):
        assert n == 0


@pytest.mark.parametrize("name", ALL)
def test_engine_matches_reference_fixture(name, impl):
    tr, K, stake = gs.make_trace(name)
    if impl == "wide" and tr.M > 64:
        pytest.skip("M > 64 always runs the wide kernels")
    g = load_golden(name)
    r = _run(tr, K, stake)
    _check_round_kernel(impl, tr, K, r)
    assert_same(g, r, what=name)
    assert bytes(g["can_see_sha256"]) == hashlib.sha256(r["can_see"].tobytes()).digest(), name + ": can_see differs"
    assert np.array_equal(witness_flags_from_table(g["witness_table"], tr.N), r["witness"])


@pytest.mark.parametrize("M,N,K,seed", [
    (2, 300, 1, 1), (3, 500, 5, 2), (4, 1500, 1, 7), (5, 1500, 3, 8), (8, 4000, 64, 9), (13, 5000, 100, 10),
    (31, 6000, 999, 11), (32, 6000, 1000, 12), (33, 6000, 1001, 13), (48, 8000, 8000, 14), (64, 12000, 3000, 15)])
def test_engine_matches_oracle_gossip(M, N, K, seed, impl):
    from swirld_b200 import traces
    tr = traces.gossip(M, N, seed)
    o = orc.run_oracle(tr, K)
    r = _run(tr, K)
    _check_round_kernel(impl, tr, K, r)
    assert_same(o, r, what=tr.name)
    assert np.array_equal(o["oracle"].can_see(), r["can_see"])


@pytest.mark.parametrize("M,N,K,seed,pc,ps", [
    (4, 3000, 1, 21, 0.1, 0.3), (6, 4000, 17, 22, 0.05, 0.5), (16, 9000, 300, 23, 0.01, 0.3),
    (40, 9000, 2048, 24, 0.02, 0.4), (64, 12000, 4096, 25, 0.03, 0.3)])
def test_engine_matches_oracle_adversarial(M, N, K, seed, pc, ps, impl):
    from swirld_b200 import traces
    tr = traces.adversarial(M, N, seed, pc, ps)
    o = orc.run_oracle(tr, K)
    r = _run(tr, K)
    assert_same(o, r, what=tr.name)
    assert np.array_equal(o["oracle"].can_see(), r["can_see"])


@pytest.mark.parametrize("M,N,K,seed", [(8, 3000, 40, 31), (64, 10000, 2500, 32)])
def test_engine_matches_oracle_tick_and_tied(M, N, K, seed, impl):
    from swirld_b200 import traces
    for tr in (traces.tick(M, N, seed), traces.gossip(M, N, seed, tied=16)):
        o = orc.run_oracle(tr, K)
        r = _run(tr, K)
        assert_same(o, r, what=tr.name)


def _late_joiner(M, N, join_at, seed):
    from swirld_b200 import traces
    return traces.late_joiner(M, N, join_at, seed)


@pytest.mark.parametrize("M,N,join_at,K", [(9, 6000, 3000, 6000), (9, 6000, 3000, 2500), (33, 20000, 14000, 4096)])
def test_engine_late_joiner_hands_over(M, N, join_at, K, impl):
    """A chain that starts > 32 rounds behind: the cluster round kernel hands the chunk to the grid-wide one."""
    tr = _late_joiner(M, N, join_at, 77)
    o = orc.run_oracle(tr, K)
    assert int(o["round"].max()) > 40
    r = _run(tr, K)
    assert_same(o, r, what=tr.name)
    assert np.array_equal(o["oracle"].can_see(), r["can_see"])


def test_engine_stake_and_coin_period(impl):
    from swirld_b200 import engine, traces
    tr = traces.gossip(9, 4000, 41)
    stake = [2, 1, 1, 1, 1, 1, 1, 1, 1]
    for C in (6, 3, 2):
        o = orc.run_oracle(tr, 25, stake, C)
        r = engine.run_engine(tr, 25, stake, C)
        assert_same(o, r, what="stake C=%d" % C)


def test_engine_rejects_bad_events():
    from swirld_b200 import engine
    e = engine.Engine(3, 64)
    sig = np.zeros((1, 64), np.uint8)
    t = np.zeros(1)
    e.append([-1], [-1], [0], t, sig)
    e.append([-1], [-1], [1], t, sig)
    with pytest.raises(engine.EngineError) as ei:      # second root of member 0: fork
        e.append([-1], [-1], [0], t, sig)
    assert ei.value.code == -7
    with pytest.raises(engine.EngineError) as ei:      # other-parent by the same creator
        e.append([0], [0], [0], t, sig)
    assert ei.value.code == -6
    with pytest.raises(engine.EngineError) as ei:      # unknown parent
        e.append([0], [5], [0], t, sig)
    assert ei.value.code == -6
    e.append([0], [1], [0], t, sig)
    with pytest.raises(engine.EngineError) as ei:      # self-parent is not the head: fork
        e.append([0], [1], [0], t, sig)
    assert ei.value.code == -7
    assert e.n_events == 3
    with pytest.raises(KeyError):
        e.divide_rounds(0, 5)
    e.divide_rounds(0, 3)
    assert e.rounds().tolist() == [0, 0, 0]
    assert e.decide_fame() == []


def test_engine_reset_is_clean():
    from swirld_b200 import engine, traces
    tr = traces.gossip(16, 5000, 51)
    e = engine.Engine(16, tr.N)
    outs = []
    for _ in range(2):
        e.reset()
        for first, cnt in traces.chunks(tr.N, 700):
            e.append_trace(tr, first, cnt)
            e.divide_rounds(first, cnt)
            e.find_order(e.decide_fame())
        outs.append(e.results())
    assert_same(outs[0], outs[1], what="reset")


def test_full_size_properties_config2():
    """BASELINE config 2 (16 members, 100k events) at full size: the fixture
    already pins it bit for bit; here the size-independent invariants."""
    from swirld_b200 import traces
    tr = traces.gossip(16, 100000, 1)
    r = _run(tr, 4096)
    _properties(tr, r)


def _properties(tr, r):
    rnd, cs, tx = r["round"], r["can_see"], r["transactions"]
    N, M = tr.N, tr.M
    nz = tr.p0 >= 0
    # rounds never decrease along edges and grow by at most one per event
    pr = np.maximum(rnd[tr.p0[nz]], rnd[tr.p1[nz]])
    assert np.all((rnd[nz] == pr) | (rnd[nz] == pr + 1))
    # can_see: own column is the event itself, every entry is an event of that member, rows dominate parents
    assert np.all(cs[np.arange(N), tr.creator] == np.arange(N))
    valid = cs >= 0
    assert np.all(tr.creator[cs[valid]] == np.nonzero(valid)[1])
    assert np.all(cs[nz] >= np.maximum(cs[tr.p0[nz]], cs[tr.p1[nz]]) - 0)
    # witnesses: exactly the events whose round exceeds their self-parent's (or roots)
    wit = np.ones(N, bool)
    wit[nz] = rnd[nz] > rnd[tr.p0[nz]]
    assert np.array_equal(wit.astype(np.uint8), r["witness"])
    # the consensus order is a permutation of distinct events, parents before children
    assert len(np.unique(tx)) == len(tx)
    pos = np.full(N, -1, np.int64)
    pos[tx] = np.arange(len(tx))
    ordered = tx[tr.p0[tx] >= 0]
    assert np.all(pos[tr.p0[ordered]] >= 0) and np.all(pos[tr.p1[ordered]] >= 0)
    # famous is only ever set on witnesses
    assert np.all(r["witness"][r["famous"] >= 0] == 1)


def test_engine_edge_cases(impl):
    """Empty calls, exact-fit and exhausted capacity, ragged schedules, 64 members x tiny chunks."""
    from swirld_b200 import engine, traces
    tr = traces.gossip(64, 3000, 77)
    e = engine.Engine(64, tr.N)                      # capacity == N exactly
    with pytest.raises(engine.EngineError):          # decide_fame before any witness: max() of an empty dict
        e.decide_fame()
    e.divide_rounds(0, 0)                            # empty chunk: no-op
    assert e.find_order([]) == 0
    o = orc.Oracle(64)
    o.append(tr)
    sizes, first = [1, 2, 3, 5, 64, 1, 1, 700, 31, 33], 0
    i = 0
    while first < tr.N:
        cnt = min(sizes[i % len(sizes)], tr.N - first)
        i += 1
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        o.divide_rounds(first, cnt)
        nc_e, nc_o = e.decide_fame(), o.decide_fame()
        assert sorted(nc_e) == sorted(nc_o)
        e.find_order(nc_e)
        o.find_order(nc_o)
        first += cnt
    assert_same(o.results(), e.results(), what="ragged schedule")
    assert np.array_equal(o.can_see(), e.can_see())
    with pytest.raises(engine.EngineError) as ei:    # one event too many
        e.append([0], [1], [0], np.zeros(1), np.zeros((1, 64), np.uint8))
    assert ei.value.code in (-5, -7, -6)
    with pytest.raises(engine.EngineError):          # M above this build's limit
        engine.Engine(1025, 16)


@pytest.mark.parametrize("M,N,K,gen", [(16, 100000, 4096, "gossip"), (64, 262144, 65536, "gossip"),
                                       (64, 40000, 8192, "adversarial")])
def test_append_everything_first(M, N, K, gen):
    """The bench's resident pattern: every event appended before the first divide_rounds, so can_see is
    scanned for the whole trace at once (hundreds of blocks; 4096-event blocks from 200 000 events on),
    then the same engine is rewound and run again (sw_rewind keeps the columns, clears the consensus)."""
    from swirld_b200 import engine, traces
    from swirld_b200.traces import chunks
    tr = getattr(traces, gen)(M, N, 5)
    o = orc.run_oracle(tr, K)
    e = engine.Engine(M, N)
    e.append_trace(tr)
    for rep in range(2):
        if rep:
            e.rewind()
        for first, cnt in chunks(N, K):
            e.divide_rounds(first, cnt)
            e.decide_fame()
        assert np.array_equal(o["round"], e.rounds()), "rounds differ (pass %d)" % rep
        assert np.array_equal(o["oracle"].can_see(), e.can_see()), "can_see differs (pass %d)" % rep
        r = e.results()
        assert np.array_equal(o["famous"], r["famous"]) and np.array_equal(o["witness"], r["witness"])


@pytest.mark.parametrize("seed", [1, 2, 3, 4, 5])
def test_find_order_with_already_ordered_famous_witness(seed, impl):
    """Traces on which some consensus round has a famous witness that an earlier round already ordered
    (tests/test_order_model.py counts them): k_order_cuts must take the reach over the other witnesses."""
    from swirld_b200 import traces
    tr = traces.adversarial(8, 4000, seed, 0.02, 0.5)
    o = orc.run_oracle(tr, 37)
    r = _run(tr, 37)
    assert_same(o, r, what=tr.name)


# ---------------------------------------------------------------- beyond 64 members (swirld_wide.cuh)
@pytest.mark.parametrize("gen,M,N,K,seed,stake", [
    ("gossip", 65, 9000, 777, 61, None), ("gossip", 100, 16000, 4000, 62, None), ("adversarial", 130, 30000, 8192, 63, None),
    ("tick", 200, 24000, 5000, 64, None), ("gossip", 256, 40000, 16384, 65, None), ("gossip", 300, 36000, 36000, 66, None),
    ("gossip", 72, 9000, 500, 67, "mixed"), ("adversarial", 96, 12000, 1, 68, None),
    # one member past a mask width (NJ = 4, 8, 16, 32): the last 32-bit word of every member mask holds one live bit
    pytest.param("gossip", 97, 12000, 1000, 91, None, id="boundary-97"),
    pytest.param("gossip", 97, 12000, 1000, 91, "mixed", id="boundary-97-mixed"),
    pytest.param("gossip", 129, 16000, 3000, 92, None, id="boundary-129"),
    pytest.param("gossip", 129, 16000, 3000, 92, "mixed", id="boundary-129-mixed"),
    pytest.param("gossip", 257, 30000, 7000, 93, None, id="boundary-257"),
    pytest.param("gossip", 257, 30000, 7000, 93, "mixed", id="boundary-257-mixed"),
    pytest.param("gossip", 513, 40000, 10000, 94, None, id="boundary-513"),
    pytest.param("gossip", 513, 40000, 10000, 94, "mixed", id="boundary-513-mixed")])
def test_wide_engine_matches_oracle(gen, M, N, K, seed, stake):
    from swirld_b200 import traces
    tr = getattr(traces, gen)(M, N, seed)
    if K == 1:
        tr = tr.slice(0, 1500)                   # the reference's own cadence: one event per call
    st = [1 + (i % 5 == 0) + 2 * (i % 7 == 3) for i in range(M)] if stake else None
    o = orc.run_oracle(tr, K, st)
    r = _run(tr, K, st)
    assert_same(o, r, what=tr.name)
    assert np.array_equal(o["oracle"].can_see(), r["can_see"])


def test_wide_engine_1024_members_against_oracle():
    """Config 5's member count on a prefix the literal oracle finishes in about a minute."""
    from swirld_b200 import traces
    tr = traces.gossip(1024, 40000, 9)
    o = orc.run_oracle(tr, 20000)
    r = _run(tr, 20000)
    assert_same(o, r, what=tr.name)
    assert np.array_equal(o["oracle"].can_see(), r["can_see"])


# ---------------------------------------------------------------- the append-ahead pipeline (INTEGRATION.md section 3)
@pytest.mark.parametrize("M,N,K,ahead", [(4, 2000, 50, 2), (16, 30000, 700, 3), (64, 60000, 5000, 2), (96, 30000, 3000, 2)])
def test_append_ahead_from_pinned_memory(M, N, K, ahead):
    """Chunks appended `ahead` calls before their divide_rounds, from page-locked memory (truly asynchronous copies),
    on a fresh engine: small chunks take the lazy can_see scan, which must wait for EVERY appended batch."""
    import torch
    from swirld_b200 import engine, traces
    from swirld_b200.traces import chunks
    tr = traces.gossip(M, N, 71)
    o = orc.run_oracle(tr, K)
    pin = {k: torch.from_numpy(np.ascontiguousarray(getattr(tr, k))).pin_memory().numpy() for k in ("p0", "p1", "creator", "t", "sig")}
    sched = list(chunks(N, K))
    e = engine.Engine(M, N)

    def feed(i):
        first, cnt = sched[i]
        s = slice(first, first + cnt)
        e.append(pin["p0"][s], pin["p1"][s], pin["creator"][s], pin["t"][s], pin["sig"][s])
    for i in range(min(ahead, len(sched))):
        feed(i)
    ncs = []
    for i, (first, cnt) in enumerate(sched):
        e.divide_rounds(first, cnt)
        if i + ahead < len(sched):
            feed(i + ahead)
        nc = e.decide_fame()
        e.find_order(nc)
        ncs.append(sorted(nc))
    r = e.results()
    r["new_c_per_call"] = ncs
    assert_same(o, r, what="append-ahead " + tr.name)
    assert np.array_equal(o["oracle"].can_see(), e.can_see())


def test_lazy_scan_then_eager_scan_without_a_sync():
    """append(small); divide_rounds (lazy scan on the compute stream, asynchronous); append(big) (eager scan on the
    copy stream) with no synchronising call in between: the two scans share scratch and must not overlap."""
    from swirld_b200 import engine, traces
    tr = traces.gossip(32, 40000, 72)
    o = orc.Oracle(32)
    o.append(tr)
    o.divide_rounds(0, tr.N)
    e = engine.Engine(32, tr.N)
    e.append_trace(tr, 0, 3000)
    e.divide_rounds(0, 3000)
    e.append_trace(tr, 3000, 30000)
    e.divide_rounds(3000, 30000)
    e.append_trace(tr, 33000, 7000)
    e.divide_rounds(33000, 7000)
    assert np.array_equal(o.can_see(), e.can_see())
    assert np.array_equal(o.results()["round"], e.rounds())


# ---------------------------------------------------------------- the headline configuration at full length
def test_headline_config3_full_length():
    """64 members x 1 000 000 events, K = 65 536 (BASELINE.json configs[2]) element-wise against the oracle."""
    from swirld_b200 import traces
    tr = traces.gossip(64, 1000000, 1)
    o = orc.run_oracle(tr, 65536)
    r = _run(tr, 65536)
    assert_same(o, r, what="config 3 full length")
    assert np.array_equal(witness_flags_from_table(o["witness_table"], tr.N), r["witness"])
    _properties(tr, r)


# ---------------------------------------------------------------- checkpoint / resume, native ingest (SURVEY.md section 8f-2, 8f-4)
@pytest.mark.parametrize("M,N,K", [(16, 20000, 700), (96, 20000, 3000)])
def test_checkpoint_resume(M, N, K, tmp_path):
    """Half the trace, sw_save, sw_load into a new (larger) engine, the other half on both: the resumed engine, the
    uninterrupted one and the oracle agree on everything, the final order included."""
    from swirld_b200 import engine, traces
    from swirld_b200.traces import chunks
    tr = traces.gossip(M, N, 81)
    o = orc.run_oracle(tr, K)
    sched = list(chunks(N, K))
    half = len(sched) // 2
    e = engine.Engine(M, N)
    ncs = []
    for first, cnt in sched[:half]:
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        ncs.append(sorted(nc))
    path = str(tmp_path / "ckpt.swb")
    e.save(path)
    e2 = engine.Engine.load(path, capacity=N + 1000)
    assert e2.M == M and e2.n_events == e.n_events and e2.n_divided == e.n_divided and e2.n_transactions == e.n_transactions
    assert np.array_equal(e.can_see(), e2.can_see())
    outs = []
    for eng in (e, e2):
        calls = list(ncs)
        for first, cnt in sched[half:]:
            eng.append_trace(tr, first, cnt)
            eng.divide_rounds(first, cnt)
            nc = eng.decide_fame()
            eng.find_order(nc)
            calls.append(sorted(nc))
        r = eng.results()
        r["new_c_per_call"] = calls
        outs.append(r)
    assert_same(o, outs[0], what="uninterrupted")
    assert_same(o, outs[1], what="resumed from the checkpoint")
    assert np.array_equal(o["oracle"].can_see(), e2.can_see())


def test_native_ingest_orders_and_validates():
    """sw_ingest: events by 32-byte id in a shuffled batch -> parents-first order, known ids skipped, forks and orphans
    (and what hangs below them) rejected; consensus on the ingested graph equals the oracle on the same arrival order."""
    import hashlib
    from swirld_b200 import engine, traces
    tr = traces.gossip(12, 6000, 91)
    N = tr.N
    ids = np.stack([np.frombuffer(hashlib.blake2b(b"ev%d" % i, digest_size=32).digest(), np.uint8) for i in range(N)])
    zero = np.zeros(32, np.uint8)
    pid = lambda a: np.stack([ids[x] if x >= 0 else zero for x in a])
    e = engine.Engine(12, N + 8)
    rng = np.random.default_rng(5)
    arrival = np.full(N, -1, np.int64)
    first = 0
    for cnt in [12, 1, 7, 500, 3, 2477, 3000]:
        sl = np.arange(first, first + cnt)
        perm = rng.permutation(sl)                        # the batch arrives in any order
        extra = perm[:min(3, first)] - first if first else perm[:0]
        batch = np.concatenate([perm, rng.integers(0, first, 2) if first else perm[:0]]).astype(np.int64)   # + two known events
        out, m = e.ingest(ids[batch], pid(tr.p0[batch]), pid(tr.p1[batch]), tr.creator[batch], tr.t[batch], tr.sig[batch])
        assert m == cnt and np.all(out >= 0)
        assert np.array_equal(np.sort(out[:cnt]), np.arange(first, first + cnt))      # the new ones got the next indices
        arrival[batch[:cnt]] = out[:cnt]
        assert np.array_equal(out[cnt:], arrival[batch[cnt:]])                        # known ids: their old index
        first += cnt
    assert np.array_equal(e.lookup(ids[:50]), arrival[:50])
    # rejected: a fork (second child on an old self-parent), an orphan (unknown parent), and the orphan's child
    bad_ids = np.stack([np.frombuffer(hashlib.blake2b(b"bad%d" % i, digest_size=32).digest(), np.uint8) for i in range(3)])
    c0 = int(tr.creator[100])
    other = int(np.nonzero(tr.creator[:100] != c0)[0][-1])
    p0s = np.stack([ids[100], bad_ids[2] ^ 0xFF, bad_ids[1]])
    p1s = np.stack([ids[other], ids[other], ids[other]])
    crs = np.array([c0, c0, c0], np.int32)
    out, m = e.ingest(bad_ids, p0s, p1s, crs, np.zeros(3), np.zeros((3, 64), np.uint8))
    assert m == 0 and out.tolist() == [-1, -1, -1] and e.n_events == N
    # consensus on the ingested graph == the oracle on the same arrival order
    order = np.argsort(arrival)
    inv = arrival
    from swirld_b200.traces import Trace
    remap = lambda p: np.where(p >= 0, inv[np.maximum(p, 0)], -1).astype(np.int32)
    tr2 = Trace(12, remap(tr.p0[order]), remap(tr.p1[order]), tr.creator[order], tr.t[order], tr.sig[order], "ingested")
    K = 900
    o = orc.run_oracle(tr2, K)
    from swirld_b200.traces import chunks
    ncs = []
    for f0, cnt in chunks(N, K):
        e.divide_rounds(f0, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        ncs.append(sorted(nc))
    r = e.results()
    r["new_c_per_call"] = ncs
    assert_same(o, r, what="ingested graph")


# ---------------------------------------------------------------- several node-views per launch (SURVEY.md section 8f-3)
@pytest.mark.parametrize("M,N,K,B", [(4, 2000, 50, 5), (16, 30000, 4096, 8), (64, 40000, 8192, 3), (33, 9000, 1500, 40)])
def test_batched_views_match_the_oracle(M, N, K, B):
    """B independent node-views (own traces) advanced together by sw_batch_divide_rounds: every view equals the
    oracle on its own trace and schedule (40 views need more than one cooperative launch at 33 members)."""
    from swirld_b200 import engine, traces
    from swirld_b200.traces import chunks
    trs = [traces.gossip(M, N - 7 * v, 100 + v) for v in range(B)]       # ragged: the views differ in length
    engs = [engine.Engine(M, tr.N) for tr in trs]
    for e, tr in zip(engs, trs):
        e.append_trace(tr)
    ncs = [[] for _ in range(B)]
    scheds = [list(chunks(tr.N, K)) for tr in trs]
    for i in range(max(len(s) for s in scheds)):
        live = [v for v in range(B) if i < len(scheds[v])]
        engine.batch_divide_rounds([engs[v] for v in live], [scheds[v][i][0] for v in live], [scheds[v][i][1] for v in live])
        for v in live:
            nc = engs[v].decide_fame()
            engs[v].find_order(nc)
            ncs[v].append(sorted(nc))
    for v in range(0, B, max(1, B // 6)):
        o = orc.run_oracle(trs[v], K)
        r = engs[v].results()
        r["new_c_per_call"] = ncs[v]
        assert_same(o, r, what="view %d of %d" % (v, B))
        assert np.array_equal(o["oracle"].can_see(), engs[v].can_see())
