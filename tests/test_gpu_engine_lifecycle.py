"""The engine's buffers grow between ordinary calls, and an engine can be destroyed in any state.  Every buffer that grows
on demand does so here in the middle of a trace, while earlier work may still run on the engine's streams: the cluster
round kernel's rows (a call longer than any before, with two round-stream pieces queued), find_order's per-round
scratch (calls that order more rounds than any before), the batched calls' parameter blocks and the staging ring of
packed appends (batches growing from 1 view to n_sm + 3), and sw_flush_l2's buffer.  sw_destroy runs with pieces
still queued on the round stream, on the first engine of a batch before the other views, and on the failure path of
sw_load.  Every result is compared bit for bit with the oracle on the same trace and call schedule."""
import numpy as np
import pytest

import oracle as orc
from util import assert_same

pytestmark = pytest.mark.gpu


def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sched(sizes, N):
    """Calls of the given sizes, then one for the rest of the trace."""
    out, first = [], 0
    for s in sizes:
        out.append((first, s))
        first += s
    if first < N:
        out.append((first, N - first))
    return out


def _oracle(tr, sched):
    o = orc.Oracle(tr.M)
    o.append(tr)
    ncs = []
    for first, cnt in sched:
        o.divide_rounds(first, cnt)
        nc = o.decide_fame()
        o.find_order(nc)
        ncs.append(sorted(nc))
    r = o.results()
    r["new_c_per_call"] = ncs
    o.close()
    return r


def _call(e, first, cnt):
    e.divide_rounds(first, cnt)
    nc = e.decide_fame()
    ev, ts, rr = e.find_order_out(nc)
    base = e.n_transactions - len(ev)
    assert np.array_equal(ev, e.transactions(base)) and np.array_equal(ts.view(np.uint64), e.consensus_times(base).view(np.uint64))
    assert np.array_equal(rr, e.rounds_received(base))
    return sorted(nc)


def _check(tr, sched, e, ncs, what):
    got = e.results()
    got["new_c_per_call"] = ncs
    assert_same(_oracle(tr, sched), got, what=what)


def _engine(monkeypatch, M, N, ahead):
    from swirld_b200 import engine
    monkeypatch.setenv("SW_ROUNDS_AHEAD", "1" if ahead else "0")
    e = engine.Engine(M, N)
    monkeypatch.delenv("SW_ROUNDS_AHEAD")
    return e


def test_longer_call_with_pieces_queued(monkeypatch):
    """Calls of 2048 events queue two pieces of up to 16384 events on the round stream; the call of 100000 events after
    them needs a piece longer than the 65536 events the cluster kernel's row buffers first hold."""
    from swirld_b200 import traces
    tr = traces.gossip(8, 112000, seed=51)
    sched = _sched([2048] * 4 + [100000], tr.N)
    for ahead in (True, False):
        e = _engine(monkeypatch, tr.M, tr.N, ahead)
        e.append_trace(tr)
        ncs = [_call(e, first, cnt) for first, cnt in sched]
        if ahead:
            assert e.stats()["ms_rounds_kernel"] == 0.0, "the round kernels did not run on the round stream"
        _check(tr, sched, e, ncs, "ahead=%s" % ahead)
        e.close()


def test_order_scratch_and_flush_grow_between_calls():
    """Each call orders more rounds than any call before it (find_order's scratch starts at 64 rounds), and sw_flush_l2
    asks for a larger buffer before each one."""
    from swirld_b200 import engine, traces
    tr = traces.gossip(4, 24000, seed=52)
    sched = _sched([200, 300, 1500, 6000], tr.N)
    e = engine.Engine(tr.M, tr.N)
    e.append_trace(tr)
    ncs, most = [], 0
    for i, (first, cnt) in enumerate(sched):
        e.flush_l2((1 << 20) << (2 * i))
        ncs.append(_call(e, first, cnt))
        most = max(most, len(ncs[-1]))
    assert most > 128 and len(ncs[-1]) == most, "the last call no longer orders the most rounds: %s" % [len(n) for n in ncs]
    _check(tr, sched, e, ncs, "order scratch")


def _turn(engine, views, trs, sizes):
    """One turn of the views v = 0.. of `views`: their next call of sizes(v) events of trace trs[v] through the batched
    calls."""
    cols, firsts, ns = [], [], []
    for v, x in enumerate(views):
        n = sizes(v)
        tr, s = trs[v], slice(x.n_events, x.n_events + n)
        cols.append((tr.p0[s], tr.p1[s], tr.creator[s], tr.t[s], tr.sig[s]))
        firsts.append(x.n_divided)
        ns.append(n)
    assert engine.batch_append(views, cols) == ns
    engine.batch_divide_rounds(views, firsts, ns)
    ncs = engine.batch_decide_fame(views)
    for x, nc, (ev, ts, rr), first, n in zip(views, ncs, engine.batch_find_order_out(views, ncs), firsts, ns):
        assert np.array_equal(ev, x.transactions(x.n_transactions - len(ev)))
        assert np.array_equal(rr, x.rounds_received(x.n_transactions - len(rr)))
        x.sched.append((first, n))
        x.ncs.append(sorted(nc))


def _check_views(engs, trs):
    """Every view against the oracle on its trace so far and its calls (one oracle run per distinct pair)."""
    want = {}
    for x, tr in zip(engs, trs):
        key = (id(tr), tuple(x.sched))
        if key not in want:
            want[key] = _oracle(tr.slice(0, x.n_events), x.sched)
        got = x.results()
        got["new_c_per_call"] = x.ncs
        assert_same(want[key], got, what="view with calls %s" % (x.sched,))


def _views(engine, B, M, N):
    engs = [engine.Engine(M, N) for _ in range(B)]
    for x in engs:
        x.sched, x.ncs = [], []
    return engs


def test_batches_grow_to_more_views_than_sms():
    """Turns of sw_batch_append (packed), sw_batch_divide_rounds (calls of at most 16 events take the one-launch path,
    longer ones the chunk path), sw_batch_decide_fame and sw_batch_find_order_out over more views each turn, up to
    n_sm + 3.  The first engine's parameter blocks and staging ring grow in the middle of its own trace."""
    from swirld_b200 import engine, traces
    M, N = 4, 420
    sizes = [5, 40, 12, 64, 3, 30, 16, 50, 9]
    counts = [1, 2, 3, 8, 20, 50, _n_sm() + 3, _n_sm() + 3, 7]
    base = [traces.gossip(M, N, seed=60 + k) for k in range(3)]
    engs = _views(engine, counts[-2], M, N)
    trs = [base[v % 3] for v in range(len(engs))]
    for t, B in enumerate(counts):
        _turn(engine, engs[:B], trs, lambda v: sizes[(len(engs[v].sched) + v) % len(sizes)])
    assert max(len(x.sched) for x in engs) == len(counts)
    _check_views(engs, trs)


def test_destroy_first_view_of_a_batch():
    """The first engine of a batch owns the batch's buffers and events; destroyed before the others, it leaves them to go
    on alone, in batches and single calls."""
    from swirld_b200 import engine, traces
    M, N = 8, 3000
    trs = [traces.gossip(M, N, seed=70 + k) for k in range(4)]
    engs = _views(engine, 4, M, N)
    for t in range(3):
        _turn(engine, engs, trs, lambda v: [12, 300, 40][(t + v) % 3])
    engs[0].close()
    rest, rtrs = engs[1:], trs[1:]
    for t in range(3):
        _turn(engine, rest, rtrs, lambda v: [500, 16, 64][(t + v) % 3])
    for x in rest:
        x.append_trace(rtrs[rest.index(x)], x.n_events, N - x.n_events)
        x.sched.append((x.n_divided, N - x.n_divided))
        x.ncs.append(_call(x, *x.sched[-1]))
    _check_views(rest, rtrs)


def test_failed_load_of_a_truncated_checkpoint(tmp_path):
    """sw_load of a checkpoint cut in half creates the engine, fails reading it and frees it through sw_destroy; the
    whole file then loads and goes on to the oracle's results."""
    from swirld_b200 import engine, traces
    tr = traces.gossip(16, 20000, seed=54)
    sched = _sched([3000, 3000, 5000], tr.N)
    e = engine.Engine(tr.M, tr.N)
    e.append_trace(tr)
    ncs = [_call(e, first, cnt) for first, cnt in sched[:2]]
    full, cut = tmp_path / "full.ckpt", tmp_path / "cut.ckpt"
    e.save(str(full))
    e.close()
    data = full.read_bytes()
    cut.write_bytes(data[:len(data) // 2])
    with pytest.raises(engine.EngineError, match="truncated"):
        engine.Engine.load(str(cut))
    f = engine.Engine.load(str(full))
    ncs += [_call(f, first, cnt) for first, cnt in sched[2:]]
    _check(tr, sched, f, ncs, "loaded after a failed load")


def test_destroy_with_pieces_queued(monkeypatch):
    """sw_destroy right after a call that queued pieces on the round stream, with no synchronisation; then an engine on
    the same device runs the same trace."""
    from swirld_b200 import traces
    tr = traces.gossip(16, 30000, seed=53)
    sched = _sched([2048] * 5, tr.N)
    a = _engine(monkeypatch, tr.M, tr.N, True)
    a.append_trace(tr)
    for first, cnt in sched[:3]:
        _call(a, first, cnt)
    a.divide_rounds(*sched[3])
    a.close()
    b = _engine(monkeypatch, tr.M, tr.N, True)
    b.append_trace(tr)
    ncs = [_call(b, first, cnt) for first, cnt in sched]
    _check(tr, sched, b, ncs, "after a destroy with pieces queued")
