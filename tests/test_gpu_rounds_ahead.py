"""The rounds run ahead on their own stream (SW_ROUNDS_AHEAD, M <= 64, calls that go to the cluster round kernel): a
call whose can_see rows reach beyond its end starts the round kernels of the next piece, which run beside the call's
fame kernels.  Every case runs an engine with the round stream and a twin without it (SW_ROUNDS_AHEAD=0) through the
same calls, and after every call compares what a caller can read -- every result array, the round top, the counters
of sw_stats -- array for array, then checks the engine against the oracle."""
import numpy as np
import pytest

from util import assert_same

pytestmark = pytest.mark.gpu

COUNTERS = ("kernel_launches", "h2d_bytes", "d2h_bytes", "events", "events_divided", "rounds_cluster_launches")


def _pair(monkeypatch, M, N, stake=None, C=6):
    from swirld_b200 import engine
    monkeypatch.setenv("SW_ROUNDS_AHEAD", "1")
    a = engine.Engine(M, N, stake, C)
    monkeypatch.setenv("SW_ROUNDS_AHEAD", "0")
    b = engine.Engine(M, N, stake, C)
    monkeypatch.delenv("SW_ROUNDS_AHEAD")
    return a, b


def _state(e):
    r = e.results()
    r.update(max_round=e.max_round, n_divided=e.n_divided, n_tx=e.n_transactions,
             idx=e.idx(), times=e.consensus_times(), rr=e.rounds_received())
    st = e.stats()
    r.update({k: st[k] for k in COUNTERS})
    return r


def _same(a, b, what):
    sa, sb = _state(a), _state(b)
    assert sa.keys() == sb.keys()
    for k in sa:
        assert np.array_equal(np.asarray(sa[k]), np.asarray(sb[k])), "%s: %s differs from the twin's" % (what, k)


def _call(e, first, cnt):
    e.divide_rounds(first, cnt)
    nc = e.decide_fame()
    e.find_order(nc)
    return sorted(nc)


def _run(a, b, sched, what):
    """The schedule on both engines, compared after every call; new_c per call of the ahead engine."""
    ncs = []
    for i, (first, cnt) in enumerate(sched):
        nc = _call(a, first, cnt)
        assert nc == _call(b, first, cnt), "%s: call %d: new_c differs" % (what, i)
        _same(a, b, "%s, call %d" % (what, i))
        ncs.append(nc)
    return ncs


def _oracle(tr, sched, stake=None, C=6):
    import oracle as orc
    o = orc.Oracle(tr.M, stake, C)
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


def _check(tr, sched, a, ncs, stake=None, C=6, what=""):
    got = a.results()
    got["new_c_per_call"] = ncs
    assert_same(_oracle(tr, sched, stake, C), got, what=what)


def _went_ahead(a, b):
    """The ahead engine's round kernels ran on the round stream (they are not timed there); the twin's did not."""
    assert a.stats()["ms_rounds_kernel"] == 0.0 and b.stats()["ms_rounds_kernel"] > 0.0


@pytest.mark.parametrize("M", [4, 16, 33, 64])
@pytest.mark.parametrize("stakes", ["unit", "int"])
def test_append_all_chunked(M, stakes, monkeypatch):
    from swirld_b200 import traces
    tr = traces.gossip(M, 24000, seed=40 + M)
    stake = None if stakes == "unit" else [1 + (c * 7) % 3 for c in range(M)]
    a, b = _pair(monkeypatch, M, tr.N, stake)
    for e in (a, b):
        e.append_trace(tr)
    sched = list(traces.chunks(tr.N, 4096))
    ncs = _run(a, b, sched, "M=%d %s" % (M, stakes))
    _went_ahead(a, b)
    _check(tr, sched, a, ncs, stake, what="M=%d %s" % (M, stakes))


def test_partition_hand_over_inside_a_piece(monkeypatch):
    """A majority split at M = 64 with the trace appended first: the pieces that run ahead reach chains more than 32
    rounds behind, and the cluster kernel hands them to k_rounds_batch on the round stream."""
    import shape_cases as sc
    from swirld_b200 import traces
    case = sc.CASES["part_m64_major"]
    tr = case.trace()
    a, b = _pair(monkeypatch, tr.M, tr.N, case.stakes(), case.C)
    for e in (a, b):
        e.append_trace(tr)
        e.debug_counters()                          # (cleared)
    sched = list(traces.chunks(tr.N, case.K))
    ncs = _run(a, b, sched, "part_m64_major")
    _went_ahead(a, b)
    assert a.debug_counters()[15] > 0, "the cluster round kernel never handed a piece over"
    _check(tr, sched, a, ncs, case.stakes(), case.C, what="part_m64_major")


def test_ragged_calls(monkeypatch):
    """Calls smaller and larger than the piece the call before started, a call below the cluster kernel's size (the
    round stream's piece is given up), one of 10 events, and appends between the calls."""
    from swirld_b200 import traces
    tr = traces.gossip(33, 40000, seed=7)
    sizes = [3000, 5000, 2100, 9000, 2500, 500, 4000, 10, 6000, 2048]
    sched, first = [], 0
    for s in sizes:
        sched.append((first, s))
        first += s
    sched.append((first, tr.N - first))
    a, b = _pair(monkeypatch, tr.M, tr.N)
    for e in (a, b):
        e.append_trace(tr, 0, 30000)
    ncs = []
    for i, (first, cnt) in enumerate(sched):
        if first + cnt > 30000 and a.n_events < tr.N:
            for e in (a, b):
                e.append_trace(tr, 30000, tr.N - 30000)
        nc = _call(a, first, cnt)
        assert nc == _call(b, first, cnt), "ragged: call %d: new_c differs" % i
        _same(a, b, "ragged, call %d" % i)
        ncs.append(nc)
    # (the 500- and 10-event calls run their round kernels on the compute stream, timed, in both engines)
    assert a.stats()["ms_rounds_kernel"] < b.stats()["ms_rounds_kernel"]
    _check(tr, sched, a, ncs, what="ragged")


def test_rewind_mid_trace(monkeypatch):
    from swirld_b200 import traces
    tr = traces.gossip(64, 30000, seed=11)
    a, b = _pair(monkeypatch, tr.M, tr.N)
    for e in (a, b):
        e.append_trace(tr)
    sched = list(traces.chunks(tr.N, 4096))
    _run(a, b, sched[:3], "before the rewind")
    for e in (a, b):
        e.rewind()
    sched2 = list(traces.chunks(tr.N, 6000))
    ncs = _run(a, b, sched2, "after the rewind")
    _check(tr, sched2, a, ncs, what="after the rewind")


def test_checkpoint_with_a_piece_in_flight(monkeypatch, tmp_path):
    """sw_save right after a call that started the next piece: the file's bytes are the twin's, and the engine loaded
    from it goes on like the twin."""
    from swirld_b200 import engine, traces
    tr = traces.gossip(16, 30000, seed=12)
    a, b = _pair(monkeypatch, tr.M, tr.N)
    for e in (a, b):
        e.append_trace(tr)
    sched = list(traces.chunks(tr.N, 4096))
    ncs = _run(a, b, sched[:3], "before the checkpoint")
    pa, pb = tmp_path / "ahead.ckpt", tmp_path / "twin.ckpt"
    a.save(str(pa))
    b.save(str(pb))
    assert pa.read_bytes() == pb.read_bytes(), "the checkpoint differs from the twin's"
    ncs += _run(a, b, sched[3:5], "after the checkpoint")
    monkeypatch.setenv("SW_ROUNDS_AHEAD", "1")
    c = engine.Engine.load(str(pa))
    monkeypatch.setenv("SW_ROUNDS_AHEAD", "0")
    b2 = engine.Engine.load(str(pb))
    monkeypatch.delenv("SW_ROUNDS_AHEAD")
    ncs_c = _run(c, b2, sched[3:], "loaded")
    assert ncs_c[:2] == ncs[3:5]
    _check(tr, sched, c, ncs[:3] + ncs_c, what="loaded")


def test_batched_calls_on_a_view_with_a_piece_ahead(monkeypatch):
    """sw_batch_decide_fame, sw_batch_find_order and sw_batch_divide_rounds on a view whose last single call started
    the next piece: the batched calls wait for the piece and give it up; single calls after them start again."""
    from swirld_b200 import engine, traces
    tr = traces.gossip(64, 30000, seed=13)
    a, b = _pair(monkeypatch, tr.M, tr.N)
    for e in (a, b):
        e.append_trace(tr)
    sched = list(traces.chunks(tr.N, 4096))
    ncs = []
    for i, (first, cnt) in enumerate(sched):
        if i % 3 == 1:
            for e in (a, b):
                e.divide_rounds(first, cnt)
            nc = engine.batch_decide_fame([a])[0]
            assert nc == engine.batch_decide_fame([b])[0]
            engine.batch_find_order([a], [nc])
            engine.batch_find_order([b], [nc])
        elif i % 3 == 2:
            engine.batch_divide_rounds([a], [first], [cnt])
            engine.batch_divide_rounds([b], [first], [cnt])
            nc = engine.batch_decide_fame([a])[0]
            assert nc == engine.batch_decide_fame([b])[0]
            engine.batch_find_order([a], [nc])
            engine.batch_find_order([b], [nc])
        else:
            nc = _call(a, first, cnt)
            assert nc == _call(b, first, cnt)
        _same(a, b, "batched, call %d" % i)
        ncs.append(sorted(nc))
    _check(tr, sched, a, ncs, what="batched")
