"""The round stream's pipeline (SW_ROUNDS_AHEAD, M <= 64): a piece queued ahead covers up to several calls, two stay
queued beyond the last call, pieces shrink back to one call near the end of the rows, and the first call after a rewind
scans its own rows first and the rest beside its piece.  Every case runs an engine with the round stream and a twin
without it (SW_ROUNDS_AHEAD=0) through the same calls, compares everything a caller can read after every call (result
arrays, round top, sw_stats counters), then checks the engine against the oracle."""
import pytest

from test_gpu_rounds_ahead import _call, _check, _pair, _run, _same, _went_ahead

pytestmark = pytest.mark.gpu


def _sched(sizes, N):
    out, first = [], 0
    for s in sizes:
        if first >= N:
            break
        s = min(s, N - first)
        out.append((first, s))
        first += s
    if first < N:
        out.append((first, N - first))
    return out


def _resident(a, b, tr):
    """Everything appended, then rewound: the first call's rows are behind by the whole trace."""
    for e in (a, b):
        e.append_trace(tr)
        e.rewind()
        e.debug_counters()                          # (cleared)


@pytest.mark.parametrize("M", [4, 16, 33, 64])
@pytest.mark.parametrize("stakes", ["unit", "int"])
def test_resident_equal_calls(M, stakes, monkeypatch):
    """Append-all, rewind, then equal calls: the split scan of the first call, pieces of several calls, the shrinking
    tail.  The round stream launches the cluster kernel fewer times than there are calls."""
    from swirld_b200 import traces
    tr = traces.gossip(M, 15 * 2048, seed=60 + M)       # (every call takes the ahead path)
    stake = None if stakes == "unit" else [1 + (c * 5) % 4 for c in range(M)]
    a, b = _pair(monkeypatch, M, tr.N, stake)
    _resident(a, b, tr)
    sched = list(traces.chunks(tr.N, 2048))
    ncs = _run(a, b, sched, "M=%d %s" % (M, stakes))
    _went_ahead(a, b)
    launches = int(a.debug_counters()[7])
    assert 0 < launches < len(sched), "%d cluster launches for %d calls" % (launches, len(sched))
    _check(tr, sched, a, ncs, stake, what="M=%d %s" % (M, stakes))


def test_ragged_calls_across_pieces(monkeypatch):
    """Ragged calls after a rewind, so that piece ends fall inside calls, with a call below the cluster kernel's size
    (500 events: the pieces ahead are given up) and one of 7 events in the middle."""
    from swirld_b200 import traces
    tr = traces.gossip(33, 40000, seed=21)
    a, b = _pair(monkeypatch, tr.M, tr.N)
    _resident(a, b, tr)
    sched = _sched([2100, 5300, 2048, 7700, 3100, 500, 2600, 7, 4100, 2048, 9000, 2300], tr.N)
    ncs = _run(a, b, sched, "ragged")
    _check(tr, sched, a, ncs, what="ragged")


def test_append_while_two_pieces_are_in_flight(monkeypatch):
    """Half the trace appended; once the calls have two pieces queued over it, the rest is appended, and the later
    pieces reach into the new rows."""
    from swirld_b200 import traces
    tr = traces.gossip(64, 40000, seed=22)
    a, b = _pair(monkeypatch, tr.M, tr.N)
    for e in (a, b):
        e.append_trace(tr, 0, 20000)
    sched = list(traces.chunks(tr.N, 2500))
    ncs = []
    for i, (first, cnt) in enumerate(sched):
        if i == 2:
            for e in (a, b):
                e.append_trace(tr, 20000, tr.N - 20000)
        nc = _call(a, first, cnt)
        assert nc == _call(b, first, cnt), "append: call %d: new_c differs" % i
        _same(a, b, "append, call %d" % i)
        ncs.append(nc)
    _check(tr, sched, a, ncs, what="append while in flight")


def test_rewind_mid_piece(monkeypatch):
    from swirld_b200 import traces
    tr = traces.gossip(16, 30000, seed=23)
    a, b = _pair(monkeypatch, tr.M, tr.N)
    _resident(a, b, tr)
    sched = list(traces.chunks(tr.N, 2048))
    _run(a, b, sched[:3], "before the rewind")
    for e in (a, b):
        e.rewind()
    sched2 = list(traces.chunks(tr.N, 3000))
    ncs = _run(a, b, sched2, "after the rewind")
    _check(tr, sched2, a, ncs, what="after the rewind")


def test_checkpoint_with_two_pieces_in_flight(monkeypatch, tmp_path):
    """sw_save right after the first call after a rewind (two pieces of several calls queued behind it): the file's
    bytes are the twin's, and an engine loaded from it goes on like the twin."""
    from swirld_b200 import engine, traces
    tr = traces.gossip(64, 30000, seed=24)
    a, b = _pair(monkeypatch, tr.M, tr.N)
    _resident(a, b, tr)
    sched = list(traces.chunks(tr.N, 2048))
    ncs = _run(a, b, sched[:2], "before the checkpoint")
    pa, pb = tmp_path / "ahead.ckpt", tmp_path / "twin.ckpt"
    a.save(str(pa))
    b.save(str(pb))
    assert pa.read_bytes() == pb.read_bytes(), "the checkpoint differs from the twin's"
    ncs += _run(a, b, sched[2:4], "after the checkpoint")
    monkeypatch.setenv("SW_ROUNDS_AHEAD", "1")
    c = engine.Engine.load(str(pa))
    monkeypatch.setenv("SW_ROUNDS_AHEAD", "0")
    b2 = engine.Engine.load(str(pb))
    monkeypatch.delenv("SW_ROUNDS_AHEAD")
    ncs_c = _run(c, b2, sched[2:], "loaded")
    assert ncs_c[:2] == ncs[2:4]
    _check(tr, sched, c, ncs[:2] + ncs_c, what="loaded")


def test_batched_calls_with_pieces_ahead(monkeypatch):
    """Batched fame, order and divide calls on a view whose single calls queued pieces of several calls ahead: the
    batched calls wait for both pieces and give them up; single calls after them start again."""
    from swirld_b200 import engine, traces
    tr = traces.gossip(64, 30000, seed=25)
    a, b = _pair(monkeypatch, tr.M, tr.N)
    _resident(a, b, tr)
    sched = list(traces.chunks(tr.N, 2048))
    ncs = []
    for i, (first, cnt) in enumerate(sched):
        if i % 4 == 1:
            for e in (a, b):
                e.divide_rounds(first, cnt)
            nc = engine.batch_decide_fame([a])[0]
            assert nc == engine.batch_decide_fame([b])[0]
            engine.batch_find_order([a], [nc])
            engine.batch_find_order([b], [nc])
        elif i % 4 == 3:
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
