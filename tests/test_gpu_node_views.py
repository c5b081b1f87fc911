"""The engine on node views: one member's own arrival order of the gossip (traces.node_view), one call per sync --
roots out of member order and late, stale other-parents thousands of events and many calls below the event that reads
them, calls of a few events between bursts of thousands, so that one engine alternates between the streaming kernel,
the batch kernels, the cluster round kernel, the round stream and the eager can_see scan.  The cases are in
tests/view_cases.py (their sizes are asserted on the CPU by tests/test_view_cases.py) and the reference's replays in
tests/golden (golden_specs.NODE_FIXTURES and VIEW_FIXTURES).  Everything is compared bit for bit with the oracle:
rounds, witnesses, fame, consensus, the order with its consensus times and rounds received (from find_order_out at
every call), new_c per call, can_see, heights and idx."""
import hashlib

import numpy as np
import pytest

import golden_specs as gs
import order_meta
import view_cases as vc
from test_gpu_order_meta import KEYS as META_KEYS, _check_out, _same as _same_meta
from test_gpu_rounds_ahead import _pair, _same as _same_twin, _went_ahead
from util import assert_same

pytestmark = pytest.mark.gpu


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


def _sched(calls):
    out, first = [], 0
    for c in calls:
        out.append((first, c))
        first += c
    return out


def _fixture_view(name):
    from swirld_b200.traces import Trace
    z = np.load(gs.path(name))
    return Trace(int(z["M"]), z["p0"], z["p1"], z["creator"], z["t"], z["sig"], name), z["sizes"].tolist(), z


# ---------------------------------------------------------------- the oracle, once per view and schedule
_ORACLE = {}


def _oracle(key, tr, calls, stake=None, C=6):
    """The oracle over the calls: results(), new_c per call, can_see, heights, idx, and the order metadata."""
    if key not in _ORACLE:
        import oracle as orc
        o = orc.Oracle(tr.M, stake, C)
        o.append(tr)
        ncs = []
        for first, cnt in _sched(calls):
            o.divide_rounds(first, cnt)
            nc = o.decide_fame()
            o.find_order(nc)
            ncs.append(sorted(nc))
        r = o.results()
        h, idx = np.empty(tr.N, np.int32), np.empty(tr.N, np.int32)
        orc.lib().or_get_height(o._h, h)
        orc.lib().or_get_idx(o._h, idx)
        r.update(new_c_per_call=ncs, can_see=o.can_see(), heights=h, idx=idx,
                 meta=order_meta.run_oracle_meta(tr, list(calls), stake, C))
        o.close()
        _ORACLE[key] = r
    return _ORACLE[key]


def _check(o, e, tr, ncs, meta, what):
    """The engine e against the oracle's run o."""
    from swirld_b200 import traces
    r = e.results()
    r["new_c_per_call"] = ncs
    assert_same(o, r, what=what)
    assert np.array_equal(o["witness"], r["witness"]), what + ": witness flags differ"
    assert np.array_equal(o["can_see"], e.can_see()), what + ": can_see differs"
    h = e.heights()
    assert np.array_equal(o["heights"], h), what + ": heights differ from the oracle's"
    assert np.array_equal(traces.heights(tr), h), what + ": heights differ from traces.heights"
    assert np.array_equal(o["idx"], e.idx()), what + ": idx differs"
    if meta is not None:
        _same_meta(o["meta"], meta, what + ": order metadata")


def _run(tr, calls, stake=None, C=6, resident=False, what=""):
    """One engine through the calls (each call appends its own events, or everything first), find_order_out at
    every call; returns the engine, new_c per call and the concatenated order metadata."""
    from swirld_b200 import engine
    e = engine.Engine(tr.M, tr.N, stake, C)
    if resident:
        e.append_trace(tr)
    ncs, outs = [], []
    for i, (first, cnt) in enumerate(_sched(calls)):
        if not resident:
            e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        before = e.n_transactions
        out = e.find_order_out(nc)
        _check_out(e, before, out, "%s call %d" % (what, i))
        ncs.append(sorted(nc))
        outs.append(out)
    meta = {k: np.concatenate([o[j] for o in outs]) for j, k in enumerate(META_KEYS)}
    return e, ncs, meta


def _cluster_ran(impl, M, calls, e):
    """Under "cluster" every call above 16 events at M <= 64 launches k_rounds_cluster; "grid" and "wide" never do."""
    n = e.stats()["rounds_cluster_launches"]
    if impl == "cluster" and M <= 64 and max(calls) > vc.SMALL:
        assert n > 0, "the cluster round kernel did not run"
    if impl in ("grid", "wide"):
        assert n == 0


# ---------------------------------------------------------------- a. the reference's node fixtures
FIXTURES = gs.NODE_FIXTURES + list(gs.VIEW_FIXTURES)


@pytest.mark.parametrize("name", FIXTURES)
def test_node_fixture(name, impl):
    """Two nodes of a live 4-member simulation and three node views at 8, 16 and 33 members, one call per sync: the
    engine equals the reference's replay and the oracle's."""
    tr, sizes, z = _fixture_view(name)
    e, ncs, meta = _run(tr, sizes, what=name)
    for k in ("round", "famous", "consensus", "transactions"):
        assert np.array_equal(z[k], e.results()[k]), "%s: %s differs from the reference's" % (name, k)
    _check(_oracle(name, tr, tuple(sizes)), e, tr, ncs, meta, name)
    _cluster_ran(impl, tr.M, sizes, e)
    e.close()


# ---------------------------------------------------------------- b. the view cases
@pytest.mark.parametrize("name", list(vc.CASES))
def test_view_case(name, impl):
    case = vc.CASES[name]
    if case.M > 64 and impl != "default":
        pytest.skip("M > 64 always runs the wide kernels")
    tr, calls = case.trace(), case.calls()
    e, ncs, meta = _run(tr, calls, case.stakes(), case.C, case.resident, what=name)
    _check(_oracle(name, tr, tuple(calls), case.stakes(), case.C), e, tr, ncs, meta, "%s [%s]" % (name, impl))
    _cluster_ran(impl, tr.M, calls, e)
    e.close()


# ---------------------------------------------------------------- c. the round stream
AHEAD = [n for n, c in vc.CASES.items() if c.M <= 64 and max(c.calls()) >= vc.LARGE]


def _coarse(calls):
    """Runs of consecutive calls joined until each holds at least LARGE events (the tail joins the last run): every
    call then goes to the cluster round kernel, whose next piece the round stream rounds ahead."""
    out, acc = [], 0
    for c in calls:
        acc += c
        if acc >= vc.LARGE:
            out.append(acc)
            acc = 0
    if acc:
        out[-1:] = [out[-1] + acc] if out else [acc]
    return out


@pytest.mark.parametrize("kind", ["calls", "coarse"])
@pytest.mark.parametrize("name", AHEAD)
def test_round_stream(name, kind, monkeypatch):
    """The whole view appended first, then the case's calls ("calls": bursts between calls of a few events) or runs
    of them of at least 2048 events each ("coarse": the round stream rounds every next piece ahead), on an engine with
    the round stream and a twin without, compared after every call: the pieces rounded ahead hold late roots, chains
    far behind and stale parents thousands of events below."""
    case = vc.CASES[name]
    tr, calls = case.trace(), case.calls()
    if kind == "coarse":
        calls = _coarse(calls)
    a, b = _pair(monkeypatch, tr.M, tr.N, case.stakes(), case.C)
    for e in (a, b):
        e.append_trace(tr)
    ncs = []
    for i, (first, cnt) in enumerate(_sched(calls)):
        nc = []
        for e in (a, b):
            e.divide_rounds(first, cnt)
            nc.append(sorted(e.decide_fame()))
            e.find_order(nc[-1])
        assert nc[0] == nc[1], "%s: call %d: new_c differs" % (name, i)
        _same_twin(a, b, "%s, call %d" % (name, i))
        ncs.append(nc[0])
    if kind == "coarse":
        _went_ahead(a, b)
    _check(_oracle((name, kind), tr, tuple(calls), case.stakes(), case.C), a, tr, ncs, None, "%s %s ahead" % (name, kind))


# ---------------------------------------------------------------- d. every view of one simulation, batched
def _getall(e):
    r = e.results()
    r.update(can_see=e.can_see(), heights=e.heights(), idx=e.idx(), times=e.consensus_times(), rr=e.rounds_received())
    return r


@pytest.mark.parametrize("gen,kw,every", [
    ("partition", dict(M=8, N=12000, seed=4, split=4, start=2000, end=8000), 1),
    ("gossip", dict(M=33, N=6000, seed=8), 1),
    ("gossip", dict(M=97, N=6000, seed=9), 8),
])
def test_views_of_one_simulation_batched(gen, kw, every):
    """The views of one base (every member's, or every `every`-th above 64 members) turn by turn: one batch_append,
    one batch_divide_rounds, one batch_decide_fame and one batch_find_order_out over the live views, whose calls
    differ in size, so one batched divide holds streaming and chunk-path views.  Above 64 members only calls of at
    most 16 events may be batched; the others are single calls on the same engines in the same turn.  Every view
    equals a twin driven by single calls byte for byte, and every third view the oracle."""
    from swirld_b200 import engine, traces
    base = getattr(traces, gen)(**kw)
    M = base.M
    views = traces.node_views(base)[::every]
    V = len(views)
    engs = [engine.Engine(M, tr.N) for tr, _ in views]
    twins = [engine.Engine(M, tr.N) for tr, _ in views]
    scheds = [_sched(sizes) for _, sizes in views]
    ncs = [[] for _ in range(V)]
    outs = [[] for _ in range(V)]
    mixed = 0
    for t in range(max(len(s) for s in scheds)):
        live = [v for v in range(V) if t < len(scheds[v])]
        cols = []
        for v in live:
            tr, (first, cnt) = views[v][0], scheds[v][t]
            s = slice(first, first + cnt)
            cols.append((tr.p0[s], tr.p1[s], tr.creator[s], tr.t[s], tr.sig[s]))
        engine.batch_append([engs[v] for v in live], cols)
        batched = [v for v in live if M <= 64 or scheds[v][t][1] <= vc.SMALL]
        single = [v for v in live if v not in batched]
        if batched:
            engine.batch_divide_rounds([engs[v] for v in batched], [scheds[v][t][0] for v in batched],
                                       [scheds[v][t][1] for v in batched])
            n_small = sum(scheds[v][t][1] <= vc.SMALL for v in batched)
            mixed += 0 < n_small < len(batched)
        for v in single:
            engs[v].divide_rounds(*scheds[v][t])
        nc = engine.batch_decide_fame([engs[v] for v in live])
        out = engine.batch_find_order_out([engs[v] for v in live], nc)
        for k, v in enumerate(live):
            ncs[v].append(sorted(nc[k]))
            outs[v].append(out[k])
            tw = twins[v]
            tr, (first, cnt) = views[v][0], scheds[v][t]
            tw.append_trace(tr, first, cnt)
            tw.divide_rounds(first, cnt)
            tnc = tw.decide_fame()
            assert sorted(tnc) == ncs[v][-1], "view %d, turn %d: new_c differs from the single calls'" % (v, t)
            tout = tw.find_order_out(tnc)
            for x, y in zip(out[k], tout):
                assert x.tobytes() == y.tobytes(), "view %d, turn %d: find_order_out differs" % (v, t)
    if M <= 64:
        assert mixed > 0, "no batched divide held both streaming and chunk-path views"
    for v in range(V):
        a, b = _getall(engs[v]), _getall(twins[v])
        for k in a:
            x, y = np.asarray(a[k]), np.asarray(b[k])
            assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), \
                "view %d: %s differs from the single calls'" % (v, k)
        if v % 3 == 0:
            tr, sizes = views[v]
            o = _oracle("%s%r view %d" % (gen, sorted(kw.items()), v * every), tr, tuple(sizes))
            meta = {k: np.concatenate([x[j] for x in outs[v]]) for j, k in enumerate(META_KEYS)}
            _check(o, engs[v], tr, ncs[v], meta, "view %d of %s" % (v * every, base.name))
    for e in engs + twins:
        e.close()


# ---------------------------------------------------------------- e. ingest by id, one sync per call
def test_ingest_one_sync_per_call():
    """A partition view's syncs through sw_ingest, each burst shuffled: the engine puts every burst in its own parents-
    first order, a topological order other than the view's.  The engine equals the oracle on the arrival order
    sw_ingest reports."""
    from swirld_b200 import engine
    from swirld_b200.traces import Trace
    name = "view_g5_m8_n12000_s3_x0"
    tr, sizes, _ = _fixture_view(name)
    N = tr.N
    ids = np.stack([np.frombuffer(hashlib.blake2b(tr.sig[i].tobytes(), digest_size=32).digest(), np.uint8)
                    for i in range(N)])
    zero = np.zeros((1, 32), np.uint8)
    pid = lambda a: np.where((a >= 0)[:, None], ids[np.maximum(a, 0)], zero)
    e = engine.Engine(tr.M, N)
    rng = np.random.default_rng(11)
    arrival = np.full(N, -1, np.int64)
    ncs, moved = [], 0
    for first, cnt in _sched(sizes):
        burst = rng.permutation(np.arange(first, first + cnt))
        out, m = e.ingest(ids[burst], pid(tr.p0[burst]), pid(tr.p1[burst]), tr.creator[burst], tr.t[burst],
                          tr.sig[burst])
        assert m == cnt and np.array_equal(np.sort(out), np.arange(first, first + cnt))
        arrival[burst] = out
        moved += int((out != burst).sum())
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        ncs.append(sorted(nc))
    assert moved > 0, "sw_ingest kept the view's own order everywhere"
    order = np.argsort(arrival)
    remap = lambda p: np.where(p >= 0, arrival[np.maximum(p, 0)], -1).astype(np.int32)
    tr2 = Trace(tr.M, remap(tr.p0[order]), remap(tr.p1[order]), tr.creator[order], tr.t[order], tr.sig[order],
                name + " ingested")
    o = _oracle(name + " ingested", tr2, tuple(sizes))
    _check(o, e, tr2, ncs, None, name + " ingested")
