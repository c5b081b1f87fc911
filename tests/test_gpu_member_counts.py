"""The engine at every member count its kernels branch on (tests/member_cases.py): every M from 1 to 64 under the four
implementations, every mask-word and NJ edge up to 1024 members, batched views at the edges, and the can_see scan's
multi-block and narrow-tile shapes above 256 members.  Everything the oracle computes is compared bit for bit: rounds,
witnesses, fame, consensus, the order with its consensus times and rounds received (find_order_out, call by call),
new_c per call, can_see, heights and idx."""
import numpy as np
import pytest

import member_cases as mc
import oracle as orc
import order_meta
from test_gpu_order_meta import KEYS as META_KEYS, _check_out, _same as _same_meta
from test_gpu_parity import impl  # noqa: F401  (the fixture: default, grid, cluster, wide)
from util import assert_same

pytestmark = pytest.mark.gpu

SMALL = 16        # calls up to this size take the one-launch streaming kernel
LARGE = 2048      # calls from this size take the cluster round kernel (SW_RC_MIN_N) at M <= 64


# ---------------------------------------------------------------- the oracle, once per trace and schedule
_ORACLE = {}


def _oracle(key, tr, sched, stake=None, C=6):
    """One oracle run over the calls, with order_meta riding along: results(), new_c per call, what find_order
    appended at each call (events, consensus times, rounds received), can_see, heights and idx.  Cached: the four
    implementations share it."""
    if key not in _ORACLE:
        o = orc.Oracle(tr.M, stake, C)
        o.append(tr)
        m = order_meta.OrderMeta(o)
        m.add_columns(tr.p0, tr.creator, tr.t)
        ncs, outs = [], []
        for first, cnt in sched:
            o.divide_rounds(first, cnt)
            nc = sorted(o.decide_fame())
            ncs.append(nc)
            outs.append(m.find_order(nc, first + cnt))
        r = o.results()
        h, idx = np.empty(tr.N, np.int32), np.empty(tr.N, np.int32)
        orc.lib().or_get_height(o._h, h)
        orc.lib().or_get_idx(o._h, idx)
        r.update(new_c_per_call=ncs, outs=outs, can_see=o.can_see(), heights=h, idx=idx)
        o.close()
        _ORACLE[key] = r
    return _ORACLE[key]


def _meta(out):
    return dict(zip(META_KEYS, out))


def _check(o, e, tr, ncs, outs, what):
    """The engine e (its calls' new_c and find_order_out outputs) against the oracle's run o."""
    from swirld_b200 import traces
    r = e.results()
    r["new_c_per_call"] = ncs
    assert_same(o, r, what=what)
    assert np.array_equal(o["witness"], r["witness"]), what + ": witness flags differ"
    assert len(outs) == len(o["outs"])
    for i, (a, b) in enumerate(zip(o["outs"], outs)):
        _same_meta(_meta(a), _meta(b), "%s call %d: find_order_out" % (what, i))
    assert np.array_equal(o["can_see"], e.can_see()), what + ": can_see differs"
    h = e.heights()
    assert np.array_equal(o["heights"], h), what + ": heights differ from the oracle's"
    assert np.array_equal(traces.heights(tr), h), what + ": heights differ from traces.heights"
    assert np.array_equal(o["idx"], e.idx()), what + ": idx differs"


def _run(tr, sched, stake=None, C=6, what="", cap=None):
    """One engine through the calls, each appending its own events, find_order_out at every call.  Returns the
    engine, new_c and the output per call, the cluster round kernel's launches per call and the launches of each
    append."""
    from swirld_b200 import engine
    e = engine.Engine(tr.M, cap or tr.N, stake, C)
    ncs, outs, rc, app = [], [], [], []
    for i, (first, cnt) in enumerate(sched):
        k0 = e.stats()["kernel_launches"]
        e.append_trace(tr, first, cnt)
        s = e.stats()
        app.append(s["kernel_launches"] - k0)
        e.divide_rounds(first, cnt)
        rc.append(e.stats()["rounds_cluster_launches"] - s["rounds_cluster_launches"])
        nc = e.decide_fame()
        before = e.n_transactions
        out = e.find_order_out(nc)
        _check_out(e, before, out, "%s call %d" % (what, i))
        ncs.append(sorted(nc))
        outs.append(out)
    return e, ncs, outs, rc, app


# ---------------------------------------------------------------- 1. every M from 2 to 64, four implementations
@pytest.mark.parametrize("name", list(mc.NARROW))
def test_narrow_member_count(name, impl):  # noqa: F811
    """Calls of <= 16, 17..2047 and >= 2048 events in turn.  "cluster" launches k_rounds_cluster for every call above
    16 events, "default" for exactly the calls of >= 2048; "grid" and "wide" never do."""
    case = mc.NARROW[name]
    tr = case.trace()
    sched = case.schedule(tr.N)
    e, ncs, outs, rc, _ = _run(tr, sched, case.stakes(), case.C, what=name)
    _check(_oracle(name, tr, sched, case.stakes(), case.C), e, tr, ncs, outs, "%s [%s]" % (name, impl))
    for (first, cnt), n in zip(sched, rc):
        want = {"default": cnt >= LARGE, "cluster": cnt > SMALL}.get(impl, False)
        assert (n > 0) == want, "%s [%s]: call [%d, +%d) launched k_rounds_cluster %d times" % (name, impl, first, cnt, n)
    e.close()


# ---------------------------------------------------------------- 2. one member
def test_one_member(impl):  # noqa: F811
    """M = 1: the root is a witness of round 0, no round is ever decided and nothing is ordered; a second root is a
    fork, and an event with parents has no other-parent to name.  sw_create takes 1 to 1024 members."""
    from swirld_b200 import engine, traces
    tr = traces.Trace(1, np.array([-1], np.int32), np.array([-1], np.int32), np.array([0], np.int32), np.zeros(1),
                      traces.make_sigs(1, 1), "one member")
    sched = [(0, 1)]
    e, ncs, outs, rc, _ = _run(tr, sched, what="M=1", cap=8)       # (room for the events it must refuse)
    assert ncs == [[]] and len(outs[0][0]) == 0 and rc == [0]
    assert e.rounds().tolist() == [0] and e.witness_flags().tolist() == [1] and e.witness_table().tolist() == [[0]]
    assert e.find_order([]) == 0 and e.n_transactions == 0
    _check(_oracle("M=1", tr, sched), e, tr, ncs, outs, "M=1 [%s]" % impl)
    sig, t = np.zeros((1, 64), np.uint8), np.zeros(1)
    with pytest.raises(engine.EngineError) as ei:
        e.append([-1], [-1], [0], t, sig)
    assert ei.value.code == -7                             # SW_E_FORK
    for p0, p1 in ((0, 0), (0, -1), (-1, 0)):
        with pytest.raises(engine.EngineError) as ei:
            e.append([p0], [p1], [0], t, sig)
        assert ei.value.code == -6, (p0, p1)               # SW_E_PARENT
    assert e.n_events == 1 and e.decide_fame() == []
    e.close()
    with pytest.raises(engine.EngineError) as ei:
        engine.Engine(0, 16)
    assert ei.value.code == -1                             # SW_E_ARG
    with pytest.raises(engine.EngineError) as ei:
        engine.Engine(1025, 16)
    assert ei.value.code == -8                             # SW_E_UNSUPPORTED
    engine.Engine(1024, 16).close()


# ---------------------------------------------------------------- 3. every mask-word and NJ edge, and the scan above 256
@pytest.mark.parametrize("name", list(mc.WIDE) + list(mc.SCAN))
def test_wide_member_count(name):
    """The wide kernels (any implementation: above 64 members they are the only ones).  The SCAN cases' long call is
    appended at once, so sw_append scans it: the 9 launches of the multi-block scan."""
    case = mc.ORACLE_CASES[name]
    tr = case.trace()
    sched = case.schedule(tr.N)
    e, ncs, outs, _, app = _run(tr, sched, case.stakes(), case.C, what=name)
    _check(_oracle(name, tr, sched, case.stakes(), case.C), e, tr, ncs, outs, name)
    if name in mc.SCAN:
        long = [i for i, (first, cnt) in enumerate(sched) if mc.cs_blocks(tr.M, first, cnt) > 2 and cnt >= 4096]
        assert long and all(app[i] == 9 for i in long), "%s: appends of the long calls made %s launches" % (
            name, [app[i] for i in long])
    e.close()


# ---------------------------------------------------------------- 4. batched views at the edges
def _view_sched(M, N, v):
    """View v's calls: at most 16 events above 64 members; at M <= 64 also chunk-path calls, rotated by view so that
    one batched divide holds streaming and chunk-path views."""
    sizes = (16, 1, 7, 16, 3) if M > 64 else (1, 16, 5, 700, 3, 2100, 9, 300)
    sizes = sizes[v % len(sizes):] + sizes[:v % len(sizes)]
    out, first, i = [], 0, 0
    while first < N:
        cnt = min(sizes[i % len(sizes)], N - first)
        out.append((first, cnt))
        first += cnt
        i += 1
    return out


@pytest.mark.parametrize("M,N", [(2, 4000), (31, 4000), (32, 4000), (33, 4000), (63, 4000), (64, 4000),
                                 (127, 3500), (255, 3000), (1023, 2500)])
def test_batched_views_at_the_edges(M, N):
    """Three views of different seeds turn by turn: one batch_append, one batch_divide_rounds, one batch_decide_fame
    and one batch_find_order_out over the live views.  Every view equals a twin driven by single calls byte for byte,
    and the oracle.  (Above 64 members every call is a streaming one, and the oracle's decide_fame per call of a
    few events keeps these views short.)"""
    from swirld_b200 import engine, traces
    trs = [traces.gossip(M, N - 7 * v, 300 + v) for v in range(3)]
    scheds = [_view_sched(M, tr.N, v) for v, tr in enumerate(trs)]
    engs = [engine.Engine(M, tr.N) for tr in trs]
    twins = [engine.Engine(M, tr.N) for tr in trs]
    ncs, outs = [[] for _ in trs], [[] for _ in trs]
    mixed = 0
    for t in range(max(len(s) for s in scheds)):
        live = [v for v in range(3) if t < len(scheds[v])]
        cols = []
        for v in live:
            first, cnt = scheds[v][t]
            s = slice(first, first + cnt)
            cols.append((trs[v].p0[s], trs[v].p1[s], trs[v].creator[s], trs[v].t[s], trs[v].sig[s]))
        engine.batch_append([engs[v] for v in live], cols)
        engine.batch_divide_rounds([engs[v] for v in live], [scheds[v][t][0] for v in live],
                                   [scheds[v][t][1] for v in live])
        n_small = sum(scheds[v][t][1] <= SMALL for v in live)
        mixed += 0 < n_small < len(live)
        nc = engine.batch_decide_fame([engs[v] for v in live])
        out = engine.batch_find_order_out([engs[v] for v in live], nc)
        for k, v in enumerate(live):
            ncs[v].append(sorted(nc[k]))
            outs[v].append(out[k])
            tw, (first, cnt) = twins[v], scheds[v][t]
            tw.append_trace(trs[v], first, cnt)
            tw.divide_rounds(first, cnt)
            tnc = tw.decide_fame()
            assert sorted(tnc) == ncs[v][-1], "M=%d view %d, turn %d: new_c differs from the single calls'" % (M, v, t)
            tout = tw.find_order_out(tnc)
            for x, y in zip(out[k], tout):
                assert x.tobytes() == y.tobytes(), "M=%d view %d, turn %d: find_order_out differs" % (M, v, t)
    if M <= 64:
        assert mixed > 0, "no batched divide held both streaming and chunk-path views"
    for v, tr in enumerate(trs):
        for k, (x, y) in enumerate(zip((engs[v].results(), engs[v].can_see(), engs[v].heights(), engs[v].idx()),
                                       (twins[v].results(), twins[v].can_see(), twins[v].heights(), twins[v].idx()))):
            for a, b in (zip(x.values(), y.values()) if isinstance(x, dict) else [(x, y)]):
                assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), \
                    "M=%d view %d: differs from the single calls' (item %d)" % (M, v, k)
        what = "M=%d batched view %d" % (M, v)
        _check(_oracle(what, tr, scheds[v]), engs[v], tr, ncs[v], outs[v], what)
    for e in engs + twins:
        e.close()


# ---------------------------------------------------------------- 5. narrow scan tiles
def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("ct,stale", [(16, False), (16, True), (8, False)])
def test_scan_tile_width(ct, stale):
    """The can_see scan with tiles ct columns wide: the first SCAN_CT case for which the host's choice (restated in
    member_cases.cs_tile_width) picks that width on this device's SM count, appended in one call, which sw_append scans
    in the 9 launches of the multi-block scan.  can_see and heights are compared with the exact host recurrences
    (traces.can_see_rows, traces.heights); rounds are not checked here (the oracle would take hours at these sizes;
    test_wide_member_count checks them on the multi-block scans at 300 members)."""
    from swirld_b200 import engine, traces
    n_sm = _n_sm()
    name = mc.pick_ct(n_sm, ct, stale)
    if name is None:
        pytest.skip("no candidate scans with CT = %d %s stale parents on %d SMs" % (ct, "with" if stale else "without",
                                                                                    n_sm))
    case = mc.SCAN_CT[name]
    tr = case.trace()
    CT, nb = mc.scan_shape(case, tr, n_sm)
    assert CT == ct and nb > 1, (name, CT, nb)
    e = engine.Engine(tr.M, tr.N)
    k0 = e.stats()["kernel_launches"]
    e.append_trace(tr)
    assert e.stats()["kernel_launches"] - k0 == 9, name + ": not the multi-block scan"
    e.divide_rounds(0, tr.N)
    got = e.can_see()
    want = traces.can_see_rows(tr)
    if not np.array_equal(want, got):
        bad = np.argwhere(want != got)
        raise AssertionError("%s (CT %d, %d blocks, %d SMs): can_see differs in %d entries, first %s" % (
            name, CT, nb, n_sm, len(bad), bad[:5].tolist()))
    del got, want
    assert np.array_equal(traces.heights(tr), e.heights()), name + ": heights differ"
    print("%s: CT %d, %d blocks, %d SMs" % (name, CT, nb, n_sm))
    e.close()
