"""decide_fame and find_order for several node-views per launch (sw_batch_decide_fame / sw_batch_find_order): every
view must end exactly where single calls would have left it.  Each view is checked against the oracle on its own trace
and schedule (per-call new_c and can_see included) and against a twin engine that made the same calls one view at a
time (every result array byte for byte).  The batches mix views in different states at one member count: more than
1024 new rounds, a backlog, one event per call, no new round in a call, coin rounds, partitions, zero stakes and a
single seer (swirld.py:305 IndexError) beside healthy views.  The named traces are those of tests/fame_cases.py and
tests/shape_cases.py; each case asserts the oracle counters or sizes it is there for."""
import ctypes as C
import functools

import numpy as np
import pytest

import fame_cases as fc
import oracle as orc
import shape_cases as sc
from util import assert_same

pytestmark = pytest.mark.gpu

ARRAYS = ("round", "witness", "witness_table", "famous", "consensus", "transactions", "idx")


def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gossip(M, N, seed, K, stake=None, C=6):
    return fc.Case("gossip", dict(M=M, N=N, seed=seed), K, stake, C)


_ORACLE = {}


def _oracle(case):
    """The case's oracle run, once per case: results(), new_c per call and the oracle (and, from fame_cases.run_oracle,
    coverage() and the call that raised IndexError, -1: none)."""
    if repr(case) not in _ORACLE:
        _ORACLE[repr(case)] = fc.run_oracle(case)
    return _ORACLE[repr(case)]


@functools.lru_cache(maxsize=None)
def _sizes(name):
    """A shape case's oracle run with its sizes (shape_cases.sizes), which also serves as its _oracle."""
    case = sc.CASES[name]
    s = sc.sizes(case)
    assert not sc.missing(case, s), "%s no longer exceeds %s" % (name, sc.missing(case, s))
    _ORACLE[repr(case)] = s
    return s


def _covers(name, case):
    o = _oracle(case)
    assert not fc.missing(case, o["coverage"]), "%s no longer reaches %s" % (name, fc.missing(case, o["coverage"]))


def _arrays(e):
    r = e.results()
    r["idx"] = e.idx()
    return r


def _run_batch(cases, batch_divide=True, raise_at=None):
    """Every view's calls side by side: its append and divide_rounds (one sw_batch_divide_rounds for all views, or one
    call per view), then one batch_decide_fame and one batch_find_order over the views that still have calls.  A view
    whose find_order fails leaves the batch.  raise_at[v] = the call at which view v is expected to fail: its results()
    between its decide_fame and find_order of that call are kept.  Returns the engines, new_c per call of every view,
    {view: (call, exception)} and those kept results."""
    from swirld_b200 import engine
    B = len(cases)
    trs = [c.trace() for c in cases]
    scheds = [c.schedule(tr.N) for c, tr in zip(cases, trs)]
    engs = [engine.Engine(tr.M, tr.N, c.stakes(), c.C) for c, tr in zip(cases, trs)]
    ncs, failed, before = [[] for _ in range(B)], {}, {}
    for i in range(max(len(s) for s in scheds)):
        live = [v for v in range(B) if i < len(scheds[v]) and v not in failed]
        if not live:
            break
        for v in live:
            engs[v].append_trace(trs[v], *scheds[v][i])
        if batch_divide:
            engine.batch_divide_rounds([engs[v] for v in live], [scheds[v][i][0] for v in live],
                                       [scheds[v][i][1] for v in live])
        else:
            for v in live:
                engs[v].divide_rounds(*scheds[v][i])
        got = engine.batch_decide_fame([engs[v] for v in live])
        for v, nc in zip(live, got):
            ncs[v].append(sorted(nc))
            if raise_at and raise_at.get(v) == i:
                before[v] = engs[v].results()
        try:
            engine.batch_find_order([engs[v] for v in live], got)
        except ExceptionGroup as g:
            for ex in g.exceptions:
                failed[live[ex.view]] = (i, ex)
            assert [g.results[k] is None for k in range(len(live))] == [live[k] in failed for k in range(len(live))]
    return engs, ncs, failed, before


def _run_single(case, stop_at=-1):
    """The twin: the same calls through the single-view ABI (stop_at: the call whose find_order raises IndexError)."""
    from swirld_b200 import engine
    tr = case.trace()
    e = engine.Engine(tr.M, tr.N, case.stakes(), case.C)
    for i, (first, cnt) in enumerate(case.schedule(tr.N)):
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        if i == stop_at:
            with pytest.raises(IndexError):
                e.find_order(nc)
            break
        e.find_order(nc)
    return e


def _same_arrays(a, b, what):
    for k in ARRAYS:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), "%s: %s differs from single calls" % (what, k)


def _check(cases, engs, ncs, oracle_views=None, twins=True, names=None):
    """Views against the oracle (oracle_views: which; all by default) and every view against its single-call twin."""
    for v, case in enumerate(cases):
        what = names[v] if names else "view %d of %d" % (v, len(cases))
        if oracle_views is None or v in oracle_views:
            o = _oracle(case)
            r = engs[v].results()
            r["new_c_per_call"] = ncs[v]
            assert_same(o, r, what=what)
            assert np.array_equal(o["oracle"].can_see(), engs[v].can_see()), what + ": can_see differs"
        if twins:
            _same_arrays(_arrays(engs[v]), _arrays(_run_single(case)), what)


# ---------------------------------------------------------------- 1 + 2: parity with the oracle and with single calls
NARROW = [(4, 2000, 50, 5), (16, 12000, 2000, 6), (33, 9000, 1500, 8), (64, 24000, 8192, 3)]
WIDE = [(97, 12000, 3000, 3), (129, 16000, 4000, 3), (300, 30000, 8192, 2)]


def _ragged(M, N, K, B):
    return [_gossip(M, N - 7 * v, 100 + v, K) for v in range(B)]


@pytest.mark.parametrize("M,N,K,B", NARROW)
@pytest.mark.parametrize("family", ["default", "wide"])
def test_batch_matches_oracle_and_single_calls(M, N, K, B, family, monkeypatch):
    """Ragged views of one member count: sw_batch_divide_rounds, then the batched fame and order.  "wide" selects the
    any-M kernels (SW_FORCE_WIDE=1), whose views divide one by one (sw_batch_divide_rounds is the M <= 64 kernels')."""
    monkeypatch.setenv("SW_FORCE_WIDE", "1" if family == "wide" else "0")
    cases = _ragged(M, N, K, B)
    engs, ncs, failed, _ = _run_batch(cases, batch_divide=family == "default")
    assert not failed
    _check(cases, engs, ncs, oracle_views={0, B // 2, B - 1})


@pytest.mark.parametrize("M,N,K,B", WIDE)
def test_batch_wide_matches_oracle_and_single_calls(M, N, K, B):
    """Above 64 members (NJ = 4, 8 and 16 words per member mask): each view divides on its own."""
    cases = _ragged(M, N, K, B)
    engs, ncs, failed, _ = _run_batch(cases, batch_divide=False)
    assert not failed
    _check(cases, engs, ncs, oracle_views={0, B - 1})


# ---------------------------------------------------------------- 3: views in different states in one batch
def test_mixed_states_m4():
    """More than 1024 new rounds in one call (a second copy for that view), a backlog that arrives late, one event per
    call with C = 2, and integer stakes with a zero at C = 3, whose calls often bring no new round while others do."""
    one, backlog = sc.CASES["big_m4_one_call"], sc.CASES["big_m4_backlog"]
    k1 = _gossip(4, 600, 11, 1, None, 2)
    zero = _gossip(4, 3000, 5, 37, [2, 1, 1, 0], 3)
    assert len(_sizes("big_m4_one_call")["new_c_per_call"][0]) > sc.SPEC
    assert len(_sizes("big_m4_backlog")["new_c_per_call"][-1]) > sc.SPEC
    assert _oracle(k1)["coverage"]["coin_votes"] > 0 and _oracle(zero)["coverage"]["coin_votes"] > 0
    cases = [one, backlog, k1, zero]
    engs, ncs, failed, _ = _run_batch(cases, batch_divide=False)         # (stakes differ: views divide one by one)
    assert not failed
    # some call asks a view for no new round while another view of the batch orders some
    assert any(not ncs[3][i] and any(len(ncs[v]) > i and ncs[v][i] for v in range(3)) for i in range(len(ncs[3])))
    _check(cases, engs, ncs, names=["big_m4_one_call", "big_m4_backlog", "k1_c2", "zero_c3"])


def test_mixed_states_m129():
    """Coin rounds at C = 2, tied times at C = 3 and both partitions of 129 members in one batch (NJ = 8)."""
    names = ["coin_nj8_m129_gossip_c2", "tied_m129_gossip_c3", "part_m129_major", "part_m129_even"]
    for n in names[:2]:
        _covers(n, fc.CASES[n])
    for n in names[2:]:
        _sizes(n)
    cases = [fc.CASES[n] for n in names[:2]] + [sc.CASES[n] for n in names[2:]]
    engs, ncs, failed, _ = _run_batch(cases, batch_divide=False)
    assert not failed
    _check(cases, engs, ncs, names=names)


def test_mixed_states_m64():
    """Coin rounds on two-word masks beside a majority partition (one member count, unit stakes: one
    sw_batch_divide_rounds per call)."""
    _covers("coin_m64_adv_c3", fc.CASES["coin_m64_adv_c3"])
    _sizes("part_m64_major")
    cases = [fc.CASES["coin_m64_adv_c3"], sc.CASES["part_m64_major"]]
    engs, ncs, failed, _ = _run_batch(cases, batch_divide=True)
    assert not failed
    _check(cases, engs, ncs, names=["coin_m64_adv_c3", "part_m64_major"])


# ---------------------------------------------------------------- 4: a single seer in a batch
@pytest.mark.parametrize("seer,healthy", [
    ("seer_m4", [(4, 900, 21, 20), (4, 1200, 22, 20), (4, 700, 23, 7)]),
    ("seer_m80", [(80, 6000, 31, 500), (80, 5000, 32, 500), (80, 6000, 33, 700)]),
])
def test_single_seer_in_a_batch(seer, healthy):
    """The seer view gets IndexError at the call the oracle raises, with the oracle's state at that call and then
    whatever the single call leaves; the healthy views run their whole schedules, equal to the oracle."""
    case = fc.SEER_CASES[seer]
    o = _oracle(case)
    assert o["coverage"]["single_seer"] == 1 and o["raised_at"] >= 0
    cases = [_gossip(*h) for h in healthy[:2]] + [case] + [_gossip(*h) for h in healthy[2:]]
    engs, ncs, failed, before = _run_batch(cases, batch_divide=False, raise_at={2: o["raised_at"]})
    assert list(failed) == [2]
    call, ex = failed[2]
    assert call == o["raised_at"] and isinstance(ex, IndexError) and ex.view == 2
    assert ncs[2] == o["new_c_per_call"]
    # the oracle's state at the raise, its events appended call by call (as test_gpu_fame_order.py compares it)
    tr, sched = case.trace(), case.schedule(case.trace().N)
    oc = orc.Oracle(tr.M, case.stakes(), case.C)
    for i, (first, cnt) in enumerate(sched[:call + 1]):
        oc.append(tr.slice(first, first + cnt))
        oc.divide_rounds(first, cnt)
        nc = oc.decide_fame()
        if i < call:
            oc.find_order(nc)
        else:
            with pytest.raises(IndexError):
                oc.find_order(nc)
    assert_same(oc.results(), before[2], what=seer + " before the raise")
    # afterwards the device error stays in the view's scalars, as after the single call: every synchronising getter
    # raises it; the arrays the plain getters read must equal the single-call twin's
    twin = _run_single(case, stop_at=call)
    nr = before[2]["witness_table"].shape[0]
    for e in (engs[2], twin):
        with pytest.raises(IndexError):
            e.sync()
    after = [dict(round=e.rounds(), witness=e.witness_flags(), famous=e.famous(), transactions=e.transactions(),
                  idx=e.idx(), witness_table=e.witness_table(0, nr), consensus=np.zeros(0)) for e in (engs[2], twin)]
    _same_arrays(after[0], after[1], seer + " after the raise")
    _check([c for v, c in enumerate(cases) if v != 2], [e for v, e in enumerate(engs) if v != 2],
           [n for v, n in enumerate(ncs) if v != 2], twins=False)


# ---------------------------------------------------------------- 5: more views than SMs
def test_more_views_than_sms():
    """n_sm + 3 views of 8 members in one batch: one grid row per view, every view against the oracle."""
    B = _n_sm() + 3
    cases = [_gossip(8, 6000 - 7 * v, 100 + v, 1000) for v in range(B)]
    engs, ncs, failed, _ = _run_batch(cases)
    assert not failed
    _check(cases, engs, ncs, twins=False)


# ---------------------------------------------------------------- 6: refusals
def _raw_order(engs, new_c, offsets, B=None):
    from swirld_b200 import engine
    lib = engs[0]._lib
    B = len(engs) if B is None else B
    arr = (C.c_void_p * max(1, len(engs)))(*[e._h for e in engs])
    flat = np.ascontiguousarray(new_c, np.int32)
    offs = np.ascontiguousarray(offsets, np.int32)
    cnt = np.full(max(1, len(engs)), 12345, np.int32)
    rc = lib.sw_batch_find_order(C.cast(arr, C.c_void_p), B, engine._ptr(flat), engine._ptr(offs), engine._ptr(cnt))
    return rc, cnt


def test_refusals_change_nothing(monkeypatch):
    """Every argument error refuses the whole call before anything runs: mixed member counts, a repeated engine, mixed
    kernel families, a view with nothing divided, an unknown round, offsets that go down, no view at all.  count_out
    stays unwritten, and every view, continued with single calls, still equals the oracle."""
    from swirld_b200 import engine
    from swirld_b200.engine import EngineError
    cases = [_gossip(8, 3000, 41, 500), _gossip(8, 2500, 42, 500), _gossip(8, 3000, 43, 700)]
    trs = [c.trace() for c in cases]
    odd = _gossip(9, 2000, 44, 500)
    e9 = engine.Engine(9, 2000)
    engs = [engine.Engine(8, tr.N) for tr in trs]
    monkeypatch.setenv("SW_FORCE_WIDE", "1")
    ew = engine.Engine(8, trs[0].N)
    monkeypatch.delenv("SW_FORCE_WIDE")
    undiv = engine.Engine(8, trs[0].N)
    undiv.append_trace(trs[0])
    scheds = [c.schedule(tr.N) for c, tr in zip(cases, trs)]
    for e, tr, s in zip(engs + [ew], trs + [trs[0]], scheds + [scheds[0]]):
        e.append_trace(tr)
        e.divide_rounds(*s[0])
    e9.append_trace(odd.trace())
    e9.divide_rounds(*odd.schedule(2000)[0])

    def code(exc_info):
        return exc_info.value.code

    for views, want in [(engs + [e9], -8), (engs + [engs[1]], -1), (engs + [ew], -8), (engs + [undiv], -1)]:
        with pytest.raises(EngineError) as ei:
            engine.batch_decide_fame(views)
        assert code(ei) == want
    with pytest.raises(EngineError) as ei:
        engine.batch_find_order(engs + [e9], [[], [], [], []])
    assert code(ei) == -8
    with pytest.raises(KeyError):
        engine.batch_find_order(engs, [[], [10 ** 7], []])
    rc, cnt = _raw_order(engs, [0, 1], [0, 2, 1, 2])
    assert rc == -1 and (cnt == 12345).all()
    rc, cnt = _raw_order(engs, [0], [0, 0, 0, 0], B=0)
    assert rc == -1 and (cnt == 12345).all()
    # nothing ran: each view continues with single calls from where it stood
    for v, (e, case, tr, s) in enumerate(zip(engs + [ew, undiv], cases + [cases[0]] * 2, trs + [trs[0]] * 2,
                                           scheds + [scheds[0]] * 2)):
        ncs = []
        for i, (first, cnt_) in enumerate(s):
            if i > 0 or e is undiv:
                e.divide_rounds(first, cnt_)
            nc = e.decide_fame()
            e.find_order(nc)
            ncs.append(sorted(nc))
        r = e.results()
        r["new_c_per_call"] = ncs
        assert_same(_oracle(case), r, what="view %d after the refusals" % v)


# ---------------------------------------------------------------- 7: launches do not grow with the batch
def test_launch_count_does_not_grow_with_views():
    """One batch_decide_fame + batch_find_order at M = 33 costs the same kernel launches, summed over all engines, for
    1 view and for 40."""
    from swirld_b200 import engine
    per = {}
    for B in (1, 40):
        cases = [_gossip(33, 3000 - 7 * v, 100 + v, 3000) for v in range(B)]
        engs = []
        for c in cases:
            tr = c.trace()
            e = engine.Engine(33, tr.N)
            e.append_trace(tr)
            e.divide_rounds(0, tr.N)
            engs.append(e)
        before = sum(e.stats()["kernel_launches"] for e in engs)
        ncs = engine.batch_decide_fame(engs)
        assert ncs[0], "view 0 brings no new round: find_order would launch nothing"
        engine.batch_find_order(engs, ncs)
        per[B] = sum(e.stats()["kernel_launches"] for e in engs) - before
    assert per[1] == per[40], per


# ---------------------------------------------------------------- 8: checkpoint after batched calls
@pytest.mark.parametrize("M,N,K", [(16, 8000, 1000), (97, 8000, 1500)])
def test_checkpoint_after_batched_calls(M, N, K, tmp_path):
    """sw_save a view after half its calls went through the batched calls, sw_load it, and the rest with single calls:
    equal to the oracle (the batch path must keep the host mirrors sw_save writes: n_tx, the scalars)."""
    from swirld_b200 import engine
    cases = _ragged(M, N, K, 2)
    half = len(cases[1].schedule(cases[1].trace().N)) // 2
    short = [fc.Case(c.gen, c.kw, K, c.stake, c.C, slice_to=half * K) for c in cases]
    engs, ncs, failed, _ = _run_batch(short, batch_divide=M <= 64)
    assert not failed
    path = str(tmp_path / "view1.swb")
    engs[1].save(path)
    engs[1].close()
    e = engine.Engine.load(path, capacity=N)
    tr = cases[1].trace()
    for first, cnt in cases[1].schedule(tr.N)[half:]:
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        ncs[1].append(sorted(nc))
    r = e.results()
    r["new_c_per_call"] = ncs[1]
    o = _oracle(cases[1])
    assert_same(o, r, what="view 1 resumed")
    assert np.array_equal(o["oracle"].can_see(), e.can_see())
