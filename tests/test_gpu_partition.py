"""The engine through network partitions and on calls larger than one launch: traces that fill the fixed-size windows
of the round kernels (the 256-event rings, the cluster kernel's 128-row window and 32-round Wf mirror) and run the
second trips of the fame and order kernels' grid- and block-stride loops.  The cases and the sizes each must exceed
are in tests/shape_cases.py; every test asserts those sizes from its own oracle run, then compares the engine with
the oracle bit for bit (per-call new_c included) and can_see."""
import functools

import numpy as np
import pytest

import shape_cases as sc
from test_gpu_parity import _check_round_kernel, impl  # noqa: F401  (impl: the four M <= 64 implementations)
from util import assert_same

pytestmark = pytest.mark.gpu

NARROW = [n for n, c in sc.CASES.items() if n.startswith("part") and c.M <= 64]
WIDE = [n for n, c in sc.CASES.items() if n.startswith("part") and c.M > 64]


def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """The case's oracle run, once per case for all four implementations."""
    case = sc.CASES[name]
    s = sc.sizes(case)
    assert not sc.missing(case, s), "%s no longer exceeds %s" % (name, sc.missing(case, s))
    return s


def _engine(case, tr):
    from swirld_b200 import engine
    e = engine.Engine(tr.M, tr.N, case.stakes(), case.C)
    ncs = []
    for first, cnt in case.schedule(tr.N):
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        ncs.append(sorted(nc))
    r = e.results()
    r.update(new_c_per_call=ncs, can_see=e.can_see(), stats=e.stats(), dbg=e.debug_counters())
    return r


def _parity(name):
    case = sc.CASES[name]
    tr = case.trace()
    o = _oracle(name)
    r = _engine(case, tr)
    assert_same(o, r, what=name)
    assert np.array_equal(o["oracle"].can_see(), r["can_see"]), name + ": can_see differs"
    return case, tr, o, r


def _hands_over(case, impl):
    """Chains more than RB_WR rounds apart at a call start of >= 2048 events: the cluster round kernel (under "default"
    and "cluster") must hand the chunk to the grid-wide kernel."""
    return (("behind", sc.RB_WR) in case.needs and impl in ("default", "cluster")
            and isinstance(case.K, int) and case.K >= 2048)


# ---------------------------------------------------------------- partitions, M <= 64
@pytest.mark.parametrize("name", NARROW)
def test_partition_matches_oracle(name, impl):
    """Stalled chains hundreds of events deep in one round, calls that end inside the stall, minority chains dozens
    of rounds behind, and a heal round that orders thousands of events, on all four implementations."""
    case, tr, o, r = _parity(name)
    if isinstance(case.K, int):
        _check_round_kernel(impl, tr, case.K, r)
    if _hands_over(case, impl):
        assert r["dbg"][15] > 0, "%s: the cluster round kernel never handed over (behind = %d)" % (name, o["behind"])


# ---------------------------------------------------------------- partitions above 64 members (swirld_wide.cuh)
@pytest.mark.parametrize("name", WIDE)
def test_partition_wide(name):
    """NJ = 4 and 8, even and majority splits: runs longer than RW_RING."""
    _parity(name)


# ---------------------------------------------------------------- the bench's resident pattern through a partition
def test_partition_resident_rewind():
    """Every event appended before the first divide_rounds, so one can_see scan covers the whole partition (whose
    rows mostly fail the finality check and go to the slow-row kernels); then rewind and the same calls again."""
    from swirld_b200 import engine
    name = "part_m64_even"
    case = sc.CASES[name]
    tr = case.trace()
    o = _oracle(name)
    e = engine.Engine(tr.M, tr.N)
    e.append_trace(tr)
    for rep in range(2):
        if rep:
            e.rewind()
        ncs = []
        for first, cnt in case.schedule(tr.N):
            e.divide_rounds(first, cnt)
            nc = e.decide_fame()
            e.find_order(nc)
            ncs.append(sorted(nc))
        r = e.results()
        r["new_c_per_call"] = ncs
        assert_same(o, r, what="%s resident, pass %d" % (name, rep))
        assert np.array_equal(o["oracle"].can_see(), e.can_see()), "can_see differs (pass %d)" % rep
        assert np.array_equal(o["witness"], r["witness"])


# ---------------------------------------------------------------- checkpoint in the middle of a stall
@pytest.mark.parametrize("name", ["part_m8_even", "part_m40_even"])
def test_partition_checkpoint_mid_stall(name, impl, tmp_path):
    """sw_save while the chains sit more than RB_RING events into one round, sw_load, and the rest of the calls: the
    ring of recent events and the members' totals must round-trip, and sw_load must rebuild the count snapshots the
    chunk preparation reads."""
    from swirld_b200 import engine
    case = sc.CASES[name]
    tr = case.trace()
    o = _oracle(name)
    sched = case.schedule(tr.N)
    half = len(sched) // 2
    assert o["ring_gap_per_call"][half] > sc.RB_RING, "the save is not inside the stall"
    e = engine.Engine(tr.M, tr.N, case.stakes(), case.C)
    ncs = []
    for first, cnt in sched[:half]:
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        ncs.append(sorted(nc))
    path = str(tmp_path / "ckpt.swb")
    e.save(path)
    e.close()
    e2 = engine.Engine.load(path, capacity=tr.N + 1000)
    for first, cnt in sched[half:]:
        e2.append_trace(tr, first, cnt)
        e2.divide_rounds(first, cnt)
        nc = e2.decide_fame()
        e2.find_order(nc)
        ncs.append(sorted(nc))
    r = e2.results()
    r["new_c_per_call"] = ncs
    assert_same(o, r, what=name + " resumed mid-stall")
    assert np.array_equal(o["oracle"].can_see(), e2.can_see())


# ---------------------------------------------------------------- calls larger than one launch
def _open_beyond_grid(o, calls=None):
    """More open rounds in one decide_fame call than k_fame_rounds / k_w_fame_rounds have CTAs (2 * n_sm + 1 at
    most): the grid-stride round loop takes a second trip."""
    opens = o["open_per_call"] if calls is None else [o["open_per_call"][i] for i in calls]
    assert max(opens) > 2 * _n_sm() + 1, "open rounds per call %s, n_sm %d" % (max(opens), _n_sm())


@pytest.mark.parametrize("name", ["big_m4_one_call", "big_m33_one_call", "big_m33_one_call_stake"])
def test_one_call_larger_than_one_launch(name, impl):
    """One call over the whole trace: more than 1024 new consensus rounds (the speculative copy is not enough), more
    open rounds than CTAs, fame_collect and k_fame_finish over more rounds than threads."""
    o = _oracle(name)
    _open_beyond_grid(o)
    _parity(name)


def test_one_call_wide_more_open_rounds_than_ctas():
    """M = 65 (NJ = 4), one call: more open rounds than k_w_fame_rounds has CTAs."""
    o = _oracle("big_m65_one_call")
    _open_beyond_grid(o)
    _parity("big_m65_one_call")


def test_backlog_arrives_late(impl):
    """Calls of 1000 events, then the other half of the trace in one call: max_c is far from zero when the fame kernels
    meet more open rounds than CTAs, so the grid-stride loop and fame_collect start away from round 0."""
    name = "big_m4_backlog"
    o = _oracle(name)
    assert o["max_c_per_call"][-1] > 0
    _open_beyond_grid(o, [-1])
    assert len(o["new_c_per_call"][-1]) > sc.SPEC
    _parity(name)


# ---------------------------------------------------------------- more node-views than SMs
@pytest.mark.parametrize("N,K", [(6000, 1000), (20000, 4096)])
def test_batched_views_more_than_sms(N, K):
    """n_sm + 3 views of 8 members: sw_batch_divide_rounds runs them in two groups (one view per SM each).  Chunks of
    1000 events take the grid-wide views kernel at one CTA per view; chunks of 4096 take one k_rounds_cluster_views
    launch of n_sm clusters first.  View 0 is a majority partition, whose chunks the views kernel hands over.  Every
    view is compared with the oracle."""
    import oracle as orc
    from swirld_b200 import engine, traces
    from swirld_b200.traces import chunks
    B = _n_sm() + 3
    part = sc.Case("partition", dict(M=8, N=N, seed=1, split=6, start=N // 6, end=2 * N // 3), K)
    po = sc.sizes(part)
    assert K < 2048 or po["behind"] > sc.RB_WR
    trs = [part.trace()] + [traces.gossip(8, N - 7 * v, 100 + v) for v in range(1, B)]
    engs = [engine.Engine(8, tr.N) for tr in trs]
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
    for v in range(B):
        o = po if v == 0 else orc.run_oracle(trs[v], K)
        r = engs[v].results()
        r["new_c_per_call"] = ncs[v]
        assert_same(o, r, what="view %d of %d" % (v, B))
        assert np.array_equal(o["oracle"].can_see(), engs[v].can_see()), "view %d of %d: can_see differs" % (v, B)
    if K >= 2048:
        assert engs[0].stats()["rounds_cluster_launches"] > 0
        assert engs[0].debug_counters()[15] > 0, "the views kernel never handed the partition view over"
