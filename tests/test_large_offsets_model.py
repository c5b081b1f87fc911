"""The restatements and comparisons of tests/large_offsets.py against the oracle, without a GPU.

tests/test_gpu_large_offsets.py checks the engine at M = 1024 past 2^31 table elements with these restatements alone,
so here each must equal the oracle event for event (can_see rows, rounds, witness flags and the witness table, consensus
times, the sync summary and reply), on G1 at M = 97 and 1024, on an adversarial trace with stale other-parents and on a
partition; and each check must fail on a copy of the oracle's output with one element changed."""
import numpy as np
import pytest

import large_offsets as lo
import oracle as orc
import sync_model as sm
from order_meta import run_oracle_meta
from swirld_b200 import traces

CASES = {
    "g1-97": lambda: (traces.gossip(97, 6000, seed=3), 700),
    "g1-1024": lambda: (traces.gossip(1024, 20000, seed=4), 8192),
    "g2-stale": lambda: (traces.adversarial(16, 6000, seed=5, p_cross=0.05, p_stale=0.5), 250),
    "partition": lambda: (traces.partition(40, 8000, seed=6, start=1500, end=5000), 900),
}


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    tr, K = CASES[request.param]()
    o = orc.run_oracle(tr, K)
    res = {k: o[k] for k in ("round", "witness", "witness_table", "famous")}
    res["rows"] = o["oracle"].can_see()
    res["height"] = traces.heights(tr)
    o["oracle"].close()
    return request.param, tr, K, res


def _source(rows):
    return lambda first, n: rows[first:first + n]


def test_can_see_recurrence_equals_oracle(case):
    _, tr, _, r = case
    lo.check_can_see(_source(r["rows"]), tr.p0, tr.p1, tr.creator, r["height"], 0, tr.N, tr.M, chunk=1000)


def test_rounds_and_witnesses_equal_oracle(case):
    name, tr, _, r = case
    rnd = r["round"]
    assert rnd.max() >= (1 if tr.M == 1024 else 3)
    first = tr.N - 6000 if tr.M == 1024 else 0           # (the O(M^2) restatement, where 1024 members reach round 1)
    exp = lo.expected_rounds(_source(r["rows"]), rnd, np.ones(tr.M, np.int64), tr.p0, tr.p1, r["height"], first,
                             tr.N - first, tr.M)
    lo.assert_equal("round", rnd[first:], exp, offset=first)
    lo.assert_equal("witness", r["witness"], lo.expected_witness(rnd, tr.p0, 0, tr.N))
    lo.check_witness_table(r["witness_table"], r["witness"], rnd, tr.creator, tr.N // 2, [(tr.N // 2, tr.N)])


def test_rounds_with_stakes_equal_oracle():
    """Unequal stakes: hits are stake sums, while the count of members past min_s is compared with min_s itself."""
    tr = traces.gossip(9, 3000, seed=41)
    stake = [2, 1, 1, 1, 1, 1, 1, 1, 5]
    o = orc.run_oracle(tr, 25, stake)
    rows = o["oracle"].can_see()
    exp = lo.expected_rounds(_source(rows), o["round"], stake, tr.p0, tr.p1, traces.heights(tr), 0, tr.N, tr.M)
    lo.assert_equal("round", o["round"], exp)


def test_consensus_times_equal_order_meta():
    """The consensus timestamps of the events ordered from some index on, restated from the rows of those events and
    later ones only, equal the oracle's (tests/order_meta.py, pinned to the reference by its fixtures)."""
    tr = traces.gossip(16, 8000, seed=7)
    meta = run_oracle_meta(tr, 500, extra=True)
    res = meta["results"]
    o = orc.run_oracle(tr, 500)
    rows = o["oracle"].can_see()
    X = meta["transactions"].astype(np.int64)
    sel = np.flatnonzero(X >= 5000)
    assert sel.size > 500
    read = []

    def get(first, n):
        read.append((first, n))
        return rows[first:first + n]
    got = lo.consensus_times(get, tr.N, tr.p0, tr.creator, tr.t, res["witness_table"], res["famous"], X[sel],
                             meta["round_received"][sel])
    lo.assert_equal("consensus time", meta["consensus_time"][sel], got)
    assert read[0] == (int(X[sel].min()), tr.N - int(X[sel].min())) and min(f for f, _ in read) >= 5000 - 2 * lo.GAP
    ts = meta["consensus_time"][sel].copy()
    ts[-7] += 1
    assert "first at (%d,)" % (sel.size - 7) in lo.first_mismatch("consensus time", ts, got)


def test_sync_expected_equals_bfs():
    base = traces.gossip(16, 3000, seed=8)
    tr, _ = traces.node_view(base, 3)
    v = sm.View(tr)
    head, old = tr.N - 1, tr.N - 500
    S, S_old, reply = lo.sync_expected({head: v.row[head], old: v.row[old]}, v.height, tr.creator, head, old)
    lo.assert_equal("summary", sm.summary(v, head), S)
    lo.assert_equal("reply", sm.bfs_reply(v, head, sm.summary(v, old)), reply)
    assert reply.size > 100


# ---------------------------------------------------------------- each check fails on one changed element
def _mutated(a, at, value):
    b = a.copy()
    b[at] = value
    return b


def test_can_see_check_catches_one_entry(case):
    _, tr, _, r = case
    rows = r["rows"]
    h = tr.N - 777
    c = (int(tr.creator[h]) + 1) % tr.M
    bad = _mutated(rows, (h, c), rows[h, c] - 1)
    with pytest.raises(AssertionError, match=r"can_see: .* first at \(%d, %d\)" % (h, c)):
        lo.check_can_see(_source(bad), tr.p0, tr.p1, tr.creator, r["height"], h - 100, 200, tr.M)


def test_round_check_catches_one_round(case):
    _, tr, _, r = case
    h = tr.N - 500
    bad = _mutated(r["round"], h, r["round"][h] + 1)
    exp = lo.expected_rounds(_source(r["rows"]), bad, np.ones(tr.M, np.int64), tr.p0, tr.p1, r["height"], h - 50, 100, tr.M)
    assert lo.first_mismatch("round", bad[h - 50:h + 50], exp, h - 50).startswith("round: ")
    assert "first at (%d,)" % h in lo.first_mismatch("round", bad[h - 50:h + 50], exp, h - 50)


def test_witness_checks_catch_one_flag(case):
    _, tr, _, r = case
    wit, rnd = r["witness"], r["round"]
    h = int(np.flatnonzero(wit[tr.N // 2:])[0]) + tr.N // 2          # a witness, and the event after it
    for x in (h, h + 1):
        bad = _mutated(wit, x, 1 - wit[x])
        assert lo.first_mismatch("witness", bad[x - 10:x + 10], lo.expected_witness(rnd, tr.p0, x - 10, 20)) is not None
        with pytest.raises(AssertionError, match="witness"):
            lo.check_witness_table(r["witness_table"], bad, rnd, tr.creator, tr.N // 2, [(tr.N // 2, tr.N)])


def test_chunked_comparison_catches_one_element():
    rows = np.arange(50000 * 8, dtype=np.int32).reshape(50000, 8)
    lo.compare_rows("rows", _source(rows), _source(rows.copy()), 3, 49990, chunk=4096)
    bad = _mutated(rows, (41000, 5), -1)
    with pytest.raises(AssertionError, match=r"rows: 1 elements differ, the first at \(41000, 5\)"):
        lo.compare_rows("rows", _source(rows), _source(bad), 3, 49990, chunk=4096)
    with pytest.raises(AssertionError, match="shape"):
        lo.assert_equal("rows", rows[:10], rows[:9])


def test_gather_rows_in_ranges():
    rows = np.arange(30000 * 4, dtype=np.int32).reshape(30000, 4)
    calls = []

    def get(first, n):
        calls.append((first, n))
        return rows[first:first + n]
    idx = np.array([29999, 5, 5, 6, 9000, 4100, 29000, 0])
    assert np.array_equal(lo.gather_rows(get, idx, 4), rows[idx])
    assert calls == [(0, 4101), (9000, 1), (29000, 1000)]
