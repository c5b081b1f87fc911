"""Every kernel family past 2^31 table elements.

The can_see table (`row`, N x M int32) passes 2^31 elements at 2^25 events for M = 64, and the signature column
(64 bytes per event) passes 2^31 bytes at the same event.  C5 (1024 x 8 M) runs there on every chunk after its first,
so every offset the kernels and the host compute into these arrays must be 64-bit; a missing cast shows only here.

- M = 64, N = 2^25 + 2^20: both kernel families (the default cluster / round-stream path, and the any-M kernels that
  SW_FORCE_WIDE=1 selects) against one oracle run, element for element: rounds, witness flags and table, fame,
  consensus, new rounds per call, the order and its idx, can_see (one fetch of more than 2^31 bytes across event 2^25),
  consensus times and rounds received from 2^25 - 2^16 on, 64 batched turns beside a 20 000-event view with its own
  oracle, and single calls of 1 to 16 events at the end.  The default-family run also answers a sync request at the head.
- M = 1024, N = 2^21 + 2^18: past the oracle's reach, so the can_see recurrence, the rounds and the witness flags are
  restated in numpy (tests/large_offsets.py, checked against the oracle in tests/test_large_offsets_model.py) around
  event 2^21, from the first round step after that, and at the end; then a sync request, and a checkpoint round trip
  followed by three calls on both engines.

Each test skips, with the numbers, when the device or the host has less free memory than it needs, and prints its wall
time and the peak device and host memory it saw (run pytest with -s to see them)."""
import os
import resource
from concurrent.futures import ThreadPoolExecutor
import shutil
import tempfile
import time

import numpy as np
import pytest

import large_offsets as lo
import oracle as orc
from swirld_b200 import engine as E
from swirld_b200 import traces

pytestmark = pytest.mark.gpu

GB = 1 << 30
B31 = 1 << 31

# ---- M = 64
PAST64 = 1 << 25                     # the first event whose row starts past 2^31 elements (and whose signature past 2^31 bytes)
M64, N64, SEED64 = 64, PAST64 + (1 << 20), 25
K64 = 49157                          # not a power of two: event 2^24 and 2^25 fall inside calls (and round-stream pieces)
TAIL = [1, 3, 16] * 51 + [1, 3]      # the last 1024 events, one launch each (k_stream_divide)
BIG_TURNS = [1, 16, 17, 300, 5, 2048, 3, 4097] * 8           # the big view's 64 batched turns
SMALL_TURNS = [7, 16, 400, 211, 2, 1200, 9, 333] * 8         # ... and the 20 000-event view's
SMALL_N, SMALL_SEED = 20000, 26
# ---- M = 1024
PAST1K = 1 << 21                     # ... at M = 1024
M1K, N1K, SEED1K = 1024, PAST1K + (1 << 18), 27
K1K, OFF1K = 262144, 12345


def _host_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def _guard(device_bytes, host_bytes):
    import torch
    free, total = torch.cuda.mem_get_info()
    host = _host_available()
    if free < device_bytes or host < host_bytes:
        pytest.skip("needs %.1f GB of free device memory (%.1f of %.1f free) and %.1f GB of available host memory "
                    "(%.1f available)" % (device_bytes / GB, free / GB, total / GB, host_bytes / GB, host / GB))
    return free


class _Peak:
    """Wall time, and the peak device memory in use (sampled, above the free memory at the start, or at `since`'s start)
    and the peak host RSS of the process, for one test or fixture."""

    def __init__(self, what, since=None):
        import torch
        self.torch, self.what, self.t0 = torch, what, time.time()
        self.free0 = torch.cuda.mem_get_info()[0] if since is None else since.free0
        self.used = 0 if since is None else since.used

    def sample(self):
        self.used = max(self.used, self.free0 - self.torch.cuda.mem_get_info()[0])

    def report(self):
        self.sample()
        print("\n%s: %.0f s, peak device memory %.1f GB (sampled, above the start), peak host RSS %.1f GB" % (
            self.what, time.time() - self.t0, self.used / GB,
            resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024 / GB), flush=True)


def _sizes(sizes, first=0):
    out = []
    for n in sizes:
        out.append((first, n))
        first += n
    return out


def schedule64():
    """(single calls of K64, the big view's batched turns, the single calls of the tail) as (first, n)."""
    head = N64 - sum(TAIL) - sum(BIG_TURNS)
    single = list(traces.chunks(head, K64))
    turns = _sizes(BIG_TURNS, head)
    tail = _sizes(TAIL, head + sum(BIG_TURNS))
    assert sum(TAIL) == 1024 and tail[-1][0] + tail[-1][1] == N64
    return single, turns, tail


def small_schedule():
    """The 20 000-event view: one call before the turns, then one call per turn."""
    pre = SMALL_N - sum(SMALL_TURNS)
    return (0, pre), _sizes(SMALL_TURNS, pre)


def _oracle_run(tr, calls, progress=0):
    """The oracle over calls [(first, n)]: results, new rounds per call, the rounds received of its order (one
    find_order per round, tests/order_meta.py), idx and heights.  progress: print a line every that many calls."""
    o = orc.Oracle(tr.M)
    o.append(tr)
    L = orc.lib()
    ncs, rr = [], []
    t0 = time.time()
    for i, (first, n) in enumerate(calls):
        if progress and i % progress == 0:
            print("oracle, M = %d: %d of %d events, %.0f s" % (tr.M, first, tr.N, time.time() - t0), flush=True)
        o.divide_rounds(first, n)
        nc = sorted(o.decide_fame())
        ncs.append(nc)
        for r in nc:
            before = L.or_n_transactions(o._h)
            o.find_order([r])
            rr += [r] * (L.or_n_transactions(o._h) - before)
    res = o.results()
    res["new_c_per_call"] = ncs
    res["round_received"] = np.array(rr, np.int32)
    res["idx"] = np.empty(o.n, np.int32)
    L.or_get_idx(o._h, res["idx"])
    res["height"] = np.empty(o.n, np.int32)
    L.or_get_height(o._h, res["height"])
    return o, res


@pytest.fixture(scope="module")
def big64():
    """The M = 64 trace, the 20 000-event view with its oracle results, and the big trace's oracle run, which goes on
    in a thread (the oracle's calls release the GIL) while the first test runs its engine: (o, results) = .result()."""
    _guard(0, 32 * GB)
    t0 = time.time()
    tr = traces.gossip_np(M64, N64, SEED64)
    single, turns, tail = schedule64()

    def run():
        out = _oracle_run(tr, single + turns + tail, progress=100)
        print("M = 64 oracle run over %d events: %.0f s with the trace" % (N64, time.time() - t0), flush=True)
        return out
    pool = ThreadPoolExecutor(1)
    big = pool.submit(run)
    small = traces.gossip(M64, SMALL_N, SMALL_SEED)
    pre, sturns = small_schedule()
    so, sres = _oracle_run(small, [pre] + sturns)
    sres["can_see"] = so.can_see()
    so.close()
    yield tr, big, small, sres
    big.result()[0].close()
    pool.shutdown()


def _check_view(what, exp, e, ncs):
    for k in ("round", "witness", "witness_table", "famous", "consensus", "transactions", "idx"):
        got = {"round": e.rounds, "witness": e.witness_flags, "witness_table": e.witness_table, "famous": e.famous,
               "consensus": e.consensus, "transactions": e.transactions, "idx": e.idx}[k]()
        lo.assert_equal("%s: %s" % (what, k), exp[k], got)
    bad = [i for i, (a, b) in enumerate(zip(exp["new_c_per_call"], ncs)) if list(a) != list(b)]
    assert len(ncs) == len(exp["new_c_per_call"]) and not bad, "%s: new rounds differ at calls %s" % (what, bad[:5])


@pytest.mark.parametrize("family", ["default", "wide"])
def test_m64_past_2_31_against_oracle(big64, family, monkeypatch):
    tr, big, small, sres = big64
    monkeypatch.setenv("SW_FORCE_WIDE", "1" if family == "wide" else "0")
    _guard(16 * GB, 8 * GB)
    peak = _Peak("M = 64, %s family" % family)
    single, turns, tail = schedule64()
    (spre, sturns) = small_schedule()
    e = E.Engine(M64, N64)
    s = E.Engine(M64, SMALL_N)
    peak.sample()
    ncs, sncs, batched = [], [], []

    def one(first, n):
        e.append_trace(tr, first, n)
        e.divide_rounds(first, n)
        nc = e.decide_fame()
        e.find_order_out(nc)
        ncs.append(sorted(nc))
    for first, n in single:
        one(first, n)
    s.append_trace(small, *spre)
    s.divide_rounds(*spre)
    nc = s.decide_fame()
    s.find_order(nc)
    sncs.append(sorted(nc))
    # 64 batched turns, the big view past 2^31 beside the small one (the any-M kernels take calls of more than 16
    # events one view at a time: sw_batch_divide_rounds refuses them)
    views = [e, s]
    for (bf, bn), (sf, sn) in zip(turns, sturns):
        E.batch_append(views, [tuple(getattr(x.slice(f, f + n), k) for k in ("p0", "p1", "creator", "t", "sig"))
                               for x, f, n in ((tr, bf, bn), (small, sf, sn))])
        if family == "default" or max(bn, sn) <= 16:
            E.batch_divide_rounds(views, [bf, sf], [bn, sn])
        else:
            e.divide_rounds(bf, bn)
            s.divide_rounds(sf, sn)
        nb, ns = E.batch_decide_fame(views)
        outs = E.batch_find_order_out(views, [nb, ns])
        batched.append(outs[0])
        ncs.append(sorted(nb))
        sncs.append(sorted(ns))
    for first, n in tail:
        one(first, n)
    peak.sample()

    o, res = big.result()
    # the small view against its own oracle
    _check_view("20 000-event view", sres, s, sncs)
    lo.assert_equal("20 000-event view: can_see", sres["can_see"], s.can_see())
    s.close()
    # the big view against the oracle
    assert e.n_divided == N64 and (e.n_divided - 1) * M64 >= B31
    _check_view("M = 64, %s" % family, res, e, ncs)
    a, n = PAST64 - PAST64 // 4, N64 - PAST64 + PAST64 // 4       # one fetch of 2.4 GB: from 2^25 - 2^23 to the end
    assert n * M64 * 4 > B31 and a < PAST64 < a + n
    lo.assert_equal("can_see [%d, %d)" % (a, a + n), o.can_see(a, n), e.can_see(a, n), offset=a)
    lo.compare_rows("can_see", o.can_see, e.can_see, 0, a)
    # the batched turns returned what the order holds
    tx = e.transactions()
    ts, rr = e.consensus_times(), e.rounds_received()
    ev = np.concatenate([b[0] for b in batched])
    at = np.flatnonzero(np.isin(tx, ev))
    lo.assert_equal("batched find_order_out: events", tx[at], ev)
    lo.assert_equal("batched find_order_out: times", ts[at], np.concatenate([b[1] for b in batched]))
    lo.assert_equal("batched find_order_out: rounds received", rr[at], np.concatenate([b[2] for b in batched]))
    # consensus times and rounds received of every event ordered from 2^25 - 2^16 on
    sel = np.flatnonzero(tx >= PAST64 - PAST64 // 512)
    lo.assert_equal("rounds received", res["round_received"][sel], rr[sel])
    exp_ts = lo.consensus_times(e.can_see, N64, tr.p0, tr.creator, tr.t, res["witness_table"], res["famous"],
                                tx[sel].astype(np.int64), rr[sel])
    lo.assert_equal("consensus times", exp_ts, ts[sel])
    # coverage: these checks reached the events past 2^31 row elements (and 2^31 signature bytes)
    past = PAST64
    wit = np.flatnonzero(res["witness"])
    n_past = N64 - past
    assert (wit >= past).sum() > n_past // 1000 and (np.flatnonzero(res["famous"] == 1) >= past).sum() > n_past // 1000
    assert (res["transactions"] >= past).sum() > n_past // 2 and sel.size > n_past // 2
    assert any(n <= 16 and f >= past for f, n in tail)
    if family == "default":
        assert e.stats()["rounds_cluster_launches"] > 0
        # a sync request at the head, with a summary taken 500 events earlier
        head, old = N64 - 1, N64 - 501
        S, S_old, reply = lo.sync_expected({head: e.can_see(head, 1)[0], old: e.can_see(old, 1)[0]}, res["height"],
                                           tr.creator, head, old)
        lo.assert_equal("sync summary", S, e.sync_summary(head))
        lo.assert_equal("sync reply", reply, e.sync_reply(head, S_old, rows=False))
        assert reply.size > 100
    else:
        assert e.stats()["rounds_cluster_launches"] == 0
    peak.report()
    e.close()


# ---------------------------------------------------------------- M = 1024 past 2^31 row elements
def schedule1k():
    """One call of OFF1K events, then calls of K1K (2^21 falls inside one), then 64 calls of 1 to 16 events."""
    tail = [int(x) for x in np.random.default_rng(SEED1K).integers(1, 17, 64)]
    head = N1K - sum(tail)
    calls = [(0, OFF1K)] + [(OFF1K + f, n) for f, n in traces.chunks(head - OFF1K, K1K)] + _sizes(tail, head)
    assert any(f < PAST1K < f + n for f, n in calls if n == K1K)
    return calls


@pytest.fixture(scope="module")
def run1k():
    """The M = 1024 engine through every call but the last three (the checkpoint test makes those)."""
    _guard(24 * GB, 6 * GB)
    peak = _Peak("M = 1024 run")
    tr = traces.gossip_np(M1K, N1K, SEED1K)
    calls = schedule1k()
    e = E.Engine(M1K, N1K)
    for first, n in calls[:-3]:
        e.append_trace(tr, first, n)
        e.divide_rounds(first, n)
        e.find_order(e.decide_fame())
    peak.report()
    yield tr, calls, e, peak
    e.close()


def test_m1024_past_2_31_recurrences(run1k):
    tr, calls, e, run = run1k
    peak = _Peak("M = 1024 recurrences", since=run)
    n = e.n_divided
    assert (n - 1) * M1K >= B31 and n == calls[-3][0]
    height = traces.heights(tr)
    lo.check_can_see(e.can_see, tr.p0, tr.p1, tr.creator, height, PAST1K - PAST1K // 8, n - PAST1K + PAST1K // 8, M1K)
    rnd, wit = e.rounds(), e.witness_flags()
    # besides the events around 2^21 and the last ones: 2048 events from the first one after those around 2^21 whose
    # round exceeds both parents' rounds, so that the `> min_s` tests pass at least once past 2^31 row elements
    h = np.arange(PAST1K + 2048, n)
    h = h[tr.p0[h] >= 0]
    step = h[rnd[h] > np.maximum(rnd[tr.p0[h]], rnd[tr.p1[h]])]
    assert step.size, "no round step after event %d" % (PAST1K + 2048)
    s0 = int(step[0])
    windows = [(PAST1K - 2048, PAST1K + 2048), (s0, min(s0 + 2048, n)), (n - 2048, n)]
    for a, b in windows:
        exp = lo.expected_rounds(e.can_see, rnd, np.ones(M1K, np.int64), tr.p0, tr.p1, height, a, b - a, M1K)
        lo.assert_equal("round", exp, rnd[a:b], offset=a)
        lo.assert_equal("witness", lo.expected_witness(rnd, tr.p0, a, b - a), wit[a:b], offset=a)
    assert sum(int(wit[a:b].sum()) for a, b in windows) > 10
    lo.check_witness_table(e.witness_table(), wit, rnd, tr.creator, PAST1K, windows)
    head, old = n - 1, n - 501
    S, S_old, reply = lo.sync_expected({head: e.can_see(head, 1)[0], old: e.can_see(old, 1)[0]}, height, tr.creator,
                                       head, old)
    lo.assert_equal("sync summary", S, e.sync_summary(head))
    lo.assert_equal("sync reply", reply, e.sync_reply(head, S_old, rows=False))
    assert reply.size > 100
    peak.report()


def test_m1024_checkpoint_then_three_calls(run1k):
    tr, calls, e, run = run1k
    peak = _Peak("M = 1024 checkpoint", since=run)
    need = e.n_events * (M1K * 4 + 200) + (256 << 20)
    tmp = tempfile.gettempdir()
    room = shutil.disk_usage(tmp).free
    if room < need * 1.1:
        pytest.skip("the checkpoint needs about %.1f GB in %s, which has %.1f GB free" % (need / GB, tmp, room / GB))
    path = os.path.join(tempfile.mkdtemp(), "m1024.swb")
    try:
        e.save(path)
        f = E.Engine.load(path, capacity=N1K)
    finally:
        if os.path.exists(path):
            os.remove(path)
        os.rmdir(os.path.dirname(path))
    peak.sample()
    outs = []
    for x in (e, f):
        for first, n in calls[-3:]:
            x.append_trace(tr, first, n)
            x.divide_rounds(first, n)
            x.find_order(x.decide_fame())
        r = x.results()
        r.update(idx=x.idx(), ts=x.consensus_times(), rr=x.rounds_received())
        outs.append(r)
    for k in outs[0]:
        lo.assert_equal("after the checkpoint: %s" % k, outs[0][k], outs[1][k])
    assert e.n_divided == f.n_divided == N1K
    lo.compare_rows("can_see after the checkpoint", e.can_see, f.can_see, 0, N1K)
    f.close()
    peak.report()
