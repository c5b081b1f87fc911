"""The counters of every call, single and batched: the kernel launches, the bytes copied each way and the launches of
the cluster round kernel that sw_stats reports for sw_append, sw_divide_rounds, sw_decide_fame and sw_find_order and
for their sw_batch_* forms.  The single and batched calls share their launch code; these numbers pin what each call
costs, so that a change to that code which adds or drops a launch or a copy on either side shows up here.

Each case runs two views through one schedule twice: once with single calls, once with the batched calls (where the
batched divide would refuse the call, a call of more than 16 events in the any-M family, the views divide one by one).
Schedules: the reference's cadence (3 events per call), a 4096-event chunk (the eager can_see scan, and the cluster
round kernel at M <= 64), a 17-event call (the chunk path) and, at M = 8, one call with more than 1024 new rounds
(decide_fame's second copy)."""
import pytest

import test_gpu_batch_consensus as tbc

pytestmark = pytest.mark.gpu

KEYS = ("kernel_launches", "h2d_bytes", "d2h_bytes", "rounds_cluster_launches")
CALLS = ("append", "divide", "fame", "order", "batch_append", "batch_divide", "batch_fame", "batch_order")
CADENCE = (3, 4096, 3, 17)
# name: (M, SW_FORCE_WIDE, trace events, schedule)
CASES = {
    "m8": (8, "0", sum(CADENCE), CADENCE),
    "m8_wide": (8, "1", sum(CADENCE), CADENCE),
    "m64": (64, "0", sum(CADENCE), CADENCE),
    "m64_wide": (64, "1", sum(CADENCE), CADENCE),
    "m97": (97, "0", sum(CADENCE), CADENCE),
    "m8_1024_rounds": (8, "0", 60000, 60000),
    "m8_wide_1024_rounds": (8, "1", 60000, 60000),
}


def _counters(engs):
    return [[e.stats()[k] for k in KEYS] for e in engs]


def run_case(name, monkeypatch):
    """Per call of the case's schedule, per call in CALLS: the increments of KEYS summed over the two views."""
    from swirld_b200 import engine
    M, force_wide, N, K = CASES[name]
    monkeypatch.setenv("SW_FORCE_WIDE", force_wide)
    wide = M > 64 or force_wide == "1"
    trs = [tbc._gossip(M, N, 500 + v, K).trace() for v in range(2)]
    single = [engine.Engine(M, N) for _ in trs]
    batched = [engine.Engine(M, N) for _ in trs]
    out = []
    for first, cnt in tbc._gossip(M, N, 500, K).schedule(N):
        row = []

        def step(engs, fn):
            before = _counters(engs)
            r = fn()
            after = _counters(engs)
            row.append([sum(a[k] - b[k] for a, b in zip(after, before)) for k in range(len(KEYS))])
            return r

        s = slice(first, first + cnt)
        step(single, lambda: [e.append_trace(tr, first, cnt) for e, tr in zip(single, trs)])
        step(single, lambda: [e.divide_rounds(first, cnt) for e in single])
        ncs = step(single, lambda: [e.decide_fame() for e in single])
        step(single, lambda: [e.find_order(nc) for e, nc in zip(single, ncs)])
        step(batched, lambda: engine.batch_append(batched, [(tr.p0[s], tr.p1[s], tr.creator[s], tr.t[s], tr.sig[s])
                                                             for tr in trs]))
        if wide and cnt > 16:
            step(batched, lambda: [e.divide_rounds(first, cnt) for e in batched])
        else:
            step(batched, lambda: engine.batch_divide_rounds(batched, [first] * 2, [cnt] * 2))
        bncs = step(batched, lambda: engine.batch_decide_fame(batched))
        step(batched, lambda: engine.batch_find_order(batched, bncs))
        assert [sorted(x) for x in ncs] == [sorted(x) for x in bncs]
        out.append(row)
    for e in single + batched:
        e.close()
    return out


# measured on an H100 before the single and batched calls shared their launch code; per call of the schedule, one
# [kernel_launches, h2d_bytes, d2h_bytes, rounds_cluster_launches] per entry of CALLS
EXPECTED = {
    "m64": [
        [[2, 558, 0, 0], [2, 0, 0, 0], [2, 0, 952, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [2, 256, 8256, 0], [0, 0, 0, 0]],
        [[18, 761856, 0, 0], [12, 0, 0, 2], [2, 0, 952, 0], [10, 32, 64, 0], [18, 761856, 0, 0], [10, 0, 0, 1], [2, 256, 8256, 0], [6, 496, 64, 0]],
        [[2, 558, 0, 0], [2, 0, 0, 0], [2, 0, 952, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [2, 256, 8256, 0], [0, 0, 0, 0]],
        [[2, 3162, 0, 0], [12, 0, 0, 0], [2, 0, 952, 0], [0, 0, 0, 0], [1, 3162, 0, 0], [11, 0, 0, 0], [2, 256, 8256, 0], [0, 0, 0, 0]],
    ],
    "m64_wide": [
        [[2, 558, 0, 0], [2, 0, 0, 0], [6, 0, 952, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [4, 256, 8256, 0], [0, 0, 0, 0]],
        [[18, 761856, 0, 0], [10, 0, 0, 0], [6, 0, 952, 0], [10, 32, 64, 0], [18, 761856, 0, 0], [10, 0, 0, 0], [4, 256, 8256, 0], [6, 496, 64, 0]],
        [[2, 558, 0, 0], [2, 0, 0, 0], [6, 0, 952, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [4, 256, 8256, 0], [0, 0, 0, 0]],
        [[2, 3162, 0, 0], [12, 0, 0, 0], [6, 0, 952, 0], [0, 0, 0, 0], [1, 3162, 0, 0], [12, 0, 0, 0], [4, 256, 8256, 0], [0, 0, 0, 0]],
    ],
    "m8": [
        [[2, 558, 0, 0], [2, 0, 0, 0], [2, 0, 5680, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [2, 256, 8256, 0], [0, 0, 0, 0]],
        [[18, 761856, 0, 0], [12, 0, 0, 2], [2, 0, 5680, 0], [10, 628, 64, 0], [18, 761856, 0, 0], [10, 0, 0, 1], [2, 256, 8256, 0], [6, 1092, 64, 0]],
        [[2, 558, 0, 0], [2, 0, 0, 0], [2, 0, 5680, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [2, 256, 8256, 0], [0, 0, 0, 0]],
        [[2, 3162, 0, 0], [12, 0, 0, 0], [2, 0, 5680, 0], [0, 0, 0, 0], [1, 3162, 0, 0], [11, 0, 0, 0], [2, 256, 8256, 0], [0, 0, 0, 0]],
    ],
    "m8_1024_rounds": [
        [[18, 11160000, 0, 0], [12, 0, 0, 2], [2, 0, 17996, 0], [10, 9740, 64, 0], [18, 11160000, 0, 0], [10, 0, 0, 1], [2, 256, 17996, 0], [6, 10204, 64, 0]],
    ],
    "m8_wide": [
        [[2, 558, 0, 0], [2, 0, 0, 0], [6, 0, 5680, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [4, 256, 8256, 0], [0, 0, 0, 0]],
        [[18, 761856, 0, 0], [10, 0, 0, 0], [6, 0, 5680, 0], [10, 628, 64, 0], [18, 761856, 0, 0], [10, 0, 0, 0], [4, 256, 8256, 0], [6, 1092, 64, 0]],
        [[2, 558, 0, 0], [2, 0, 0, 0], [6, 0, 5680, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [4, 256, 8256, 0], [0, 0, 0, 0]],
        [[2, 3162, 0, 0], [12, 0, 0, 0], [6, 0, 5680, 0], [0, 0, 0, 0], [1, 3162, 0, 0], [12, 0, 0, 0], [4, 256, 8256, 0], [0, 0, 0, 0]],
    ],
    "m8_wide_1024_rounds": [
        [[18, 11160000, 0, 0], [10, 0, 0, 0], [6, 0, 17996, 0], [10, 9740, 64, 0], [18, 11160000, 0, 0], [10, 0, 0, 0], [4, 256, 17996, 0], [6, 10204, 64, 0]],
    ],
    "m97": [
        [[2, 558, 0, 0], [2, 0, 0, 0], [6, 0, 696, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [4, 256, 8256, 0], [0, 0, 0, 0]],
        [[8, 761856, 0, 0], [10, 0, 0, 0], [6, 0, 696, 0], [10, 8, 64, 0], [8, 761856, 0, 0], [10, 0, 0, 0], [4, 256, 8256, 0], [6, 472, 64, 0]],
        [[2, 558, 0, 0], [2, 0, 0, 0], [6, 0, 696, 0], [0, 0, 0, 0], [1, 558, 0, 0], [1, 400, 0, 0], [4, 256, 8256, 0], [0, 0, 0, 0]],
        [[2, 3162, 0, 0], [12, 0, 0, 0], [6, 0, 696, 0], [0, 0, 0, 0], [1, 3162, 0, 0], [12, 0, 0, 0], [4, 256, 8256, 0], [0, 0, 0, 0]],
    ],
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_call_counters(name, monkeypatch):
    got = run_case(name, monkeypatch)
    for i, (want_row, got_row) in enumerate(zip(EXPECTED[name], got)):
        for call, w, g in zip(CALLS, want_row, got_row):
            assert g == w, "%s, call %d, %s: %s" % (name, i, call, dict(zip(KEYS, zip(w, g))))
    assert len(got) == len(EXPECTED[name])
