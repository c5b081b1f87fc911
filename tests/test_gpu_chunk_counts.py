"""The per-member counts that group a chunk's events by creator come from snapshots the host takes while it appends
(every 4096 events, and at the end of every append that is not divided yet), for both kernel families.  Chunks that
end inside appends, an append much longer than a chunk, an append refused half-way through (the snapshots it took
before the refusal must go with it), and many small appends divided, rewound and divided again with another schedule."""
import numpy as np
import pytest

# (member count, SW_FORCE_WIDE): the M <= 64 kernels, and the any-M kernels below and above 64 members
FAMILIES = [(8, "0"), (8, "1"), (97, "0")]


def _run(e, tr, K):
    """divide_rounds + decide_fame over the appended trace with the call schedule K; results() + new_c per call."""
    from swirld_b200 import traces
    ncs = []
    for first, cnt in traces.chunks(tr.N, K):
        e.divide_rounds(first, cnt)
        ncs.append(sorted(e.decide_fame()))
    got = e.results()
    got["new_c_per_call"] = ncs
    return got


def _oracle(tr, K):
    import oracle as orc
    exp = orc.run_oracle(tr, K)
    exp["oracle"].close()
    return exp


def _refused_append(M, seed):
    """Chunks of 3001 events around an append refused after it crossed a 4096-event snapshot, against the oracle."""
    from swirld_b200 import engine, traces
    from util import assert_same
    tr = traces.gossip(M, 20000, seed=seed)
    K = 3001                                        # no chunk ends where an append ends; the last chunk is grid-wide
    e = engine.Engine(tr.M, tr.N)
    e.append_trace(tr, 0, 9000)
    # 4999 valid events of one member (past the snapshot at 12288), then a second root of that member: refused whole
    n, c0 = 5000, int(tr.creator[8999])
    other = max(i for i in range(9000) if tr.creator[i] != c0)
    p0 = np.array([8999] + list(range(9000, 9000 + n - 2)) + [-1], np.int32)
    p1 = np.array([other] * (n - 1) + [-1], np.int32)
    with pytest.raises(engine.EngineError):
        e.append(p0, p1, np.full(n, c0, np.int32), np.zeros(n), np.zeros((n, 64), np.uint8))
    assert e.n_events == 9000
    e.append_trace(tr, 9000, tr.N - 9000)
    assert_same(_oracle(tr, K), _run(e, tr, K), keys=["round", "witness_table", "famous", "consensus"],
                what="refused append, M=%d" % M)


@pytest.mark.gpu
def test_chunk_counts_after_a_refused_append():
    _refused_append(8, 5)


@pytest.mark.gpu
@pytest.mark.parametrize("M,force", [(8, "1"), (97, "0")])
def test_wide_chunk_counts_after_a_refused_append(M, force, monkeypatch):
    """The any-M kernels group their chunks from the same snapshots."""
    monkeypatch.setenv("SW_FORCE_WIDE", force)
    _refused_append(M, 6)


@pytest.mark.gpu
@pytest.mark.parametrize("M,force", FAMILIES)
def test_chunk_counts_small_appends_rewind(M, force, monkeypatch):
    """Three events per append (the reference's cadence), a divide every 40 appends, then sw_rewind and the whole
    trace again with a different schedule: after the rewind the counts come from the 4096-event snapshots alone (the
    end-of-append ones below the divided events are gone), and chunks start where no append ended."""
    from swirld_b200 import engine, traces
    from util import assert_same
    monkeypatch.setenv("SW_FORCE_WIDE", force)
    tr = traces.gossip(M, 9000, seed=8)
    K1, K2 = 120, 1999
    e = engine.Engine(tr.M, tr.N)
    ncs = []
    for first in range(0, tr.N, 3):
        e.append_trace(tr, first, min(3, tr.N - first))
        if e.n_events % K1 == 0 or e.n_events == tr.N:
            d = e.n_divided
            e.divide_rounds(d, e.n_events - d)
            ncs.append(sorted(e.decide_fame()))
    got = e.results()
    got["new_c_per_call"] = ncs
    keys = ["round", "witness_table", "famous", "consensus"]
    assert_same(_oracle(tr, K1), got, keys=keys, what="small appends, M=%d" % M)
    e.rewind()
    assert_same(_oracle(tr, K2), _run(e, tr, K2), keys=keys, what="after rewind, M=%d" % M)


@pytest.mark.gpu
@pytest.mark.parametrize("M,force", FAMILIES)
def test_divide_rounds_launches(M, force, monkeypatch):
    """Kernels per divide_rounds call once the can_see rows are there: the chunk's grouping (k_rb_prep), the round
    kernel and the three that follow it, in both families; at M <= 64 the cluster round kernel adds one."""
    from swirld_b200 import engine, traces
    monkeypatch.setenv("SW_FORCE_WIDE", force)
    tr = traces.gossip(M, 8192, seed=9)
    e = engine.Engine(tr.M, tr.N)
    e.append_trace(tr)                              # (one append of >= 4096 events: its can_see scan runs right here)
    per_call = []
    for first, cnt in traces.chunks(tr.N, 4096):
        before = e.stats()["kernel_launches"]
        e.divide_rounds(first, cnt)
        st = e.stats()
        per_call.append(st["kernel_launches"] - before)
    cluster = e.stats()["rounds_cluster_launches"]
    assert per_call == [5 + (1 if cluster else 0)] * 2
    if force == "1" or M > 64:
        assert cluster == 0
