"""The per-member counts that group a chunk's events by creator come from snapshots the host takes while it appends
(every 4096 events and at the end of every append).  Chunks that end inside appends, an append much longer than a
chunk, and an append refused half-way through: the snapshots it took before the refusal must go with it."""
import numpy as np
import pytest


@pytest.mark.gpu
def test_chunk_counts_after_a_refused_append():
    import oracle as orc
    from swirld_b200 import engine, traces
    from util import assert_same
    tr = traces.gossip(8, 20000, seed=5)
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
    ncs = []
    for first, cnt in traces.chunks(tr.N, K):
        e.divide_rounds(first, cnt)
        ncs.append(sorted(e.decide_fame()))
    got = e.results()
    got["new_c_per_call"] = ncs
    exp = orc.run_oracle(tr, K)
    exp["oracle"].close()
    assert_same(exp, got, keys=["round", "witness_table", "famous", "consensus"], what="refused append")
