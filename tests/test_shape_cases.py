"""The cases of tests/shape_cases.py reach the sizes they are there for.  Runs the oracle only (no GPU), so a generator
or schedule change that shrinks a case fails here, before any parity run could pass without filling a window.  Run
with -rA or -s to see each case's sizes."""
import numpy as np
import pytest

import fame_cases as fc
import shape_cases as sc
from util import assert_same


@pytest.mark.parametrize("name", list(sc.CASES))
def test_case_exceeds_its_sizes(name):
    case = sc.CASES[name]
    s = sc.sizes(case)
    print("%s: %s" % (name, " ".join("%s=%d" % kv for kv in sc.short(s).items())))
    assert not sc.missing(case, s), "%s no longer exceeds %s" % (name, sc.missing(case, s))
    # find_order one round at a time orders what the per-call run orders
    r = fc.run_oracle(case)
    assert r["raised_at"] == -1
    assert_same(r, s, what=name + ": find_order per round vs per call")


def test_partition_generator():
    """Inside [start, end) every event's peer is on the creator's own side; outside, both sides meet; the default
    split is M // 2 and each side needs two members."""
    from swirld_b200 import traces
    M, N, start, end = 10, 6000, 1000, 4000
    tr = traces.partition(M, N, seed=4, start=start, end=end)
    assert tr.N == N and np.array_equal(tr.creator[:M], np.arange(M)) and np.all(tr.p0[:M] == -1)
    side = lambda e: tr.creator[e] >= M // 2
    i = np.arange(M, N)
    same = side(i) == side(tr.p1[i])
    inside = (i >= start) & (i < end)
    assert same[inside].all() and not same[~inside].all()
    assert np.all(tr.creator[tr.p1[i]] != tr.creator[i])
    assert np.all(tr.creator[tr.p0[i]] == tr.creator[i])
    assert np.array_equal(tr.p0, traces.partition(M, N, seed=4, split=M // 2, start=start, end=end).p0)
    with pytest.raises(AssertionError):
        traces.partition(M, N, split=1)
    with pytest.raises(AssertionError):
        traces.partition(M, N, split=M - 1)
