"""Pins the oracle (oracle/swirld_oracle.c) to the reference: every committed
fixture under tests/golden/ was produced by the UNMODIFIED reference
(oracle/make_golden.py); the C restatement must reproduce it bit for bit --
rounds, witness table, famous tri-state, consensus set, per-call new_c and the
final consensus order -- under the same call schedule."""
import hashlib

import numpy as np
import pytest

import golden_specs as gs
import oracle as orc
from util import assert_same, load_golden

SMALL = [n for n in gs.SPECS if gs.SPECS[n][1]["N"] <= 20000]
LARGE = [n for n in gs.SPECS if gs.SPECS[n][1]["N"] > 20000]


def _check(name):
    tr, K, stake = gs.make_trace(name)
    g = load_golden(name)
    sha = hashlib.sha256(tr.p0.tobytes() + tr.p1.tobytes() + tr.creator.tobytes() + tr.t.tobytes()
                         + tr.sig.tobytes()).digest()
    assert bytes(g["trace_sha256"]) == sha, "trace generator drifted from the fixture"
    o = orc.run_oracle(tr, K, stake)
    assert_same(g, o, what=name)
    cs = o["oracle"].can_see()
    assert bytes(g["can_see_sha256"]) == hashlib.sha256(cs.tobytes()).digest(), name + ": can_see differs"
    if "can_see" in g:
        assert np.array_equal(g["can_see"], cs)


@pytest.mark.parametrize("name", SMALL)
def test_oracle_matches_reference_fixture(name):
    _check(name)


@pytest.mark.parametrize("name", LARGE)
def test_oracle_matches_reference_fixture_large(name):
    _check(name)


@pytest.mark.parametrize("M,N,K,seed", [(4, 600, 1, 11), (5, 900, 13, 12), (16, 3000, 250, 13)])
def test_oracle_matches_live_reference(M, N, K, seed):
    """A gossip and an adversarial trace each, against what the reference computed on them (stored fixtures)."""
    for gen in ("g1", "g2"):
        _check("%s_m%d_n%d_s%d_k%d" % (gen, M, N, seed, K))


def test_oracle_index_error_single_seer():
    """swirld.py:305 raises IndexError when only one famous witness sees an
    event; the oracle reports it instead of inventing a timestamp.  Member 0
    holds all the stake, so its witness alone decides "received"."""
    from swirld_b200 import traces
    tr = traces.gossip(4, 1000, 1)
    o = orc.Oracle(4, [1, 0, 0, 0])
    o.append(tr)
    o.divide_rounds(0, 20)
    nc = o.decide_fame()
    assert nc
    with pytest.raises(IndexError):
        o.find_order(nc)
    assert o.coverage()["single_seer"] == 1
