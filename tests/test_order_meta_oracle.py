"""Consensus timestamps and rounds received on CPU: the oracle's (tests/order_meta.py) equal the unmodified reference's
on every tests/golden/meta_* fixture, bit for bit; and GpuNode's consensus_time / round_received views, over an engine
that reports them with find_order_out, equal the oracle's replay of each node's own trace and call schedule.  The
unchanged OracleEngine, which has no find_order_out, still drives GpuNode the way it always did."""
import glob
import os

import numpy as np
import pytest

import golden_specs as gs
import node_sim
import order_meta
from oracle_engine import OracleEngine
from util import assert_same

META = sorted(os.path.basename(p)[len("meta_"):-len(".npz")]
              for p in glob.glob(os.path.join(gs.GOLDEN_DIR, "meta_*.npz")))


def test_meta_fixtures_present():
    assert len(META) == 19


@pytest.mark.parametrize("name", META)
def test_oracle_matches_reference_meta(name):
    z = np.load(os.path.join(gs.GOLDEN_DIR, "meta_%s.npz" % name))
    tr, K, stake = gs.make_trace(name)
    got = order_meta.run_oracle_meta(tr, K, stake)
    assert np.array_equal(np.load(gs.path(name))["transactions"], z["transactions"])
    assert np.array_equal(got["transactions"], z["transactions"])
    assert got["consensus_time"].dtype == np.float64 and (got["consensus_time"] == z["consensus_time"]).all()
    assert np.array_equal(got["round_received"], z["round_received"])


class OracleEngineOut(OracleEngine):
    """OracleEngine with the engine's find_order_out and getters of consensus times and rounds received."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self._meta = order_meta.OrderMeta(self._o)

    def append(self, p0, p1, creator, t, sig):
        super().append(p0, p1, creator, t, sig)
        self._meta.add_columns(p0, creator, t)

    def find_order(self, new_c):
        return len(self.find_order_out(new_c)[0])

    def find_order_out(self, new_c):
        return self._meta.find_order(new_c, self._nd)

    def consensus_times(self, first=0, n=None):
        v = np.array(self._meta.ts, np.float64)
        return v[first:] if n is None else v[first:first + n]

    def rounds_received(self, first=0, n=None):
        v = np.array(self._meta.rr, np.int32)
        return v[first:] if n is None else v[first:first + n]


def replay_meta(nd):
    tr, sizes = node_sim.node_trace(nd)
    return order_meta.run_oracle_meta(tr, sizes)


def node_meta(nd):
    return {"transactions": np.array([nd._h2i[h] for h in nd.transactions], np.int32),
            "consensus_time": np.array([nd.consensus_time[h] for h in nd.transactions], np.float64),
            "round_received": np.array([nd.round_received[h] for h in nd.transactions], np.int32)}


@pytest.fixture(scope="module")
def sim_out():
    return node_sim.run_sim(4, 400, OracleEngineOut, capacity=64, seed=5)   # small capacity: growth replay too


def test_node_views_match_oracle_replay(sim_out):
    for nd in sim_out:
        assert len(nd.transactions) > 20
        assert_same(replay_meta(nd), node_meta(nd), ["transactions", "consensus_time", "round_received"],
                    "node views vs oracle replay")
        assert len(nd.consensus_time) == len(nd.round_received) == len(nd.transactions)
        assert set(nd.consensus_time) == set(nd.transactions)
        h = next(x for x in nd.hg if x not in nd._order_pos) if len(nd.hg) > len(nd.transactions) else None
        if h is not None:
            assert h not in nd.consensus_time and nd.round_received.get(h) is None
            with pytest.raises(KeyError):
                nd.consensus_time[h]
        assert nd._eng.consensus_times().tolist() == [nd.consensus_time[x] for x in nd.transactions]
        assert nd._eng.rounds_received().tolist() == [nd.round_received[x] for x in nd.transactions]


def test_node_without_find_order_out_behaves_as_before():
    assert not hasattr(OracleEngine, "find_order_out")
    for nd in node_sim.run_sim(4, 400, OracleEngine, capacity=64, seed=5):
        tr, sizes = node_sim.node_trace(nd)
        assert_same(node_sim.replay_oracle(tr, sizes), node_sim.node_results(nd), ["round", "famous", "consensus", "transactions"],
                    "fallback node vs oracle replay")
        assert len(nd.transactions) > 0 and len(nd.consensus_time) == 0 and len(nd.round_received) == 0
