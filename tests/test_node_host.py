"""The bound node's host logic on CPU: a gossip simulation (real Ed25519 signatures, BLAKE2b ids, random peers)
runs over `bind(host)` with the oracle standing in for the device, over the tests' own host; every node's state must
equal a replay of its own arrival trace and call schedule through the oracle, and the oracle's replay of stored node
traces must equal the unmodified reference's."""
import pytest

import node_sim
from oracle_engine import OracleEngine
from util import assert_same

KEYS = ["round", "famous", "consensus", "transactions"]


@pytest.fixture(scope="module")
def sim():
    return node_sim.run_sim(4, 400, OracleEngine, capacity=64, seed=5)   # small capacity: forces growth replay


def test_transactions_are_consistent(sim):
    # prefix agreement between nodes is NOT a property of the reference (its final order
    # depends on each node's call schedule, SURVEY.md section 0.5); each node's own state is
    # pinned against the oracle / the reference below.
    for nd in sim:
        assert len(nd.transactions) > 20
        assert len(set(nd.transactions)) == len(nd.transactions)


def test_views_and_attributes(sim):
    nd = sim[0]
    h = nd.head
    assert nd.hg[h].c == nd.pk and nd.height[h] >= 1
    assert nd.can_see[h][nd.pk] == h
    assert nd.round[h] >= nd.round[nd.hg[h].p[0]]
    assert set(nd.idx) == set(nd.transactions)
    assert [nd.idx[x] for x in nd.transactions] == list(range(len(nd.transactions)))
    assert nd.tbd == set(nd.hg) - set(nd.transactions)
    r0 = nd.witnesses[0]
    assert set(r0) <= set(nd.stake) and all(nd.round[w] == 0 for w in r0.values())
    fam = [x for x in nd.hg if x in nd.famous]
    assert fam and all(isinstance(nd.famous[x], bool) for x in fam)
    assert nd.famous.get(b"nope") is None
    with pytest.raises(KeyError):
        nd.round[b"nope"]


def test_each_node_matches_oracle_replay(sim):
    for nd in sim:
        tr, sizes = node_sim.node_trace(nd)
        assert_same(node_sim.replay_oracle(tr, sizes), node_sim.node_results(nd), KEYS, "node vs oracle replay")


def test_each_node_matches_reference_replay():
    """Two nodes' arrival traces and call schedules from a simulation like `sim`, and three node views of generator
    traces at 8, 16 and 33 members (traces.node_view), stored with the reference's replay of each (tests/golden,
    oracle/make_golden.py --nodes / --views): the oracle's replay must equal it."""
    import golden_specs as gs
    import numpy as np
    from swirld_b200.traces import Trace
    for name in gs.NODE_FIXTURES + list(gs.VIEW_FIXTURES):
        z = np.load(gs.path(name))
        tr = Trace(int(z["M"]), z["p0"], z["p1"], z["creator"], z["t"], z["sig"], name)
        if name in gs.VIEW_FIXTURES:                     # node_view still builds the view the reference replayed
            view, sizes = gs.make_view(name)
            assert sizes == z["sizes"].tolist(), name
            for k in ("p0", "p1", "creator", "t", "sig"):
                assert np.array_equal(getattr(view, k), z[k]), "%s: %s differs from node_view's" % (name, k)
        assert_same(z, node_sim.replay_oracle(tr, z["sizes"].tolist()), KEYS, name + ": oracle replay vs reference")


def test_forked_events_are_dropped_not_fatal():
    """A Byzantine peer's fork (a second event on the same self-parent) is treated as invalid: the node keeps working
    and its device state stays consistent (the reference would accept the fork; the engine's contract is fork-free)."""
    import host_sim
    nodes = node_sim.run_sim(3, 60, OracleEngine, seed=9)
    a, b = nodes[0], nodes[1]
    # b forges a sibling of its own head: same self-parent, other other-parent
    sp = b.hg[b.head].p
    assert sp
    other = next(h for h in b.hg if b.hg[h].c != b.pk and h != sp[1])
    h2, ev2 = host_sim.HostNode.new_event(b, "fork", (sp[0], other))
    assert host_sim.HostNode.is_valid_event(a, h2, ev2) or other not in a.hg or sp[0] not in a.hg
    n_before = len(a.hg)
    if sp[0] in a.hg and other in a.hg and a._heads.get(b.pk) != sp[0]:
        assert not a.is_valid_event(h2, ev2)             # a already holds b's real event on that self-parent
    # a second root is always a fork
    hr, evr = host_sim.HostNode.new_event(b, None, ())
    assert not a.is_valid_event(hr, evr)
    assert len(a.hg) == n_before
    loop = a.main()
    next(loop)
    loop.send(None)                                      # the node still gossips and advances
    assert len(a.hg) > n_before
    tr, sizes = node_sim.node_trace(a)
    assert_same(node_sim.replay_oracle(tr, sizes), node_sim.node_results(a), KEYS, "after the rejected fork")


def test_non_integral_stake_is_refused():
    import host_sim
    import sodium
    kp = sodium.crypto_sign_keypair()
    with pytest.raises(ValueError):
        node_sim.bound_class(host_sim.HostNode, OracleEngine)(kp, {}, 1, {kp[0]: 1.5})
